// map.cu -- HP2: query mapping, stages A..G, and the piece loop that runs stages C..H.
//
// Replaces skch::Map::mapQuery / doL1Mapping / computeL1CandidateRegions / doL2Mapping /
// computeL2MappedRegions (src/map/include/computeMap.hpp:112-497) with SlideMapper
// (slidingMap.hpp) and MIIteratorL2 (MIIteratorL2.hpp).
//
// The reference maps one fragment at a time.  Here a batch of query genomes is cut into
// fragments and every stage runs over ALL fragments (or all hits / all candidates) of a piece
// (<= 2^18 fragments of whole query genomes):
//
//   --- query sketch (QSketch: can be built once, exported, moved between GPUs; qsketch_create) ---
//   A  sketch      fragment minimizers, fragment-local windows (computeMap.hpp:260)      sketch.cu
//   A' from index  for queries that are genomes of the index: the same multiset read from the
//                  index's contig-level records + validity bitmap, no second hashing
//   B  sort/unique per fragment: sorted unique hashes Q, s = |Q| (computeMap.hpp:268-276), packed
//   --- map phase (qsketch_map: one map_piece per piece, one host function per stage) ---
//   C  lookup      Q -> bucket directory -> unique keys -> position lists (:283-299)
//   D+E hits, L1   per fragment in one CTA (hits.cu): gather, sort by record index (monotone in
//                  (seqId, wpos), i.e. the sort of :320), candidate regions of :322-352 as a LOCAL
//                  rule on the sorted hits (a hit starts a region unless its left neighbour
//                  qualifies and overlaps); oversized fragments: device-wide sort path below
//   F  L2          per candidate: sliding super-window over the position-ordered records with
//                  the winnowed-MinHash intersection of slidingMap.hpp restated in rank space:
//                      t* = max{ t : t + #(distinct window hashes not in Q, below q_t) <= s }
//                      shared = #(q_j present in the window, j <= t*)
//                  as a parallel pre-pass (bounds, closed-form event schedule) + a lean sequential
//                  sweep (each event moves t* by at most one)
//   G  report      identity / upper bound from the (s, shared) table, filter >= cutoff (:375-384),
//                  rows in (fragment, candidate) order == callback order of reportL2Mappings
//   H  CGI         the per-pair identity reduction of cgi::computeCGI                      cgi.cu
#include "common.cuh"
#include "cgi_rows.hpp"
#include <algorithm>
#include <cstring>
#include <deque>

namespace bani {

// ------------------------------------------------------------------ B: per-fragment sort + unique
static constexpr int SU_THREADS = 128;
static constexpr int SU_CAP = 4096;

__global__ void __launch_bounds__(SU_THREADS)
sort_unique_kernel(uint32_t *fragHash, const uint32_t *segStart, int32_t F, int32_t *sCount,
                   int *smax, int *err, int minN /* fragments of at most this many raw minimizers are skipped */)
{
  __shared__ uint32_t a[SU_CAP];
  __shared__ uint32_t wsum[SU_THREADS / 32];
  const int f = blockIdx.x, tid = threadIdx.x;
  const uint32_t beg = segStart[f];
  const int n = (int)(segStart[f + 1] - beg);
  if (n <= minN) return;                                   // done by sort_unique_warp_kernel
  if (n > SU_CAP) { if (tid == 0) { atomicExch(err, 1); sCount[f] = 0; } return; }
  if (n == 0) { if (tid == 0) sCount[f] = 0; return; }
  int n2 = 1; while (n2 < n) n2 <<= 1;
  for (int i = tid; i < n2; i += SU_THREADS) a[i] = i < n ? fragHash[beg + i] : 0xFFFFFFFFu;
  __syncthreads();
  for (int k2 = 2; k2 <= n2; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < n2; i += SU_THREADS) {
        int p = i ^ j;
        if (p > i) {
          uint32_t x = a[i], y = a[p];
          bool asc = (i & k2) == 0;
          if ((x > y) == asc) { a[i] = y; a[p] = x; }
        }
      }
      __syncthreads();
    }
  // unique: each thread owns a contiguous run of the sorted array
  const int per = (n + SU_THREADS - 1) / SU_THREADS;
  const int i0 = min(tid * per, n), i1 = min(i0 + per, n);
  uint32_t cnt = 0;
  for (int i = i0; i < i1; i++) cnt += (i == 0 || a[i] != a[i - 1]);
  uint32_t incl = cnt; const int lane = tid & 31, wid = tid >> 5;
  for (int o = 1; o < 32; o <<= 1) { uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) wsum[wid] = incl;
  __syncthreads();
  uint32_t base = 0, total = 0;
  for (int i = 0; i < SU_THREADS / 32; i++) { if (i < wid) base += wsum[i]; total += wsum[i]; }
  uint32_t o = base + incl - cnt;
  for (int i = i0; i < i1; i++) if (i == 0 || a[i] != a[i - 1]) fragHash[beg + o++] = a[i];
  if (tid == 0) { sCount[f] = (int32_t)total; atomicMax(smax, (int)total); }
}

// Warp per fragment for the common sizes (<= 512 raw minimizers: every default parameter set): the same bitonic network in
// a 2 KB slice of shared memory, warp-synchronous (no block barrier per sub-stage), unique + count by ballots.  Larger
// fragments are counted in *nBig and left to the CTA kernel above.
static constexpr int SUW_CAP = 512;
static constexpr int SUW_WARPS = 4;

__global__ void __launch_bounds__(SUW_WARPS * 32)
sort_unique_warp_kernel(uint32_t *fragHash, const uint32_t *segStart, int32_t F, int32_t *sCount, int *smax, int *nBig)
{
  __shared__ uint32_t sm[SUW_WARPS][SUW_CAP];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int f = blockIdx.x * SUW_WARPS + wid;
  if (f >= F) return;
  uint32_t *a = sm[wid];
  const uint32_t beg = segStart[f];
  const int n = (int)(segStart[f + 1] - beg);
  if (n > SUW_CAP) { if (lane == 0) atomicAdd(nBig, 1); return; }
  if (n == 0) { if (lane == 0) sCount[f] = 0; return; }
  int n2 = 32; while (n2 < n) n2 <<= 1;
  for (int i = lane; i < n2; i += 32) a[i] = i < n ? fragHash[beg + i] : 0xFFFFFFFFu;
  __syncwarp();
  for (int k2 = 2; k2 <= n2; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int t = lane; t < (n2 >> 1); t += 32) {          // pair t: the lower index has bit j clear
        const int i = 2 * t - (t & (j - 1)), p = i + j;
        const uint32_t x = a[i], y = a[p];
        const bool asc = (i & k2) == 0;
        if ((x > y) == asc) { a[i] = y; a[p] = x; }
      }
      __syncwarp();
    }
  uint32_t run = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const bool head = i < n && (i == 0 || a[i] != a[i - 1]);
    const uint32_t bal = __ballot_sync(0xffffffffu, head);
    if (head) fragHash[beg + run + __popc(bal & ((1u << lane) - 1u))] = a[i];
    run += __popc(bal);
  }
  if (lane == 0) { sCount[f] = (int32_t)run; atomicMax(smax, (int)run); }
}

// ------------------------------------------------------------------ C: lookup
__device__ __forceinline__ int seg_of(const uint32_t *segStart, int F, uint32_t t)
{
  int lo = 0, hi = F - 1;          // last f with segStart[f] <= t
  while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (segStart[mid] <= t) lo = mid; else hi = mid - 1; }
  return lo;
}

// Thread per query hash.  One 32-byte sector of the probe table answers almost every probe (hit or miss): bucket = low
// bits of the hash, 4 entries {x = (hash & ~0xFF) | min(count, 255), y = offset}.  Only a full bucket without a match, or a
// saturated count, walks the sorted keys (bucket directory over the top bits, then a short binary search).
// walkCtr (null unless the context counts paths): probes that walked for a saturated count [0] / a full bucket [1].
__global__ void lookup_kernel(const uint32_t *fragHash, uint32_t T, const uint2 *tab, uint32_t tabMask,
                              const uint32_t *ukeys, const uint32_t *uoff, const uint32_t *dir, int dirBits,
                              const uint32_t *filt, uint32_t filtMask, uint32_t *hitLo, uint32_t *hitCnt,
                              unsigned long long *walkCtr)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > T) return;
  if (t == T) { hitCnt[t] = 0; hitLo[t] = 0; return; }
  const uint32_t h = __ldg(&fragHash[t]);
  // small shards: an L2-resident membership bit decides most misses without a DRAM access
  if (filt && !((__ldg(&filt[(h & filtMask) >> 5]) >> (h & 31u)) & 1u)) { hitLo[t] = 0; hitCnt[t] = 0; return; }
  const uint4 *bp = reinterpret_cast<const uint4 *>(tab) + 2 * (size_t)(h & tabMask);
  const uint4 e0 = __ldg(bp), e1 = __ldg(bp + 1);
  const uint32_t key = h & 0xFFFFFF00u;
  const uint32_t ex[4] = {e0.x, e0.z, e1.x, e1.z}, ey[4] = {e0.y, e0.w, e1.y, e1.w};
  uint32_t cnt = 0, lo0 = 0;
  bool full = true, found = false;
#pragma unroll
  for (int sl = 0; sl < 4; sl++) {
    if (ex[sl] == 0u) full = false;
    else if ((ex[sl] & 0xFFFFFF00u) == key) { found = true; cnt = ex[sl] & 0xFFu; lo0 = ey[sl]; }
  }
  if ((found && cnt == 255u) || (!found && full)) {
    if (walkCtr) atomicAdd(&walkCtr[found ? 0 : 1], 1ull);
    cnt = 0; lo0 = 0;
    const uint32_t b = h >> (32 - dirBits);
    uint32_t lo = dir[b], hi = dir[b + 1];
    const uint32_t end = hi;
    while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (ukeys[mid] < h) lo = mid + 1; else hi = mid; }
    if (lo < end && ukeys[lo] == h) { lo0 = uoff[lo]; cnt = uoff[lo + 1] - lo0; }
  }
  hitLo[t] = lo0; hitCnt[t] = cnt;
}

// ------------------------------------------------------------------ D: gather hits as 64-bit keys
__global__ void gather_kernel(const uint32_t *segStart, int32_t F, uint32_t T, const uint32_t *hitLo, const uint32_t *hitCnt,
                              const unsigned long long *hitOff, const uint32_t *posIdx, unsigned long long *keys)
{
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const uint32_t cnt = hitCnt[t];
  if (!cnt) return;
  const unsigned long long f = (unsigned long long)seg_of(segStart, F, t);
  const uint32_t lo = hitLo[t];
  unsigned long long o = hitOff[t];
  for (uint32_t j = 0; j < cnt; j++) keys[o + j] = (f << 32) | posIdx[lo + j];
}

// hit counts of the fragments left to the device-wide path (class 4), zero for everything else
__global__ void mask_hits_kernel(const uint32_t *segStart, int32_t F, uint32_t T, const uint32_t *hitCnt, const uint32_t *fragClass,
                                 uint32_t *bigCnt)
{
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > T) return;
  bigCnt[t] = (t < T && fragClass[seg_of(segStart, F, t)] == (uint32_t)FRAG_NCLASS) ? hitCnt[t] : 0u;
}

// ------------------------------------------------------------------ E: L1 candidate regions (device-wide path)
struct L1Args {
  const unsigned long long *keys; unsigned long long N;
  const uint32_t *segStart; const unsigned long long *hitOff; const int32_t *sCount;
  const int32_t *minHits;          // LUT indexed by s
  const int32_t *recSeq; const int32_t *recWpos;
  int fragLen;
};

// does sorted hit i start a (raw) candidate?  (computeMap.hpp:324-336)
__device__ __forceinline__ bool l1_qual(const L1Args &a, unsigned long long i, unsigned long long fragEnd, int mh,
                                        uint32_t ra, int32_t &start)
{
  if (i + (unsigned long long)mh > fragEnd) return false;
  const uint32_t rb = (uint32_t)a.keys[i + mh - 1];
  if (a.recSeq[rb] != a.recSeq[ra]) return false;
  const int32_t wb = a.recWpos[rb];
  if (wb - a.recWpos[ra] >= a.fragLen) return false;
  start = max(0, wb - a.fragLen + 1);
  return true;
}

// flags: bit0 = head of a merged region, bit1 = tail of a merged region
__device__ __forceinline__ uint32_t l1_flags(const L1Args &a, unsigned long long i, int32_t &start, uint32_t &ra_out, int &f_out)
{
  const unsigned long long key = a.keys[i];
  const int f = (int)(key >> 32); const uint32_t ra = (uint32_t)key;
  ra_out = ra; f_out = f;
  const unsigned long long fragBeg = a.hitOff[a.segStart[f]], fragEnd = a.hitOff[a.segStart[f + 1]];
  const int mh = a.minHits[a.sCount[f]];
  if (!l1_qual(a, i, fragEnd, mh, ra, start)) return 0;
  uint32_t fl = 0;
  // merged with the left neighbour iff it qualifies, same contig, and its end (= its wpos) >= our start (:342-350)
  bool merged = false;
  if (i > fragBeg) {
    const uint32_t rp = (uint32_t)a.keys[i - 1]; int32_t sp;
    if (a.recSeq[rp] == a.recSeq[ra] && l1_qual(a, i - 1, fragEnd, mh, rp, sp) && a.recWpos[rp] >= start) merged = true;
  }
  if (!merged) fl |= 1;
  bool nextMerges = false;
  if (i + 1 < fragEnd) {
    const uint32_t rn = (uint32_t)a.keys[i + 1]; int32_t sn;
    if (a.recSeq[rn] == a.recSeq[ra] && l1_qual(a, i + 1, fragEnd, mh, rn, sn) && a.recWpos[ra] >= sn) nextMerges = true;
  }
  if (!nextMerges) fl |= 2;
  return fl;
}

__global__ void l1_flag_kernel(const L1Args a, uint32_t *head)
{
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > a.N) return;
  if (i == a.N) { head[i] = 0; return; }
  int32_t start; uint32_t ra; int f;
  head[i] = l1_flags(a, i, start, ra, f) & 1u;
}

__global__ void l1_write_kernel(const L1Args a, const uint32_t *head, const uint32_t *headScan,
                                int32_t *cFrag, int32_t *cSeq, int32_t *cStart, int32_t *cEnd)
{
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.N) return;
  int32_t start; uint32_t ra; int f;
  const uint32_t fl = l1_flags(a, i, start, ra, f);
  if (fl & 1) { const uint32_t c = headScan[i]; cFrag[c] = f; cSeq[c] = a.recSeq[ra]; cStart[c] = start; }
  if (fl & 2) { const uint32_t c = headScan[i] + head[i] - 1; cEnd[c] = a.recWpos[ra]; }
}

// ------------------------------------------------------------------ F: L2 (thread per candidate, state in global scratch)
struct L2Args {
  const int32_t *cFrag, *cSeq, *cStart, *cEnd; uint32_t C;
  const uint32_t *fragHash; const uint32_t *segStart; const int32_t *sCount;
  const uint32_t *recHash; const int32_t *recWpos; const uint32_t *recLink; const uint32_t *contigRecOff;
  int fragLen, cmw, smax;
  uint8_t *scratch; size_t stride;
  int32_t *cPos, *cBest;
  int onlyFlagged;
};

__device__ __forceinline__ uint32_t lb_wpos(const int32_t *wpos, uint32_t lo, uint32_t hi, int32_t v)
{
  while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (wpos[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}
__device__ __forceinline__ int lb_q(const uint32_t *Q, int s, uint32_t h)
{
  int lo = 0, hi = s;
  while (lo < hi) { int mid = (lo + hi) >> 1; if (Q[mid] < h) lo = mid + 1; else hi = mid; }
  return lo;
}

__global__ void __launch_bounds__(64)
l2_kernel(const L2Args a)
{
  const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x, nslots = gridDim.x * blockDim.x;
  uint16_t *gap = (uint16_t *)(a.scratch + (size_t)slot * a.stride);
  uint8_t *pres = (uint8_t *)(gap + a.smax + 2);
  for (uint32_t c = slot; c < a.C; c += nslots) {
    if (a.onlyFlagged && a.cBest[c] != -1) continue;           // the fast path already solved it
    const int f = a.cFrag[c];
    const int s = a.sCount[f];
    const uint32_t *Q = a.fragHash + a.segStart[f];
    const int seq = a.cSeq[c];
    const uint32_t lo = a.contigRecOff[seq], hi = a.contigRecOff[seq + 1];
    uint32_t b = lb_wpos(a.recWpos, lo, hi, a.cStart[c]);
    uint32_t e = lb_wpos(a.recWpos, lo, hi, a.recWpos[b] + a.cmw);
    const uint32_t last = lb_wpos(a.recWpos, lo, hi, a.cEnd[c] + a.fragLen);
    for (int i = 0; i <= s; i++) gap[i] = 0;
    for (int i = 0; i < s; i++) pres[i] = 0;
    int t = s, G = 0, P = 0;

    auto insert = [&](uint32_t r, uint32_t wb) {
      const uint32_t pd = a.recLink[r] >> 16;
      if (pd != 0xFFFFu && r - pd >= wb) return;              // an earlier twin is inside the window
      const uint32_t h = a.recHash[r];
      const int j = lb_q(Q, s, h);
      if (j < s && Q[j] == h) { pres[j] = 1; if (j < t) P++; }
      else { gap[j]++; if (j < t) G++; while (t + G > s) { t--; G -= gap[t]; P -= pres[t]; } }
    };
    auto remove = [&](uint32_t r, uint32_t we) {
      const uint32_t nd = a.recLink[r] & 0xFFFFu;
      if (nd != 0xFFFFu && r + nd < we) return;               // a later twin is still inside the window
      const uint32_t h = a.recHash[r];
      const int j = lb_q(Q, s, h);
      if (j < s && Q[j] == h) { pres[j] = 0; if (j < t) P--; }
      else { gap[j]--; if (j < t) G--; while (t < s && t + 1 + G + (int)gap[t] <= s) { G += gap[t]; P += pres[t]; t++; } }
    };

    for (uint32_t r = b; r < e; r++) insert(r, b);
    int sw = a.recWpos[b];
    int best = 0, first = 0, lastp = 0;
    while (e < last) {
      if (P > best) { best = P; first = lastp = a.recWpos[b]; }
      else if (P == best) lastp = a.recWpos[b];
      const int d1 = a.recWpos[b + 1] - sw, d2 = a.recWpos[e] - (sw + a.cmw - 1);
      const int adv = min(d1, d2);
      sw += adv;
      const uint32_t ob = b, oe = e;
      if (adv == d1) { remove(ob, oe); b++; }
      if (adv == d2) { insert(oe, b); e++; }
    }
    a.cPos[c] = (first + lastp) / 2;
    a.cBest[c] = best;
  }
}

// ------------------------------------------------------------------ F': L2 fast path = parallel pre-pass + lean sequential pass
// computeL2MappedRegions is a sequential sweep per candidate, but everything in it that does not depend on
// the sweep state can be computed for all (candidate, record) pairs in parallel:
//   l2_bounds_kernel  lane per candidate: b0 / e0 / last (the three lower_bounds of computeMap.hpp:424-436) and
//                     the exact number of window events
//   l2_events_kernel  CTA per fragment (its sketch Q + a two-level bucket directory in shared memory), lane per
//                     record: rank of the record's hash in Q, match bit, and -- from the per-record window links
//                     back / fwd / tie stored in the index (index.cu) -- the exact position of its "enters"
//                     and "leaves" events in the candidate's event stream, whether the event changes the set of
//                     DISTINCT window hashes (twin links), and whether a scoring point follows it.
//   l2_seq_kernel     lane per candidate (candidates ordered by event count so a warp's lanes finish together):
//                     streams the 16-bit codes (16-byte loads, one ahead) through the rank-space window state.
//
// Window state: ONE byte per rank j in shared memory = (number of distinct window hashes that are not in Q and
// have exactly j query hashes below them) | (q_j present in the window) << 7.  Byte j of a lane lives at
// j * 32 + lane of its warp's region, so the offset of a rank is the rank shifted: no address arithmetic, at the
// price of ~2-way bank conflicts (the four lanes that share a 32-bit word column).
//
// Event code (16 bits):  match [0] | insert [1] | score-after [2] | j [5:15]
// so that (code & 0xFFE0) is the byte offset of rank j and compares like j.  Events that do not change the set of
// distinct window hashes (a twin is inside the window), and events of hashes above every query hash, are coded as
// a "match" at rank s: they toggle the presence bit of the sentinel rank s, which no pivot position ever counts.
// A count reaching 64 (or s > 2047) hands the candidate to the exact global-memory kernel above.
static constexpr int L2_SMAX = 2047;
static constexpr int L2_SHM_BUDGET = 200 * 1024;      // dynamic shared memory granted to l2_events_kernel / l2_seq_kernel
static constexpr uint32_t EV_M = 1u, EV_D = 2u, EV_S = 4u, EV_JMASK = 0xFFE0u;
__host__ __device__ __forceinline__ uint32_t ev_rank(uint32_t j) { return j << 5; }

static constexpr int L2E_RING = 1024;             // events staged per warp of l2_events_kernel (2 KB: 6 CTAs of 8 warps per SM)
static constexpr int L2E_FLUSH_IT = 4;            // iterations of 32 records between two flushes = 16 steps of 16 events
static constexpr int L2E_BF_MAX = L2E_RING - 64 * L2E_FLUSH_IT - 96;   // 672: largest (max back + max fwd) of a staged candidate

struct L2PArgs {
  const int32_t *cFrag, *cSeq, *cStart, *cEnd; uint32_t C;
  const uint32_t *fragCandOff;
  const uint32_t *fragHash; const uint32_t *segStart; const int32_t *sCount;
  const uint4 *rec; const int32_t *recWposSoA; const uint32_t *contigRecOff;
  const uint2 *rec8; const uint32_t *recLink; const uint32_t *blkMax;      // compact L2 records + per-1024-record link bounds (index.cu)
  int fragLen, cmw, sLimit, shiftA, nBuckets;      // nBuckets: 1024 or 4096 (power of two), directory over h >> shiftA
  int stage;                                       // 0: every candidate takes the direct-store path of l2_events_kernel (switch "l2_stage")
  uint32_t *cB0, *cE0, *cLast, *cNEv, *cChunks;   // per candidate
  uint16_t *cMB;                                   // per candidate: bound on `back` of its records when its events can be staged, else 0xFFFF
  const uint32_t *cOff;                            // first 32-byte slot of the candidate's stream; step k is slot cOff + 32 * k
  const unsigned long long *grpOff;                // per warp group of 32 sorted candidates: first step row
  uint16_t *events;
  const uint32_t *perm; uint32_t warpBytes;
  int32_t *cPos, *cBest; unsigned long long *ctr_n2;
};

__global__ void frag_cand_off_kernel(const int32_t *cFrag, uint32_t C, int32_t F, uint32_t *fragCandOff)
{
  int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  uint32_t lo = 0, hi = C;                      // first candidate with cFrag >= f
  while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (cFrag[mid] < f) lo = mid + 1; else hi = mid; }
  fragCandOff[f] = lo;
}

__device__ __forceinline__ int32_t rec_wpos(const uint4 *rec, uint32_t i) { return (int32_t)(__ldg(&rec[i].y) & 0x7FFFFFFFu); }
__device__ __forceinline__ uint32_t lb_rec(const uint4 *rec, uint32_t lo, uint32_t hi, int32_t v)
{
  while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (rec_wpos(rec, mid) < v) lo = mid + 1; else hi = mid; }
  return lo;
}

__global__ void l2_bounds_kernel(const L2PArgs a)
{
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long n2 = 0;
  if (c < a.C) {
    const int seq = a.cSeq[c];
    const uint32_t lo = a.contigRecOff[seq], hi = a.contigRecOff[seq + 1];
    // the three lower_bounds probe the 4-byte position array (8 records per sector), not the 16-byte L2 records
    const uint32_t b0 = lb_wpos(a.recWposSoA, lo, hi, a.cStart[c]);
    const uint32_t e0 = lb_wpos(a.recWposSoA, b0, hi, __ldg(&a.recWposSoA[b0]) + a.cmw);
    const uint32_t last = lb_wpos(a.recWposSoA, b0, hi, a.cEnd[c] + a.fragLen);
    n2 = last - b0;
    const int s = a.sCount[a.cFrag[c]];
    uint32_t nEv = 0;
    if (e0 < last) {
      // removals scheduled = window start after the step in which record last-1 enters
      const uint32_t back = __ldg(&a.rec[last - 1].w) & 0xFFFFu;
      const uint32_t bEnd = (back > last - 1 - b0) ? b0 : last - 1 - back;
      nEv = (e0 - b0) + (last - e0) + (bEnd - b0);
    }
    a.cB0[c] = b0; a.cE0[c] = e0; a.cLast[c] = last;
    const bool fast = s >= 1 && s <= a.sLimit && nEv < (1u << 20);
    {
      // can l2_events_kernel stage this candidate's events in its shared-memory ring?  The ring has to span the event
      // positions still open between two flushes: bounded by the largest `back` plus the largest `fwd` of the records
      uint32_t mbk = 0, mfw = 0;
      if (fast && nEv) {
        const uint32_t blk1 = (last - 1) >> 10;
        for (uint32_t blk = b0 >> 10; blk <= blk1 && mbk != 0xFFFFu; blk++) { const uint32_t v = __ldg(&a.blkMax[blk]); mbk = max(mbk, v & 0xFFFFu); mfw = max(mfw, v >> 16); }
      }
      a.cMB[c] = (uint16_t)((a.stage && mbk + mfw <= (uint32_t)L2E_BF_MAX) ? mbk : 0xFFFFu);
    }
    a.cNEv[c] = fast ? nEv : 0u;
    a.cChunks[c] = fast ? (nEv + 15) >> 4 : 0u;      // 32-byte steps of 16 events
    a.cBest[c] = (fast || nEv == 0) ? 0 : -1;   // -1: exact slow kernel
    a.cPos[c] = 0;
  } else if (c == a.C) a.cChunks[c] = 0;
  for (int o = 16; o; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
  if ((threadIdx.x & 31) == 0 && n2) atomicAdd(a.ctr_n2, n2);
}

__global__ void l2_sortkey_kernel(const uint32_t *cNEv, uint32_t C, uint32_t *key, uint32_t *val)
{
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  key[c] = 0xFFFFFu - min(cNEv[c], 0xFFFFFu);   // ascending sort => longest streams first
  val[c] = c;
}

// steps of a warp group = steps of its longest member = the first in sorted order
__global__ void l2_group_steps_kernel(const uint32_t *cChunks, const uint32_t *perm, uint32_t C, uint32_t nGrp, uint32_t *grpSteps)
{
  const uint32_t G = blockIdx.x * blockDim.x + threadIdx.x;
  if (G > nGrp) return;
  grpSteps[G] = G < nGrp ? cChunks[perm[G * 32]] : 0u;
}
__global__ void l2_stream_base_kernel(const uint32_t *perm, const unsigned long long *grpOff, uint32_t C, uint32_t *cOff)
{
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= C) return;
  cOff[perm[g]] = (uint32_t)(grpOff[g >> 5] * 32ull + (g & 31u));
}
// event e of a stream that starts at 32-byte slot `base`: 16 events per slot, consecutive steps 32 slots apart
__device__ __forceinline__ size_t ev_index(uint32_t base, uint32_t e) { return ((size_t)base + (size_t)(e >> 4) * 32) * 16 + (e & 15u); }

static constexpr int L2E_BUCKETS = 4096;         // largest directory over h >> shiftA (clamped): ~1 query hash per bucket near 0;
                                                 // shards that see few candidates per fragment use 1024 (cheaper to build)

// Event schedule of one candidate in closed form.  With rb = r - b0, nInit = e0 - b0, nAll = last - b0 and the
// per-record window links of the index (back, fwd, tie; index.cu):
//   r ENTERS at position 2*rb - mb, mb = min(back, rb)  (= rb for the records of the first window, whose mb == rb... see below)
//            the window then starts at record r - mb; r adds a new distinct hash iff its previous twin is further than mb
//            back; a scoring point follows iff rb + 1 >= nInit (the first window is complete) and r is not the last record
//   r LEAVES at position 2*rb + fwd, if rb + fwd < nAll (no later than the step in which the last record enters);
//            the window then ends before record r + fwd; r removes a distinct hash iff its next twin is at least fwd
//            ahead; a scoring point follows unless another record enters in the same step (tie)
// (positions: the first window's records occupy 0 .. nInit-1 because for them back >= rb, i.e. mb = rb; afterwards
//  "enters" and "leaves" interleave by time, leaves first on ties -- the merge of computeMap.hpp:455-492.)
//
// CTA per fragment (NT threads: 256, 128 or 64 -- shards that see few candidates per fragment use small CTAs so that no
// warp idles), warp per candidate, lane per record.  Two ways to write the 16-bit codes:
//   staged  (cMB != 0xFFFF) the 8-byte compact records are read (hash | back:14 fwd:14 tie new gone); the codes go to a
//           per-warp ring in shared memory and leave it as whole 32-byte steps, one coalesced sector per lane: after the
//           records up to rb every position below 2*(rb+1) - max(back) is final, and between two flushes the open
//           positions span at most max(back) + max(fwd) + 64 * L2E_FLUSH_IT + 80 events (l2_bounds_kernel checks that
//           against the ring with the per-block bounds of the index)
//   direct  (low-complexity stretches with very long windows) 16-byte records, two 2-byte global stores per record
template <int NT>
__global__ void __launch_bounds__(NT)
l2_events_kernel(const L2PArgs a)
{
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ uint32_t s_wsum[NT / 32];
  constexpr int NW = NT / 32;
  const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t c0 = a.fragCandOff[f], c1 = a.fragCandOff[f + 1];
  if (c0 == c1) return;
  const int s = a.sCount[f];
  if (s < 1 || s > a.sLimit) return;
  uint16_t *ring = reinterpret_cast<uint16_t *>(smem) + wid * L2E_RING;                 // NW rings first (16-byte aligned)
  uint32_t *Q = smem + NW * (L2E_RING / 2);                                             // s hashes + 3 sentinels
  uint32_t *tab = Q + a.sLimit + 4;                                                     // L2E_BUCKETS + 1: bucket -> first rank
  uint2 *QP = reinterpret_cast<uint2 *>(smem + ((NW * (L2E_RING / 2) + a.sLimit + 4 + L2E_BUCKETS + 4 + 1) & ~1));   // {Q[j], Q[j+1]}: both probes in one load
  const int NB = a.nBuckets;
  {
    const uint32_t *Qg = a.fragHash + a.segStart[f];
    for (int i = tid; i < s + 3; i += NT) Q[i] = i < s ? Qg[i] : 0xFFFFFFFFu;
    for (int i = tid; i < s + 2; i += NT) QP[i] = make_uint2(i < s ? Qg[i] : 0xFFFFFFFFu, i + 1 < s ? Qg[i + 1] : 0xFFFFFFFFu);
    for (int i = tid; i <= NB; i += NT) tab[i] = 0;
    __syncthreads();
    for (int i = tid; i < s; i += NT) atomicAdd(&tab[min(Q[i] >> a.shiftA, (uint32_t)(NB - 1))], 1u);
    __syncthreads();
    // exclusive prefix over the bucket counts: every warp owns NB / NW consecutive buckets and walks them 32 at a time
    // (conflict-free reads, shuffle scan, running carry); pass 1 gives the warp totals, pass 2 writes the prefixes
    const int chunk = NB / NW, cbeg = wid * chunk;
    uint32_t wt = 0;
    for (int i = lane; i < chunk; i += 32) wt += tab[cbeg + i];
#pragma unroll
    for (int o = 16; o; o >>= 1) wt += __shfl_xor_sync(0xffffffffu, wt, o);
    if (lane == 0) s_wsum[wid] = wt;
    __syncthreads();
    uint32_t carry = 0;
    for (int i = 0; i < wid; i++) carry += s_wsum[i];
    for (int i = lane; i < chunk; i += 32) {
      const uint32_t cnt = tab[cbeg + i];
      uint32_t incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      tab[cbeg + i] = carry + incl - cnt;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (tid == NT - 1) tab[NB] = carry;
    __syncthreads();
  }
  const uint32_t nop = ev_rank((uint32_t)s) | EV_M | EV_D;
  const uint32_t bmax = (uint32_t)(NB - 1);
  // rank of h in Q: directory, then two probes (the sentinels and the sorted order make them unconditional)
  auto rank_of = [&](uint32_t h, bool &match) -> uint32_t {
    uint32_t j = tab[min(h >> a.shiftA, bmax)];
    const uint2 qq = QP[j];
    const uint32_t q0 = qq.x, q1 = qq.y;
    match = (q0 == h) || (q1 == h);
    j += (q0 < h) + (q1 < h);
    if (q1 < h) { while (Q[j] < h) j++; match = Q[j] == h; }              // crowded bucket (rare)
    return j;
  };
  for (uint32_t c = c0 + wid; c < c1; c += NW) {
    const uint32_t nEv = a.cNEv[c];
    if (nEv == 0) continue;
    const uint32_t b0 = a.cB0[c], nInit = a.cE0[c] - b0, nAll = a.cLast[c] - b0;
    const uint32_t sb = a.cOff[c];
    const uint32_t mbk = a.cMB[c];
    uint16_t *ev = a.events;
    if (mbk != 0xFFFFu) {
      // ---- staged: compact records in, whole 32-byte steps out
      const uint2 *rp = a.rec8 + b0;
      const uint32_t nIt = (nAll + 31) >> 5, nSteps = (nEv + 15) >> 4;
      uint32_t baseStep = 0;
      uint2 nxt = make_uint2(0u, 0u);
      if ((uint32_t)lane < nAll) nxt = __ldg(rp + lane);
      for (uint32_t it = 0; it < nIt; it++) {
        const uint32_t rb = it * 32 + lane;
        const uint2 rc = nxt;
        if (rb + 32 < nAll) nxt = __ldg(rp + rb + 32);
        if (rb < nAll) {
          bool match;
          const uint32_t j = rank_of(rc.x, match);
          const bool can = (int)j < s;                                        // rank s: above every query hash => no-op
          const uint32_t code = ev_rank(j) | (match ? EV_M : 0u);
          const uint32_t y = rc.y, back = y & 0x3FFFu, fwd = (y >> 14) & 0x3FFFu;
          const uint32_t mb = min(back, rb);
          // new distinct hash iff the previous twin is further than mb back: bit 29 says "further than back"; only a
          // record of the FIRST window (mb = rb < back) with a nearer twin needs the exact distance
          bool isNew = can && ((y >> 29) & 1u);
          if (can && !((y >> 29) & 1u) && rb < back) isNew = (__ldg(&a.recLink[b0 + rb]) >> 16) > rb;
          const bool sc = (rb + 1 >= nInit) && (rb + 1 != nAll);
          ring[(rb * 2 - mb) & (L2E_RING - 1)] = (uint16_t)((isNew ? (code | EV_D) : nop) | (sc ? EV_S : 0u));
          if (fwd != 0x3FFFu && rb + fwd < nAll) {
            const bool gone = can && ((y >> 30) & 1u);
            ring[(rb * 2 + fwd) & (L2E_RING - 1)] = (uint16_t)((gone ? code : nop) | (((y >> 28) & 1u) ? 0u : EV_S));
          }
        }
        const bool lastIt = it + 1 == nIt;
        if (lastIt || ((it + 1) % L2E_FLUSH_IT) == 0) {
          if (lastIt && (uint32_t)lane < ((16u - (nEv & 15u)) & 15u)) ring[(nEv + lane) & (L2E_RING - 1)] = (uint16_t)nop;   // pad the last step
          __syncwarp();
          // every position below 64 * (it + 1) - max(back) belongs to a record already processed and is never written again
          int fin = lastIt ? (int)nSteps : (((int)(64u * (it + 1)) - (int)mbk) >> 4);
          if (fin > (int)nSteps) fin = (int)nSteps;
          for (int k = (int)baseStep + lane; k < fin; k += 32) {
            const uint4 *src = reinterpret_cast<const uint4 *>(ring + ((k * 16) & (L2E_RING - 1)));
            uint4 *dst = reinterpret_cast<uint4 *>(ev + ((size_t)sb + (size_t)k * 32) * 16);
            const uint4 v0 = src[0], v1 = src[1];
            dst[0] = v0; dst[1] = v1;
          }
          if (fin > (int)baseStep) baseStep = (uint32_t)fin;
          __syncwarp();
        }
      }
      continue;
    }
    // ---- direct: 16-byte records, 2-byte stores
    if (lane < ((16u - (nEv & 15u)) & 15u)) ev[ev_index(sb, nEv + lane)] = (uint16_t)nop;    // pad the last 32-byte step
    const uint4 *rp = a.rec + b0;
    uint32_t rb = lane;
    uint4 nxt = make_uint4(0, 0, 0, 0);
    if (rb < nAll) nxt = __ldg(rp + rb);
    for (; rb < nAll; rb += 32) {
      const uint4 rc = nxt;
      if (rb + 32 < nAll) nxt = __ldg(rp + rb + 32);
      bool match;
      const uint32_t j = rank_of(rc.x, match);
      const bool can = (int)j < s;                                          // rank s: above every query hash => no-op
      const uint32_t code = ev_rank(j) | (match ? EV_M : 0u);
      const uint32_t pd = rc.z >> 16, nd = rc.z & 0xFFFFu, back = rc.w & 0xFFFFu, fwd = rc.w >> 16;
      const uint32_t rb2 = rb * 2;
      // r ENTERS
      const uint32_t mb = min(back, rb);
      const bool isNew = can && pd > mb;
      const bool sc = (rb + 1 >= nInit) && (rb + 1 != nAll);
      ev[ev_index(sb, rb2 - mb)] = (uint16_t)((isNew ? (code | EV_D) : nop) | (sc ? EV_S : 0u));
      // r LEAVES
      if (rb + fwd < nAll) {
        const bool gone = can && nd >= fwd;
        ev[ev_index(sb, rb2 + fwd)] = (uint16_t)((gone ? code : nop) | ((rc.y >> 31) ? 0u : EV_S));
      }
    }
  }
}

static constexpr int L2S_WARPS = 4;

__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr)); return v; }
__device__ __forceinline__ void sts_u8(uint32_t addr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }

__global__ void __launch_bounds__(L2S_WARPS * 32)
l2_seq_kernel(const L2PArgs a)
{
  extern __shared__ __align__(16) uint32_t smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t gid = blockIdx.x * (L2S_WARPS * 32) + threadIdx.x;
  const uint32_t wbase = (uint32_t)__cvta_generic_to_shared(smem) + (uint32_t)wid * a.warpBytes;
  for (uint32_t i = lane * 4u; i < a.warpBytes; i += 128u) sts_u32(wbase + i, 0u);
  __syncwarp();
  const uint32_t sb = wbase + (uint32_t)lane;

  uint32_t c = 0, nEv = 0; int s = 1;
  if (gid < a.C) { c = a.perm[gid]; nEv = a.cNEv[c]; s = a.sCount[a.cFrag[c]]; }
  // this lane's 32-byte slot of step k: row (grpOff[warp] + k) of 32 slots, column = lane (== cOff[c] + 32 * k)
  const unsigned long long row0 = (gid >> 5) < ((a.C + 31u) >> 5) ? a.grpOff[gid >> 5] : 0ull;
  const uint4 *strm = reinterpret_cast<const uint4 *>(a.events) + ((size_t)row0 * 32 + (size_t)lane) * 2;
  const uint32_t nSt = (nEv + 15) >> 4;                                  // 32-byte steps of this lane
  uint32_t maxSt = nSt;
  for (int o = 16; o; o >>= 1) maxSt = max(maxSt, __shfl_xor_sync(0xffffffffu, maxSt, o));
  const uint32_t nop = ev_rank((uint32_t)s) | EV_M | EV_D;
  const uint32_t nop2 = nop | (nop << 16);
  const uint4 nop4 = make_uint4(nop2, nop2, nop2, nop2);

  // pivot rank t kept as T5 = t << 5; Z = t + (#foreign hashes below the pivot) - s + 1  (invariant Z <= 1, t maximal);
  // P = query hashes present below the pivot
  uint32_t T5 = (uint32_t)s << 5;
  int Z = 1, P = 0, best = 0;
  uint32_t firstK = 0, lastK = 0, acc = 0;
  // each lane streams its own events: 32 bytes (one DRAM sector) per step, loaded two steps ahead
  uint4 n1a = nop4, n1b = nop4, n2a = nop4, n2b = nop4;
  if (nSt > 0) { n1a = __ldg(strm); n1b = __ldg(strm + 1); }
  if (nSt > 1) { n2a = __ldg(strm + 64); n2b = __ldg(strm + 65); }
  for (uint32_t stp = 0; stp < maxSt; stp++) {
    const uint4 ca = n1a, cb = n1b;
    n1a = n2a; n1b = n2b; n2a = nop4; n2b = nop4;
    if (stp + 2 < nSt) { n2a = __ldg(strm + 64 * (size_t)(stp + 2)); n2b = __ldg(strm + 64 * (size_t)(stp + 2) + 1); }
    const uint32_t wv[8] = {ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w};
    const uint32_t kb = stp * 16;
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const uint32_t ev = (q & 1) ? (wv[q >> 1] >> 16) : wv[q >> 1];      // the upper half of an even code is masked off below
      const uint32_t k = kb + q;
      // One event, written with explicit predication: the kernel is bound by the integer ALU pipe, and the
      // compiler's select-based if-conversion costs twice the operations.  Same statement in C:
      //   je = ev & 0xFFE0; g = state[je]; acc |= g; state[je] = g + (M ? 0x80 : dir)   (dir = insert ? +1 : -1)
      //   if (je < T5) { if (M) P += dir; else Z += dir; }
      //   down = Z > 1; if (down) T5 -= 32; gt = state[T5]; cnt = gt & 0x7F; pv = gt >> 7; up = Z + cnt <= 0;
      //   if (down) { Z -= cnt + 1; P -= pv; }  if (up) { Z += cnt + 1; P += pv; T5 += 32; }
      //   if (S && P >= best) { lastK = k; if (P > best) { best = P; firstK = k; } }
      asm volatile(
        "{\n\t"
        ".reg .pred pM, pD, pS, pBM, pBN, pDn, pUp, pGE, pGT;\n\t"
        ".reg .b32 je, aj, g, t1, dir, dl, nv, at, gt, cnt, pv, c1, zc;\n\t"
        "and.b32 je, %7, 0xFFE0;\n\t"
        "add.u32 aj, %8, je;\n\t"
        "ld.shared.u8 g, [aj];\n\t"
        "and.b32 t1, %7, 1;\n\t"  "setp.ne.u32 pM, t1, 0;\n\t"
        "and.b32 t1, %7, 2;\n\t"  "setp.ne.u32 pD, t1, 0;\n\t"
        "and.b32 t1, %7, 4;\n\t"  "setp.ne.u32 pS, t1, 0;\n\t"
        "selp.s32 dir, 1, -1, pD;\n\t"
        "selp.b32 dl, 0x80, dir, pM;\n\t"
        "or.b32 %6, %6, g;\n\t"
        "add.u32 nv, g, dl;\n\t"
        "st.shared.u8 [aj], nv;\n\t"
        "setp.lt.and.u32 pBM, je, %0, pM;\n\t"
        "setp.lt.and.u32 pBN, je, %0, !pM;\n\t"
        "@pBM add.s32 %2, %2, dir;\n\t"
        "@pBN add.s32 %1, %1, dir;\n\t"
        "setp.gt.s32 pDn, %1, 1;\n\t"
        "@pDn sub.u32 %0, %0, 32;\n\t"
        "add.u32 at, %8, %0;\n\t"
        "ld.shared.u8 gt, [at];\n\t"
        "and.b32 cnt, gt, 0x7F;\n\t"
        "shr.u32 pv, gt, 7;\n\t"
        "add.s32 zc, %1, cnt;\n\t"
        "setp.le.s32 pUp, zc, 0;\n\t"
        "add.s32 c1, cnt, 1;\n\t"
        "@pDn sub.s32 %1, %1, c1;\n\t"
        "@pDn sub.s32 %2, %2, pv;\n\t"
        "@pUp add.s32 %1, %1, c1;\n\t"
        "@pUp add.s32 %2, %2, pv;\n\t"
        "@pUp add.u32 %0, %0, 32;\n\t"
        "setp.ge.and.s32 pGE, %2, %3, pS;\n\t"
        "setp.gt.and.s32 pGT, %2, %3, pS;\n\t"
        "@pGE mov.u32 %5, %9;\n\t"
        "@pGT mov.u32 %4, %9;\n\t"
        "@pGT mov.s32 %3, %2;\n\t"
        "}"
        : "+r"(T5), "+r"(Z), "+r"(P), "+r"(best), "+r"(firstK), "+r"(lastK), "+r"(acc)
        : "r"(ev), "r"(sb), "r"(k)
        : "memory");
    }
  }
  if (gid < a.C && nEv) {
    if (acc & 0x40u) a.cBest[c] = -1;                        // a counter came near its 7-bit range: exact kernel
    else {
      // event index -> window start: b = b0 + #{records that left at or before that event}; the event position of
      // the removal of record r is monotone in r (same formula as in l2_events_kernel)
      const uint32_t b0 = a.cB0[c], e0 = a.cE0[c], last = a.cLast[c], nInit = e0 - b0;
      const uint32_t back = __ldg(&a.rec[last - 1].w) & 0xFFFFu;
      const uint32_t nRem = (back > last - 1 - b0) ? 0u : last - 1 - back - b0;
      auto removed_upto = [&](uint32_t K) -> uint32_t {
        uint32_t lo = 0, hi = nRem;                          // first r' with pos(b0 + r') > K
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1, r = b0 + mid;
          const uint32_t fwd = __ldg(&a.rec[r].w) >> 16;
          const uint32_t posr = nInit + mid + (r + fwd - e0);
          if (posr <= K) lo = mid + 1; else hi = mid;
        }
        return lo;
      };
      const int first = best > 0 ? rec_wpos(a.rec, b0 + removed_upto(firstK)) : 0;   // "first" stays 0 while best == 0 (as in the sweep above)
      const int lastp = rec_wpos(a.rec, b0 + removed_upto(lastK));
      a.cPos[c] = (first + lastp) / 2;
      a.cBest[c] = best;
    }
  }
}

// ------------------------------------------------------------------ G: report
struct RepArgs {
  const int32_t *cFrag, *cSeq, *cPos, *cBest; uint32_t C;
  const int32_t *sCount; const int32_t *fragSeqId;
  const uint32_t *rowOff; const float *ident, *upper; float pid; int fragLen;
};

__global__ void keep_flag_kernel(const RepArgs a, uint32_t *keep)
{
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > a.C) return;
  if (c == a.C) { keep[c] = 0; return; }
  const int s = a.sCount[a.cFrag[c]];
  keep[c] = a.upper[a.rowOff[s] + a.cBest[c]] >= a.pid ? 1u : 0u;      // computeMap.hpp:384
}

__global__ void rows_kernel(const RepArgs a, const uint32_t *keep, const uint32_t *keepScan, bani_mapping *rows,
                            int32_t *rFrag /* optional: chunk-global fragment index per row */)
{
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.C || !keep[c]) return;
  const int f = a.cFrag[c]; const int s = a.sCount[f]; const int best = a.cBest[c];
  bani_mapping r;
  r.queryLen = a.fragLen; r.refStartPos = a.cPos[c]; r.refEndPos = a.cPos[c] + a.fragLen - 1;
  r.queryStartPos = 0; r.queryEndPos = a.fragLen - 1;
  r.refSeqId = a.cSeq[c]; r.querySeqId = a.fragSeqId[f];
  r.nucIdentity = a.ident[a.rowOff[s] + best]; r.nucIdentityUpperBound = a.upper[a.rowOff[s] + best];
  r.sketchSize = s; r.conservedSketches = best;
  rows[keepScan[c]] = r;
  if (rFrag) rFrag[keepScan[c]] = f;
}

// ------------------------------------------------------------------ host orchestration
__global__ void scount_present_kernel(const int32_t *sCount, int32_t F, int smax, uint32_t *present)
{
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int s = sCount[f];
  if (s >= 1 && s <= smax) present[s] = 1u;
}

// The (s, shared) tables of stats.cpp on the device.  Sketch sizes up to LUT_DENSE get every row; beyond that (tiny
// windows: thousands of minimizers per fragment, a row costs O(s^2)) only the sizes that occur in the piece.
static constexpr int LUT_DENSE = 400;
void Ctx::upload_lut(int smaxNeeded, const int32_t *d_sCount, int32_t F)
{
  lut.k = prm.kmer_size; lut.pid = prm.perc_identity;
  bool changed = false;
  const int dense = std::min(std::max(smaxNeeded, 320), LUT_DENSE);
  if (lut.smax < dense) { lut.ensure(dense); changed = true; }
  if (smaxNeeded > LUT_DENSE) {
    if (!d_sCount) { lut.ensure(smaxNeeded); changed = true; }          // no size list: every row
    else {
      DevBuf<uint32_t> present((size_t)smaxNeeded + 1, stream);
      BANI_CUDA(cudaMemsetAsync(present.p, 0, 4 * ((size_t)smaxNeeded + 1), stream));
      scount_present_kernel<<<nblk(F), 256, 0, stream>>>(d_sCount, F, smaxNeeded, present.p);
      launches++;
      std::vector<uint32_t> h((size_t)smaxNeeded + 1);
      BANI_CUDA(cudaMemcpyAsync(h.data(), present.p, 4 * h.size(), cudaMemcpyDeviceToHost, stream));
      BANI_CUDA(cudaStreamSynchronize(stream));
      std::vector<int> svals;
      for (int sv = LUT_DENSE + 1; sv <= smaxNeeded; sv++) if (h[sv]) svals.push_back(sv);
      changed |= lut.ensure_rows(svals);
    }
  }
  if (!changed && lutUploaded > 0) return;
  d_minHits.alloc(lut.minHits.size(), stream); d_rowOff.alloc(lut.rowOff.size(), stream);
  d_ident.alloc(lut.ident.size(), stream); d_upper.alloc(lut.upper.size(), stream);
  BANI_CUDA(cudaMemcpyAsync(d_minHits.p, lut.minHits.data(), 4 * lut.minHits.size(), cudaMemcpyHostToDevice, stream));
  BANI_CUDA(cudaMemcpyAsync(d_rowOff.p, lut.rowOff.data(), 4 * lut.rowOff.size(), cudaMemcpyHostToDevice, stream));
  BANI_CUDA(cudaMemcpyAsync(d_ident.p, lut.ident.data(), 4 * lut.ident.size(), cudaMemcpyHostToDevice, stream));
  BANI_CUDA(cudaMemcpyAsync(d_upper.p, lut.upper.data(), 4 * lut.upper.size(), cudaMemcpyHostToDevice, stream));
  BANI_CUDA(cudaStreamSynchronize(stream));
  lutUploaded = 1;
}

// ------------------------------------------------------------------ query sketch (stages A + B as an object)
// Fragment descriptors of a piece, expanded on the device from one entry per fragment-bearing contig
// (Map::mapQuery, computeMap.hpp:131-189: fragment i of a contig = bases [i*fragLen, (i+1)*fragLen), id seqCounter + i).
struct FragSrc {
  const uint32_t *packed; const uint32_t *excPos; const uint8_t *excByte;
  int32_t nExc, firstFrag, seqBase, query;
  int32_t idxSeq;                               // contig ordinal inside the hint index (stage A'), else -1
};

__global__ void frag_table_kernel(const FragSrc *src, int32_t nSrc, int32_t F, int fragLen, SeqDesc *desc, int32_t *fragQuery, int32_t *fragSeqId)
{
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int lo = 0, hi = nSrc - 1;                   // last source with firstFrag <= f
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (src[mid].firstFrag <= f) lo = mid; else hi = mid - 1; }
  const FragSrc sr = src[lo];
  const int i = f - sr.firstFrag;
  SeqDesc d; d.packed = sr.packed; d.excPos = sr.excPos; d.excByte = sr.excByte; d.nExc = sr.nExc;
  d.startBase = i * fragLen; d.len = fragLen; d.seqId = sr.seqBase + i;                     // :173-175
  if (desc) desc[f] = d;
  fragQuery[f] = sr.query; fragSeqId[f] = sr.seqBase + i;
}

// ---- stage A': fragment sketches of a genome the index was built from, WITHOUT hashing it again.
// The windows of fragment [start, start + fragLen) are exactly the contig windows that lie inside it, and the index
// holds, per contig, one record for every change of the window minimizer (emitted at position e = wpos + w - 1).  So
//   Q(fragment) = { hash(r) : e_r in [A, B] }  +  hash(r*) if r* is still the minimizer at some VALID position of [A, B]
// with A = start + w - 1, B = start + fragLen - k (the fragment's first / last window end) and r* the last record
// emitted before A: it stays current until the next record is emitted, and the sketch only looks at valid positions
// (commonFunc.hpp:131), hence the validity bitmap written by the reference sketch launch.  Same multiset up to
// duplicates as sketching the fragment as a stand-alone sequence (computeMap.hpp:260); sort/unique follows as usual.
__device__ __forceinline__ bool any_valid_bit(const uint32_t *bits, unsigned long long b0, unsigned long long b1 /* inclusive */)
{
  unsigned long long wi = b0 >> 5; const unsigned long long we = b1 >> 5;
  uint32_t m = 0xFFFFFFFFu << (b0 & 31);
  for (; wi <= we; wi++, m = 0xFFFFFFFFu) {
    uint32_t v = __ldg(&bits[wi]) & m;
    if (wi == we) v &= 0xFFFFFFFFu >> (31 - (b1 & 31));
    if (v) return true;
  }
  return false;
}

__global__ void frag_ref_range_kernel(const FragSrc *src, int32_t nSrc, int32_t F, int fragLen, int k, int w,
                                      const int32_t *recWpos, const uint32_t *contigRecOff, const uint32_t *validBits,
                                      const unsigned long long *bitBase, uint32_t *rFirst, uint32_t *rCnt)
{
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  if (f == F) { rCnt[f] = 0; return; }
  int lo = 0, hi = nSrc - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (src[mid].firstFrag <= f) lo = mid; else hi = mid - 1; }
  const int seq = src[lo].idxSeq;
  const int start = (f - src[lo].firstFrag) * fragLen;
  const uint32_t rlo = contigRecOff[seq], rhi = contigRecOff[seq + 1];
  const int wA = start, wB = start + fragLen - k - w + 1;
  uint32_t first = rlo, cnt = 0;
  if (wB >= wA) {
    uint32_t a = rlo, b = rhi;
    while (a < b) { const uint32_t m = (a + b) >> 1; if (recWpos[m] < wA) a = m + 1; else b = m; }
    const uint32_t rA = a;
    b = rhi;
    while (a < b) { const uint32_t m = (a + b) >> 1; if (recWpos[m] <= wB) a = m + 1; else b = m; }
    const uint32_t rB = a;
    uint32_t inc = 0;
    if (rA > rlo) {
      const int A = start + w - 1, B = start + fragLen - k;
      const int hiPos = rA < rhi ? min(B, recWpos[rA] + w - 2) : B;       // r* is current up to the position before the next emission
      if (hiPos >= A && any_valid_bit(validBits, bitBase[seq] + (unsigned long long)A, bitBase[seq] + (unsigned long long)hiPos)) inc = 1;
    }
    first = rA - inc; cnt = rB - rA + inc;
  }
  rFirst[f] = first; rCnt[f] = cnt;
}

__global__ void frag_ref_gather_kernel(const uint32_t *recHash, const uint32_t *rFirst, const uint32_t *rawStart, int32_t F, uint32_t *raw)
{
  const int f = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (f >= F) return;
  const uint32_t a = rFirst[f], o = rawStart[f], n = rawStart[f + 1] - o;
  for (uint32_t i = lane; i < n; i += 32) raw[o + i] = recHash[a + i];
}

// sorted unique hashes of every fragment, back to back (the sort/unique kernel works in place on the raw segments)
__global__ void compact_sketch_kernel(const uint32_t *raw, const uint32_t *rawStart, const uint32_t *cOff, int32_t F, uint32_t *out)
{
  const int f = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (f >= F) return;
  const uint32_t a = rawStart[f], o = cOff[f], n = cOff[f + 1] - o;
  for (uint32_t i = lane; i < n; i += 32) out[o + i] = raw[a + i];
}

// fragments per piece: the working set of a piece (hit staging, L2 event streams: ~25 GB for 2^18 fragments of config 3)
// must fit an 80 GB device next to the index of a 1000-genome shard (~32 GB).  The switch frags_per_piece lowers it.
static constexpr uint64_t FRAG_MAX = 1u << 18;
static uint64_t frags_per_piece(const Ctx *ctx) { return std::min<uint64_t>(FRAG_MAX, (uint64_t)std::max(1ll, ctx->flags.fragsPerPiece)); }

// A query as the sketch stage sees it: a contig-length table plus either the packed bases (stage A) or the first contig
// ordinal inside the hint index (stage A': the genome is a member of the index, its bases are not needed).
struct QuerySrc { const Genome *G; int32_t nContigs; const int32_t *len; int32_t member; };

static QSketch *qsketch_build(Ctx *ctx, const std::vector<QuerySrc> &srcs, const int32_t *queryIds, const Index *hint);

QSketch *qsketch_create(Ctx *ctx, const Genome *const *queries, int32_t nq, const int32_t *queryIds, const Index *hint)
{
  const int k = ctx->prm.kmer_size, w = ctx->prm.window_size;
  const bool noReuse = !ctx->flags.sketchReuse;                                  // switch: always hash the queries
  if (hint && (noReuse || hint->device != ctx->device || hint->M == 0 || !hint->validBits.p || hint->k != k || hint->w != w)) hint = nullptr;
  std::vector<QuerySrc> srcs(nq);
  for (int i = 0; i < nq; i++) {
    const Genome *Q = queries[i];
    if (!Q) fail(BANI_ERR_ARG, "null genome handle");
    if (Q->device != ctx->device) fail(BANI_ERR_ARG, "genome lives on another device");
    int32_t mem = -1;                                                            // first contig ordinal inside the hint index
    if (hint) { auto it = hint->members.find(Q->uid); if (it != hint->members.end()) mem = it->second; }
    srcs[i] = QuerySrc{Q, Q->nContigs, Q->len.data(), mem};
  }
  return qsketch_build(ctx, srcs, queryIds, hint);
}

// Fragment sketches of genomes of the index itself, by genome ordinal: needs nothing but the index (an index loaded
// from disk serves as the query side of an all-vs-all run without any FASTA being read).  qsketch_from_index_file
// (index.cu) calls qsketch_from_records with a partial index of only the genomes asked for.
QSketch *qsketch_from_index(Ctx *ctx, const Index *ix, const int32_t *ordinals, int32_t nq, const int32_t *queryIds)
{
  if (ix->device != ctx->device) fail(BANI_ERR_ARG, "index lives on another device");
  if (ix->k != ctx->prm.kmer_size || ix->w != ctx->prm.window_size || ix->fragLen != ctx->prm.frag_len)
    fail(BANI_ERR_ARG, "index was built with other parameters (k %d w %d fragLen %d)", ix->k, ix->w, ix->fragLen);
  if (ix->M == 0 || !ix->validBits.p) fail(BANI_ERR_ARG, "the index holds no minimizers: query sketches cannot be derived from it");
  return qsketch_from_records(ctx, ix, ordinals, nq, queryIds);
}

QSketch *qsketch_from_records(Ctx *ctx, const Index *ix, const int32_t *ordinals, int32_t nq, const int32_t *queryIds)
{
  std::vector<QuerySrc> srcs(nq);
  for (int i = 0; i < nq; i++) {
    const int32_t g = ordinals[i];
    if (g < 0 || g >= ix->nGenomes) fail(BANI_ERR_ARG, "genome ordinal %d outside the index (%d genomes)", g, ix->nGenomes);
    const int32_t c0 = g ? ix->seqsByFile[g - 1] : 0, c1 = ix->seqsByFile[g];
    srcs[i] = QuerySrc{nullptr, c1 - c0, ix->contigLen.data() + c0, c0};
  }
  return qsketch_build(ctx, srcs, queryIds, ix);
}

static QSketch *qsketch_build(Ctx *ctx, const std::vector<QuerySrc> &srcs, const int32_t *queryIds, const Index *hint)
{
  cudaStream_t st = ctx->stream;
  const int32_t nq = (int32_t)srcs.size();
  const int k = ctx->prm.kmer_size, w = ctx->prm.window_size, fragLen = ctx->prm.frag_len;
  if (fragLen < 1 || fragLen > 60000) fail(BANI_ERR_LIMIT, "fragment length %d outside the supported range [1, 60000]", fragLen);
  auto qs = std::make_unique<QSketch>();
  qs->device = ctx->device; qs->k = k; qs->w = w; qs->fragLen = fragLen;
  qs->queryId.resize(nq); qs->totalFragments.assign(nq, 0);
  for (int i = 0; i < nq; i++) qs->queryId[i] = queryIds ? queryIds[i] : i;

  const uint64_t fragMax = frags_per_piece(ctx);
  int q0 = 0;
  while (q0 < nq) {
    // ---- fragment sources of this piece (Map::mapQuery, computeMap.hpp:131-189)
    std::vector<FragSrc> src;
    std::vector<int32_t> qFragOff;
    int64_t F64 = 0;
    bool pieceFromIndex = false;
    int q1 = q0;
    while (q1 < nq) {
      const QuerySrc &qsrc = srcs[q1];
      const Genome *Q = qsrc.G;
      uint64_t nf = 0;
      for (int c = 0; c < qsrc.nContigs; c++) { int L = qsrc.len[c]; if (!(L < w || L < k || L < fragLen)) nf += L / fragLen; }
      if (q1 > q0 && (uint64_t)F64 + nf > fragMax) break;
      const int32_t mem = hint ? qsrc.member : -1;
      if (mem < 0 && !Q) fail(BANI_ERR_INTERNAL, "query without bases and without an index to derive it from");
      if (mem < 0) Q->wait_ready(st);                                  // its bases are hashed: the upload must have landed
      if (q1 > q0 && (mem >= 0) != pieceFromIndex) break;           // a piece is either derived from the index or hashed
      pieceFromIndex = mem >= 0;
      qFragOff.push_back((int32_t)F64);
      int32_t seqCounter = 0;
      for (int c = 0; c < qsrc.nContigs; c++) {
        const int L = qsrc.len[c];
        if (L < w || L < k || L < fragLen) continue;                 // :138
        const int fc = L / fragLen;                                  // :152
        FragSrc sr;
        sr.packed = Q ? Q->packedBase() + Q->wordOff[c] : nullptr;
        sr.nExc = Q ? (int32_t)(Q->excOff[c + 1] - Q->excOff[c]) : 0;
        sr.excPos = sr.nExc ? Q->excPosBase() + Q->excOff[c] : nullptr;
        sr.excByte = sr.nExc ? Q->excByteBase() + Q->excOff[c] : nullptr;
        sr.firstFrag = (int32_t)F64; sr.seqBase = seqCounter; sr.query = q1 - q0; sr.idxSeq = mem >= 0 ? mem + c : -1;
        src.push_back(sr);
        F64 += fc; seqCounter += fc;
      }
      qs->totalFragments[q1] = (uint64_t)seqCounter;                 // :188-189
      q1++;
    }
    if (F64 > 0x7ffffff0ll) fail(BANI_ERR_LIMIT, "a query genome has more than 2^31 fragments");
    auto pc = std::make_unique<QPiece>();
    pc->q0 = q0; pc->nq = q1 - q0; pc->F = (int32_t)F64;
    pc->memberOf = (pieceFromIndex && hint) ? hint->uid : 0;
    qFragOff.push_back((int32_t)F64); pc->qFragOff = qFragOff;
    const int32_t F = pc->F;
    if (F > 0) {
      BANI_SCRATCH(FragSrc, d_src, src.size());
      BANI_CUDA(cudaMemcpyAsync(d_src.p, src.data(), sizeof(FragSrc) * src.size(), cudaMemcpyHostToDevice, st));
      pc->fragQuery.alloc(F, st); pc->fragSeqId.alloc(F, st);
      View<uint32_t> rawHash;
      BANI_SCRATCH(uint32_t, rawStart, (size_t)F + 1);
      uint64_t T = 0;
      if (pieceFromIndex) {
        // ---- A': the queries of this piece are genomes of the index: read their minimizers from it
        frag_table_kernel<<<nblk(F), 256, 0, st>>>(d_src.p, (int32_t)src.size(), F, fragLen, nullptr, pc->fragQuery.p, pc->fragSeqId.p);
        ctx->launches++;
        Stage sg(ctx, "q_from_index", 0);
        BANI_SCRATCH(uint32_t, rFirst, (size_t)F + 1);
        BANI_SCRATCH(uint32_t, rCnt, (size_t)F + 1);
        frag_ref_range_kernel<<<nblk((uint64_t)F + 1), 256, 0, st>>>(d_src.p, (int32_t)src.size(), F, fragLen, k, w, hint->wpos.p, hint->contigRecOff.p,
                                                                     hint->validBits.p, hint->contigBitBase.p, rFirst.p, rCnt.p);
        ctx->launches++;
        ctx->scan(rCnt.p, rawStart.p, (size_t)F + 1);
        uint32_t t32 = 0;
        BANI_CUDA(cudaMemcpyAsync(&t32, rawStart.p + F, 4, cudaMemcpyDeviceToHost, st));
        BANI_CUDA(cudaStreamSynchronize(st));
        T = t32;
        rawHash = ctx->view<uint32_t>(BANI_SLOT_ID, std::max<uint64_t>(T, 1));
        frag_ref_gather_kernel<<<nblk((uint64_t)F * 32), 256, 0, st>>>(hint->hash.p, rFirst.p, rawStart.p, F, rawHash.p);
        ctx->launches++;
        sg.bytes(8.0 * (double)T + 16.0 * F);
      } else {
      BANI_SCRATCH(SeqDesc, d_desc, F);
      frag_table_kernel<<<nblk(F), 256, 0, st>>>(d_src.p, (int32_t)src.size(), F, fragLen, d_desc.p, pc->fragQuery.p, pc->fragSeqId.p);
      ctx->launches++;

      // ---- A: fragment sketches
      uint64_t perFrag = std::max(1, fragLen - k + 1);
      uint64_t cap = std::min<uint64_t>((uint64_t)F * perFrag, (uint64_t)F * (uint64_t)(2.6 * fragLen / (w + 1) + 64));
      for (int attempt = 0; attempt < 2; attempt++) {
        if (cap > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "query chunk produces more than 2^32 minimizers");
        rawHash = ctx->view<uint32_t>(BANI_SLOT_ID, std::max<uint64_t>(cap, 1));
        Stage sg(ctx, "q_sketch", (double)F * fragLen / 4.0);
        T = sketch_sequences(ctx, d_desc.p, F, nullptr, fragLen, rawHash.p, nullptr, nullptr, cap, rawStart.p);
        sg.bytes((double)F * fragLen / 4.0 + 4.0 * (double)T);
        if (T <= cap) break;
        cap = T;
      }
      }

      // ---- B: sorted unique hashes per fragment, then packed back to back
      pc->sCount.alloc(F, st); pc->segStart.alloc((size_t)F + 1, st);
      DevBuf<int> d_flags(4, st);
      BANI_CUDA(cudaMemsetAsync(d_flags.p, 0, 16, st));
      unsigned long long T2 = 0;
      { Stage sg(ctx, "q_sort_unique", 8.0 * T);
        sort_unique_warp_kernel<<<nblk(F, SUW_WARPS), SUW_WARPS * 32, 0, st>>>(rawHash.p, rawStart.p, F, pc->sCount.p, d_flags.p, d_flags.p + 2); ctx->launches++;
        int nBig = 0;
        BANI_CUDA(cudaMemcpyAsync(&nBig, d_flags.p + 2, 4, cudaMemcpyDeviceToHost, st));
        BANI_CUDA(cudaStreamSynchronize(st));
        if (nBig > 0) { sort_unique_kernel<<<F, SU_THREADS, 0, st>>>(rawHash.p, rawStart.p, F, pc->sCount.p, d_flags.p, d_flags.p + 1, SUW_CAP); ctx->launches++; }
        BANI_SCRATCH(uint32_t, cnt1, (size_t)F + 1);
        BANI_CUDA(cudaMemcpyAsync(cnt1.p, pc->sCount.p, 4 * (size_t)F, cudaMemcpyDeviceToDevice, st));
        BANI_CUDA(cudaMemsetAsync(cnt1.p + F, 0, 4, st));
        ctx->scan(cnt1.p, pc->segStart.p, (size_t)F + 1);
        int hflags[2]; uint32_t t2 = 0;
        BANI_CUDA(cudaMemcpyAsync(hflags, d_flags.p, 8, cudaMemcpyDeviceToHost, st));
        BANI_CUDA(cudaMemcpyAsync(&t2, pc->segStart.p + F, 4, cudaMemcpyDeviceToHost, st));
        BANI_CUDA(cudaStreamSynchronize(st));
        if (hflags[1]) fail(BANI_ERR_LIMIT, "a query fragment has more than %d minimizers", SU_CAP);
        pc->smax = hflags[0]; T2 = t2;
        pc->fragHash.alloc(std::max<uint64_t>(T2, 1), st);
        compact_sketch_kernel<<<nblk((uint64_t)F * 32), 256, 0, st>>>(rawHash.p, rawStart.p, pc->segStart.p, F, pc->fragHash.p); ctx->launches++; }
      pc->T = T2;
      BANI_CUDA(cudaGetLastError());
      BANI_CUDA(cudaStreamSynchronize(st));          // src / scratch are reused by the next piece
    }
    qs->F += pc->F; qs->T += pc->T;
    qs->pieces.push_back(std::move(pc));
    q0 = q1;
  }
  return qs.release();
}

// ---- export / import: one flat DEVICE buffer, so that a query sketch can travel between GPUs (NCCL all-gather)
//   [u64 x 8: magic, nPieces, nQueries, k, w, fragLen, totalBytes, 0]
//   [nQueries x {i32 queryId, i32 firstFragmentInItsPiece, u64 totalFragments}]   [nPieces x u64 x 6: F, T, smax, q0, nq, 0]
//   per piece, each array padded to 16 bytes: segStart[F+1] sCount[F] fragQuery[F] fragSeqId[F] fragHash[T]
static inline uint64_t pad16(uint64_t b) { return (b + 15) & ~15ull; }
static constexpr uint64_t QS_MAGIC = 0x42414e4951534b31ull;

uint64_t qsketch_export_bytes(const QSketch *qs)
{
  uint64_t b = 64 + pad16(16ull * qs->queryId.size()) + 48ull * qs->pieces.size();
  for (const auto &pc : qs->pieces)
    if (pc->F > 0) b += pad16(4ull * (pc->F + 1)) + 3 * pad16(4ull * pc->F) + pad16(4ull * std::max<uint64_t>(pc->T, 1));
  return b;
}

void qsketch_export(Ctx *ctx, const QSketch *qs, void *devBuf, uint64_t cap)
{
  cudaStream_t st = ctx->stream;
  const uint64_t total = qsketch_export_bytes(qs);
  if (cap < total) fail(BANI_ERR_ARG, "export buffer too small: %llu < %llu bytes", (unsigned long long)cap, (unsigned long long)total);
  const uint64_t nQ = qs->queryId.size(), nP = qs->pieces.size();
  const uint64_t hdrBytes = 64 + pad16(16 * nQ) + 48 * nP;
  std::vector<uint8_t> h(hdrBytes, 0);
  uint64_t *h64 = (uint64_t *)h.data();
  h64[0] = QS_MAGIC; h64[1] = nP; h64[2] = nQ; h64[3] = (uint64_t)qs->k; h64[4] = (uint64_t)qs->w; h64[5] = (uint64_t)qs->fragLen; h64[6] = total;
  for (uint64_t i = 0; i < nQ; i++) {
    int32_t *e = (int32_t *)(h.data() + 64 + 16 * i);
    e[0] = qs->queryId[i]; *(uint64_t *)(e + 2) = qs->totalFragments[i];
  }
  for (const auto &pc : qs->pieces)
    for (int q = 0; q < pc->nq; q++) ((int32_t *)(h.data() + 64 + 16 * (uint64_t)(pc->q0 + q)))[1] = pc->qFragOff[q];
  uint64_t *ph = (uint64_t *)(h.data() + 64 + pad16(16 * nQ));
  for (uint64_t i = 0; i < nP; i++) {
    const QPiece &pc = *qs->pieces[i];
    ph[6 * i + 0] = (uint64_t)pc.F; ph[6 * i + 1] = pc.T; ph[6 * i + 2] = (uint64_t)pc.smax; ph[6 * i + 3] = (uint64_t)pc.q0; ph[6 * i + 4] = (uint64_t)pc.nq;
  }
  uint8_t *d = (uint8_t *)devBuf;
  BANI_CUDA(cudaMemcpyAsync(d, h.data(), hdrBytes, cudaMemcpyHostToDevice, st));
  uint64_t o = hdrBytes;
  auto put = [&](const void *p, uint64_t bytes) { BANI_CUDA(cudaMemcpyAsync(d + o, p, bytes, cudaMemcpyDeviceToDevice, st)); o += pad16(bytes); };
  for (const auto &pc : qs->pieces) {
    if (pc->F == 0) continue;
    put(pc->segStart.p, 4ull * (pc->F + 1)); put(pc->sCount.p, 4ull * pc->F); put(pc->fragQuery.p, 4ull * pc->F);
    put(pc->fragSeqId.p, 4ull * pc->F); put(pc->fragHash.p, 4ull * std::max<uint64_t>(pc->T, 1));
  }
  BANI_CUDA(cudaStreamSynchronize(st));              // h must outlive the copy
}

// A buffer that arrived from another rank is not trusted: sizes are checked against `bytes` before anything is
// allocated or copied, and the per-fragment tables are checked on the device before they are used as indices.
__global__ void qsketch_validate_kernel(const uint32_t *segStart, const int32_t *sCount, const int32_t *fragQuery, int32_t F, uint64_t T,
                                        int smax, int nq, int *bad)
{
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const uint32_t a = segStart[f], b = segStart[f + 1];
  const int s = sCount[f];
  bool ok = a <= b && (uint64_t)b <= T && s >= 0 && s <= smax && (uint32_t)s == b - a && fragQuery[f] >= 0 && fragQuery[f] < nq;
  if (f == 0 && a != 0) ok = false;
  if (f == F - 1 && (uint64_t)b != T) ok = false;
  if (f > 0 && fragQuery[f] < fragQuery[f - 1]) ok = false;
  if (!ok) atomicExch(bad, 1);
}

QSketch *qsketch_import(Ctx *ctx, const void *devBuf, uint64_t bytes)
{
  cudaStream_t st = ctx->stream;
  if (bytes < 64) fail(BANI_ERR_ARG, "not a query sketch buffer");
  uint64_t h0[8];
  BANI_CUDA(cudaMemcpyAsync(h0, devBuf, 64, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  if (h0[0] != QS_MAGIC || h0[6] > bytes) fail(BANI_ERR_ARG, "not a query sketch buffer (or truncated)");
  if ((int)h0[3] != ctx->prm.kmer_size || (int)h0[4] != ctx->prm.window_size || (int)h0[5] != ctx->prm.frag_len)
    fail(BANI_ERR_ARG, "query sketch was built with other parameters (k %d w %d fragLen %d)", (int)h0[3], (int)h0[4], (int)h0[5]);
  const uint64_t nP = h0[1], nQ = h0[2], total = h0[6];
  if (nP > (1ull << 24) || nQ > (1ull << 31)) fail(BANI_ERR_ARG, "corrupt query sketch buffer (header counts)");
  const uint64_t hdrBytes = 64 + pad16(16 * nQ) + 48 * nP;
  if (hdrBytes > total) fail(BANI_ERR_ARG, "query sketch buffer truncated (header)");
  std::vector<uint8_t> h(hdrBytes);
  BANI_CUDA(cudaMemcpyAsync(h.data(), devBuf, hdrBytes, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  auto qs = std::make_unique<QSketch>();
  qs->device = ctx->device; qs->k = (int)h0[3]; qs->w = (int)h0[4]; qs->fragLen = (int)h0[5];
  qs->queryId.resize(nQ); qs->totalFragments.resize(nQ);
  for (uint64_t i = 0; i < nQ; i++) {
    const int32_t *e = (const int32_t *)(h.data() + 64 + 16 * i);
    qs->queryId[i] = e[0]; qs->totalFragments[i] = *(const uint64_t *)(e + 2);
  }
  const uint64_t *ph = (const uint64_t *)(h.data() + 64 + pad16(16 * nQ));
  const uint8_t *d = (const uint8_t *)devBuf;
  uint64_t o = hdrBytes;
  DevBuf<int> d_bad(1, st);
  BANI_CUDA(cudaMemsetAsync(d_bad.p, 0, 4, st));
  uint64_t covered = 0;
  for (uint64_t i = 0; i < nP; i++) {
    auto pc = std::make_unique<QPiece>();
    const uint64_t F64 = ph[6 * i], T64 = ph[6 * i + 1], smax64 = ph[6 * i + 2], q064 = ph[6 * i + 3], nq64 = ph[6 * i + 4];
    if (F64 > FRAG_MAX || T64 > 0xfffffff0ull || smax64 > (uint64_t)SU_CAP || q064 != covered || nq64 > nQ - q064 || T64 > F64 * (uint64_t)SU_CAP)
      fail(BANI_ERR_ARG, "corrupt query sketch buffer (piece %llu)", (unsigned long long)i);
    pc->F = (int32_t)F64; pc->T = T64; pc->smax = (int)smax64; pc->q0 = (int)q064; pc->nq = (int)nq64;
    covered += nq64;
    for (int q = 0; q < pc->nq; q++) {
      const int32_t fo = ((const int32_t *)(h.data() + 64 + 16 * (uint64_t)(pc->q0 + q)))[1];
      if (fo < 0 || fo > pc->F || (q > 0 && fo < pc->qFragOff.back()) || (q == 0 && fo != 0)) fail(BANI_ERR_ARG, "corrupt query sketch buffer (fragment offsets)");
      pc->qFragOff.push_back(fo);
    }
    pc->qFragOff.push_back(pc->F);
    if (pc->F > 0) {
      if (pc->nq == 0) fail(BANI_ERR_ARG, "corrupt query sketch buffer (fragments without a query)");
      const uint64_t need = pad16(4ull * (pc->F + 1)) + 3 * pad16(4ull * pc->F) + pad16(4ull * std::max<uint64_t>(pc->T, 1));
      if (o + need > total) fail(BANI_ERR_ARG, "query sketch buffer truncated");
      auto get = [&](void *p, uint64_t b) { BANI_CUDA(cudaMemcpyAsync(p, d + o, b, cudaMemcpyDeviceToDevice, st)); o += pad16(b); };
      pc->segStart.alloc((size_t)pc->F + 1, st); pc->sCount.alloc(pc->F, st); pc->fragQuery.alloc(pc->F, st); pc->fragSeqId.alloc(pc->F, st);
      pc->fragHash.alloc(std::max<uint64_t>(pc->T, 1), st);
      get(pc->segStart.p, 4ull * (pc->F + 1)); get(pc->sCount.p, 4ull * pc->F); get(pc->fragQuery.p, 4ull * pc->F);
      get(pc->fragSeqId.p, 4ull * pc->F); get(pc->fragHash.p, 4ull * std::max<uint64_t>(pc->T, 1));
      qsketch_validate_kernel<<<nblk(pc->F), 256, 0, st>>>(pc->segStart.p, pc->sCount.p, pc->fragQuery.p, pc->F, pc->T, pc->smax, pc->nq, d_bad.p);
      ctx->launches++;
    }
    qs->F += pc->F; qs->T += pc->T;
    qs->pieces.push_back(std::move(pc));
  }
  if (covered != nQ) fail(BANI_ERR_ARG, "corrupt query sketch buffer (queries not covered by the pieces)");
  int bad = 0;
  BANI_CUDA(cudaMemcpyAsync(&bad, d_bad.p, 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  if (bad) fail(BANI_ERR_ARG, "corrupt query sketch buffer (fragment tables)");
  return qs.release();
}

// ---- a sub-range of whole queries of a piece as a piece of its own (offsets rebased); used when a piece gathers
//      more index hits than one pass should hold (many near-identical references)
__global__ void rebase_u32_kernel(const uint32_t *in, uint32_t delta, uint64_t n, uint32_t *out)
{
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i] - delta;
}

// ---- several sketches as one: the pieces are packed back to back into pieces of up to FRAG_MAX fragments, so that
//      the sketches a rank received from its peers are mapped in a few large passes instead of one small pass per peer
QSketch *qsketch_merge(Ctx *ctx, const QSketch *const *sketches, int32_t n)
{
  cudaStream_t st = ctx->stream;
  auto out = std::make_unique<QSketch>();
  out->device = ctx->device; out->k = ctx->prm.kmer_size; out->w = ctx->prm.window_size; out->fragLen = ctx->prm.frag_len;
  struct Src { const QPiece *pc; int qBase; };
  std::vector<Src> srcs;
  for (int i = 0; i < n; i++) {
    const QSketch *qs = sketches[i];
    if (!qs) fail(BANI_ERR_ARG, "null query sketch");
    if (qs->device != ctx->device) fail(BANI_ERR_ARG, "query sketch lives on another device");
    if (qs->k != out->k || qs->w != out->w || qs->fragLen != out->fragLen) fail(BANI_ERR_ARG, "query sketch was built with other parameters");
    const int qBase = (int)out->queryId.size();
    out->queryId.insert(out->queryId.end(), qs->queryId.begin(), qs->queryId.end());
    out->totalFragments.insert(out->totalFragments.end(), qs->totalFragments.begin(), qs->totalFragments.end());
    for (const auto &pc : qs->pieces) srcs.push_back(Src{pc.get(), qBase + pc->q0});
  }
  const uint64_t fragMax = frags_per_piece(ctx);
  size_t i = 0;
  while (i < srcs.size()) {
    size_t j = i; uint64_t F = 0, T = 0;
    while (j < srcs.size() && (j == i || (F + (uint64_t)srcs[j].pc->F <= fragMax && T + srcs[j].pc->T < 0xfffffff0ull &&
                                          srcs[j].qBase == srcs[j - 1].qBase + srcs[j - 1].pc->nq))) { F += (uint64_t)srcs[j].pc->F; T += srcs[j].pc->T; j++; }
    auto pc = std::make_unique<QPiece>();
    pc->q0 = srcs[i].qBase; pc->F = (int32_t)F; pc->T = T;
    if (F > 0) {
      pc->segStart.alloc((size_t)F + 1, st); pc->sCount.alloc(F, st); pc->fragQuery.alloc(F, st); pc->fragSeqId.alloc(F, st);
      pc->fragHash.alloc(std::max<uint64_t>(T, 1), st);
    }
    uint64_t fo = 0, to = 0; int qo = 0;
    for (size_t s = i; s < j; s++) {
      const QPiece &sp = *srcs[s].pc;
      for (int q = 0; q < sp.nq; q++) pc->qFragOff.push_back(sp.qFragOff[q] + (int32_t)fo);
      pc->smax = std::max(pc->smax, sp.smax);
      if (sp.F > 0) {
        const size_t sf = (size_t)sp.F;
        rebase_u32_kernel<<<nblk(sf + 1), 256, 0, st>>>(sp.segStart.p, (uint32_t)(0u - (uint32_t)to), sf + 1, pc->segStart.p + fo);
        rebase_u32_kernel<<<nblk(sf), 256, 0, st>>>((const uint32_t *)sp.fragQuery.p, (uint32_t)(0u - (uint32_t)qo), sf, (uint32_t *)pc->fragQuery.p + fo);
        ctx->launches += 2;
        BANI_CUDA(cudaMemcpyAsync(pc->sCount.p + fo, sp.sCount.p, 4 * sf, cudaMemcpyDeviceToDevice, st));
        BANI_CUDA(cudaMemcpyAsync(pc->fragSeqId.p + fo, sp.fragSeqId.p, 4 * sf, cudaMemcpyDeviceToDevice, st));
        if (sp.T) BANI_CUDA(cudaMemcpyAsync(pc->fragHash.p + to, sp.fragHash.p, 4 * sp.T, cudaMemcpyDeviceToDevice, st));
      }
      fo += (uint64_t)sp.F; to += sp.T; qo += sp.nq;
    }
    pc->nq = qo;
    pc->qFragOff.push_back((int32_t)F);
    out->F += F; out->T += T;
    out->pieces.push_back(std::move(pc));
    i = j;
  }
  BANI_CUDA(cudaGetLastError());
  BANI_CUDA(cudaStreamSynchronize(st));          // the sources may be destroyed when this returns
  return out.release();
}

static std::unique_ptr<QPiece> slice_piece(Ctx *ctx, const QPiece &pc, int qa, int qb)
{
  cudaStream_t st = ctx->stream;
  auto sl = std::make_unique<QPiece>();
  const int32_t fA = pc.qFragOff[qa], fB = pc.qFragOff[qb];
  sl->q0 = pc.q0 + qa; sl->nq = qb - qa; sl->F = fB - fA; sl->smax = pc.smax; sl->memberOf = pc.memberOf;
  for (int q = qa; q <= qb; q++) sl->qFragOff.push_back(pc.qFragOff[q] - fA);
  if (sl->F > 0) {
    uint32_t tA = 0, tB = 0;
    BANI_CUDA(cudaMemcpyAsync(&tA, pc.segStart.p + fA, 4, cudaMemcpyDeviceToHost, st));
    BANI_CUDA(cudaMemcpyAsync(&tB, pc.segStart.p + fB, 4, cudaMemcpyDeviceToHost, st));
    BANI_CUDA(cudaStreamSynchronize(st));
    sl->T = tB - tA;
    const size_t F = (size_t)sl->F;
    sl->segStart.alloc(F + 1, st); sl->sCount.alloc(F, st); sl->fragQuery.alloc(F, st); sl->fragSeqId.alloc(F, st);
    sl->fragHash.alloc(std::max<uint64_t>(sl->T, 1), st);
    rebase_u32_kernel<<<nblk(F + 1), 256, 0, st>>>(pc.segStart.p + fA, tA, F + 1, sl->segStart.p);
    rebase_u32_kernel<<<nblk(F), 256, 0, st>>>((const uint32_t *)pc.fragQuery.p + fA, (uint32_t)qa, F, (uint32_t *)sl->fragQuery.p);
    ctx->launches += 2;
    BANI_CUDA(cudaMemcpyAsync(sl->sCount.p, pc.sCount.p + fA, 4 * F, cudaMemcpyDeviceToDevice, st));
    BANI_CUDA(cudaMemcpyAsync(sl->fragSeqId.p, pc.fragSeqId.p + fA, 4 * F, cudaMemcpyDeviceToDevice, st));
    if (sl->T) BANI_CUDA(cudaMemcpyAsync(sl->fragHash.p, pc.fragHash.p + tA, 4 * sl->T, cudaMemcpyDeviceToDevice, st));
  }
  return sl;
}

// path counter (flags.countPaths only): candidates the exact kernel l2_kernel will solve (cBest == -1)
static uint64_t count_exact(Ctx *ctx, const int32_t *d_cBest, uint32_t C)
{
  std::vector<int32_t> h(C);
  BANI_CUDA(cudaMemcpyAsync(h.data(), d_cBest, 4 * (size_t)C, cudaMemcpyDeviceToHost, ctx->stream));
  BANI_CUDA(cudaStreamSynchronize(ctx->stream));
  return (uint64_t)std::count(h.begin(), h.end(), -1);
}

// ------------------------------------------------------------------ host orchestration of stages C..H
void map_queries(Ctx *ctx, const Index *ix, const Genome *const *queries, int32_t nq,
                 bool wantRows, bool wantCgi, MapOutput &out)
{
  std::unique_ptr<QSketch> qs(qsketch_create(ctx, queries, nq, nullptr, ix));
  ctx->mark("map: query sketches built");
  const QSketch *one = qs.get();
  qsketch_map(ctx, ix, &one, 1, wantRows, wantCgi, out);
  ctx->mark("map: qsketch_map returned");
  out.totalQueryFragments = qs->totalFragments;
  qs.reset();
  ctx->mark("map: query sketches freed");
}

// ------------------------------------------------------------------ stages C..G of one piece
// What a stage hands to the next.  The Views are scratch slots of the function that fills them: each of those
// functions runs once per piece, so the arrays stay valid until the piece is done.
struct Hits {                                   // C: index hits of the T query hashes (T + 1 entries, the last one 0)
  View<uint32_t> lo, cnt; View<unsigned long long> off;     // first posIdx entry, count, exclusive scan of the counts
  unsigned long long N = 0;
  DevBuf<unsigned long long> walkCtr;           // probes that walked the sorted keys (flags.countPaths)
};
struct Cands { View<int32_t> frag, seq, start, end; uint32_t C = 0; };     // D+E: compact L1 candidate regions
struct Scores {                                 // F: best window of every candidate, window evaluations (n2, on the device)
  View<int32_t> pos, best; View<unsigned long long> n2;
  size_t idEv = (size_t)-1; double evBytes = 0; // timer of l2_events: its bytes are set once n2 is known
};
struct Rows { View<bani_mapping> rows; DevBuf<int32_t> frag; uint32_t R = 0; };   // G: rows past the cutoff, fragment of each

// C: lookup.  N and the walk counters come back behind one synchronisation.
static void lookup(Ctx *ctx, const Index *ix, const QPiece &pc, uint64_t *pp, Hits &h)
{
  cudaStream_t st = ctx->stream;
  const uint64_t T = pc.T;
  BANI_SCRATCH(uint32_t, hitLo, T + 1);
  BANI_SCRATCH(uint32_t, hitCnt, T + 1);
  BANI_SCRATCH(unsigned long long, hitOff, T + 1);
  h.lo = hitLo; h.cnt = hitCnt; h.off = hitOff;
  if (ctx->flags.countPaths) { h.walkCtr.alloc(2, st); BANI_CUDA(cudaMemsetAsync(h.walkCtr.p, 0, 16, st)); }
  { Stage sg(ctx, "lookup", 12.0 * T);
    // the membership filter pays when most probes miss: not for queries that are genomes of this very index
    const bool useFilt = ix->filt.p && pc.memberOf != ix->uid;
    lookup_kernel<<<nblk(T + 1), 256, 0, st>>>(pc.fragHash.p, (uint32_t)T, ix->tab.p, (1u << ix->tabBits) - 1u, ix->ukeys.p, ix->uoff.p,
                                               ix->dir.p, ix->dirBits, useFilt ? ix->filt.p : nullptr,
                                               useFilt ? (uint32_t)((1ull << ix->filtBits) - 1ull) : 0u, hitLo.p, hitCnt.p, h.walkCtr.p);
    ctx->launches++;
    ctx->scan(hitCnt.p, hitOff.p, T + 1); }
  BANI_CUDA(cudaMemcpyAsync(&h.N, hitOff.p + T, 8, cudaMemcpyDeviceToHost, st));
  if (ctx->flags.countPaths) BANI_CUDA(cudaMemcpyAsync(pp + P_LOOKUP_WALK_SATURATED, h.walkCtr.p, 16, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  ctx->mark("piece: lookup done");
}

// D+E for the fragments with more hits than one CTA takes: (fragment, record) keys, one radix sort, flags + scan + write.
// The regions go to the staging area of l1_candidates, at the fragment's hit offset.
static void l1_device_wide(Ctx *ctx, const Index *ix, const QPiece &pc, const Hits &h, const uint32_t *fragClass,
                           int32_t *stSeq, int32_t *stStart, int32_t *stEnd, uint32_t *candCount)
{
  cudaStream_t st = ctx->stream;
  const int32_t F = pc.F; const uint64_t T = pc.T;
  BANI_SCRATCH(uint32_t, bigCnt, T + 1);
  BANI_SCRATCH(unsigned long long, bigOff, T + 1);
  mask_hits_kernel<<<nblk(T + 1), 256, 0, st>>>(pc.segStart.p, F, (uint32_t)T, h.cnt.p, fragClass, bigCnt.p); ctx->launches++;
  ctx->scan(bigCnt.p, bigOff.p, T + 1);
  unsigned long long NB = 0;
  BANI_CUDA(cudaMemcpyAsync(&NB, bigOff.p + T, 8, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  BANI_SCRATCH(unsigned long long, keysA, NB);
  BANI_SCRATCH(unsigned long long, keysB, NB);
  { Stage sg(ctx, "hit_gather", 12.0 * NB);
    gather_kernel<<<nblk(T), 256, 0, st>>>(pc.segStart.p, F, (uint32_t)T, h.lo.p, bigCnt.p, bigOff.p, ix->posIdx.p, keysA.p); ctx->launches++; }
  int fbits = 1; while ((1ll << fbits) < F) fbits++;
  { Stage sg(ctx, "hit_sort", 16.0 * NB);
    ctx->sort_keys(keysA.p, keysB.p, NB, 32 + fbits); }
  L1Args la; la.keys = keysB.p; la.N = NB; la.segStart = pc.segStart.p; la.hitOff = bigOff.p; la.sCount = pc.sCount.p;
  la.minHits = ctx->d_minHits.p; la.recSeq = ix->seqId.p; la.recWpos = ix->wpos.p; la.fragLen = ctx->prm.frag_len;
  BANI_SCRATCH(uint32_t, head, NB + 1);
  BANI_SCRATCH(uint32_t, headScan, NB + 1);
  { Stage sg(ctx, "l1_flags", 8.0 * NB);
    l1_flag_kernel<<<nblk(NB + 1), 256, 0, st>>>(la, head.p);
    ctx->launches++;
    ctx->scan(head.p, headScan.p, NB + 1); }
  uint32_t CB = 0;
  BANI_CUDA(cudaMemcpyAsync(&CB, headScan.p + NB, 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  if (CB == 0) return;
  BANI_SCRATCH(int32_t, bFrag, CB);
  BANI_SCRATCH(int32_t, bSeq, CB);
  BANI_SCRATCH(int32_t, bStart, CB);
  BANI_SCRATCH(int32_t, bEnd, CB);
  Stage sg(ctx, "l1_write", 8.0 * NB);
  l1_write_kernel<<<nblk(NB), 256, 0, st>>>(la, head.p, headScan.p, bFrag.p, bSeq.p, bStart.p, bEnd.p); ctx->launches++;
  cand_stage(ctx, bFrag.p, bSeq.p, bStart.p, bEnd.p, CB, pc.segStart.p, h.off.p, stSeq, stStart, stEnd, candCount);
}

// D+E: hits -> L1 candidate regions.  Fragments with at most FRAG_L1_MAX hits are handled by one CTA each (hits.cu), the
// others by l1_device_wide.  Both write their regions to a staging area addressed by the fragment's hit offset; a scan +
// copy makes them dense.
static void l1_candidates(Ctx *ctx, const Index *ix, const QPiece &pc, const Hits &h, uint64_t *pp, Cands &cd)
{
  cudaStream_t st = ctx->stream;
  const int32_t F = pc.F; const unsigned long long N = h.N;
  BANI_SCRATCH(uint32_t, candCount, (size_t)F + 1);
  BANI_SCRATCH(uint32_t, candOff, (size_t)F + 1);
  BANI_SCRATCH(uint32_t, fragClass, F);
  BANI_SCRATCH(uint32_t, classList, (size_t)FRAG_NCLASS * F);
  BANI_SCRATCH(uint32_t, classCount, FRAG_NCLASS + 2);
  BANI_SCRATCH(int32_t, stSeq, N);
  BANI_SCRATCH(int32_t, stStart, N);
  BANI_SCRATCH(int32_t, stEnd, N);
  const long long maxFast = std::max(0ll, std::min(ctx->flags.fragL1Max, (long long)FRAG_L1_MAX));
  uint32_t hClass[FRAG_NCLASS + 2];
  { Stage sg(ctx, "frag_l1", 12.0 * N);                // 4 B list entry + 8 B (seqId, wpos) per hit
    frag_classify(ctx, pc.segStart.p, h.off.p, F, candCount.p, fragClass.p, classCount.p, classList.p, (unsigned long long)maxFast);
    BANI_CUDA(cudaMemcpyAsync(hClass, classCount.p, sizeof hClass, cudaMemcpyDeviceToHost, st));
    BANI_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i <= FRAG_NCLASS; i++) pp[P_L1_CLASS0 + i] += hClass[i];
    FragL1Args fa; fa.segStart = pc.segStart.p; fa.sCount = pc.sCount.p; fa.F = F; fa.hitLo = h.lo.p; fa.hitCnt = h.cnt.p; fa.hitOff = h.off.p;
    fa.posIdx = ix->posIdx.p; fa.recPos = ix->pos8.p; fa.minHits = ctx->d_minHits.p; fa.fragLen = ctx->prm.frag_len;
    fa.keyBits = 1; while (fa.keyBits < 32 && (1ull << fa.keyBits) < ix->M) fa.keyBits++;
    fa.stSeq = stSeq.p; fa.stStart = stStart.p; fa.stEnd = stEnd.p; fa.candCount = candCount.p;
    frag_l1_fast(ctx, fa, classList.p, hClass); }
  if (hClass[FRAG_NCLASS] > 0) l1_device_wide(ctx, ix, pc, h, fragClass.p, stSeq.p, stStart.p, stEnd.p, candCount.p);
  BANI_CUDA(cudaMemsetAsync(candCount.p + F, 0, 4, st));
  ctx->scan(candCount.p, candOff.p, (size_t)F + 1);
  BANI_CUDA(cudaMemcpyAsync(&cd.C, candOff.p + F, 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  if (cd.C == 0) return;
  BANI_SCRATCH(int32_t, cFrag, cd.C);
  BANI_SCRATCH(int32_t, cSeq, cd.C);
  BANI_SCRATCH(int32_t, cStart, cd.C);
  BANI_SCRATCH(int32_t, cEnd, cd.C);
  cd.frag = cFrag; cd.seq = cSeq; cd.start = cStart; cd.end = cEnd;
  cand_compact(ctx, pc.segStart.p, h.off.p, F, candCount.p, candOff.p, stSeq.p, stStart.p, stEnd.p, cFrag.p, cSeq.p, cStart.p, cEnd.p);
}

// Fast path of F: candidates by descending event count (rank g -> warp g / 32, lane g % 32 of l2_seq_kernel), their
// window-event streams, the sequential sweep.  Stops the l2_bounds timer before the events.  Returns
// P_PIECE_SPLIT_EVENTS, with nothing launched past the scan of the group steps, when the event streams would not fit.
static PathId l2_fast(Ctx *ctx, const QPiece &pc, L2PArgs &lp, uint32_t *cOff, Stage &sgb, uint64_t *pp, Scores &sc)
{
  cudaStream_t st = ctx->stream;
  const int32_t F = pc.F; const uint32_t C = lp.C;
  BANI_SCRATCH(uint32_t, skey, C);
  BANI_SCRATCH(uint32_t, skey2, C);
  BANI_SCRATCH(uint32_t, sval, C);
  BANI_SCRATCH(uint32_t, perm, C);
  l2_sortkey_kernel<<<nblk(C), 256, 0, st>>>(lp.cNEv, C, skey.p, sval.p); ctx->launches++;
  ctx->sort_pairs(skey.p, skey2.p, sval.p, perm.p, C, 20);
  lp.perm = perm.p;
  // event streams, interleaved per warp: step k of lane l of warp G is the 32-byte slot (grpOff[G] + k) * 32 + l,
  // so a warp reads 1 KB contiguous per step while every 32-byte sector still belongs to one candidate
  const uint32_t nGrp = (C + 31) / 32;
  BANI_SCRATCH(uint32_t, grpSteps, (size_t)nGrp + 1);
  BANI_SCRATCH(unsigned long long, grpOff, (size_t)nGrp + 1);
  l2_group_steps_kernel<<<nblk((uint64_t)nGrp + 1), 256, 0, st>>>(lp.cChunks, perm.p, C, nGrp, grpSteps.p); ctx->launches++;
  ctx->scan(grpSteps.p, grpOff.p, (size_t)nGrp + 1);
  unsigned long long totalGrpSteps = 0;
  BANI_CUDA(cudaMemcpyAsync(&totalGrpSteps, grpOff.p + nGrp, 8, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  const unsigned long long totalSteps = totalGrpSteps * 32;     // 32-byte slots
  // the event streams of this piece would take more than a quarter of the device (small windows make many events per
  // hit): map its halves instead, so that they fit beside the index
  const double evLimit = ctx->flags.eventBytesPerPiece > 0 ? (double)ctx->flags.eventBytesPerPiece : 0.25 * (double)ctx->memTotal;
  if ((double)totalSteps * 32.0 > evLimit && pc.nq > 1) return P_PIECE_SPLIT_EVENTS;
  if (totalSteps > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "query chunk schedules more than 2^36 window events");
  BANI_SCRATCH(uint16_t, events, (size_t)totalSteps * 16 + 64);
  lp.events = events.p; lp.grpOff = grpOff.p;
  l2_stream_base_kernel<<<nblk(C), 256, 0, st>>>(perm.p, grpOff.p, C, cOff); ctx->launches++;
  // CTA size of the events kernel by candidates per fragment (warp per candidate: no idle warps in small shards)
  const int evNT = ((uint64_t)C >= 6ull * (uint64_t)F) ? 256 : ((uint64_t)C >= 3ull * (uint64_t)F) ? 128 : 64;
  if (ctx->flags.countPaths) {
    // candidates with window events, by the variant of l2_events_kernel that writes them
    std::vector<uint32_t> nEv(C); std::vector<uint16_t> mb(C);
    BANI_CUDA(cudaMemcpyAsync(nEv.data(), lp.cNEv, 4 * (size_t)C, cudaMemcpyDeviceToHost, st));
    BANI_CUDA(cudaMemcpyAsync(mb.data(), lp.cMB, 2 * (size_t)C, cudaMemcpyDeviceToHost, st));
    BANI_CUDA(cudaStreamSynchronize(st));
    uint64_t withEv = 0, staged = 0;
    for (uint32_t c = 0; c < C; c++) if (nEv[c]) { withEv++; staged += mb[c] != 0xFFFFu; }
    pp[evNT == 256 ? P_L2_EVENTS_NT256 : evNT == 128 ? P_L2_EVENTS_NT128 : P_L2_EVENTS_NT64] += withEv;
    pp[lp.nBuckets == L2E_BUCKETS ? P_L2_DIR4096 : P_L2_DIR1024] += withEv;
    pp[P_L2_STAGED] += staged; pp[P_L2_DIRECT] += withEv - staged;
  }
  const size_t shmE = 4 * ((size_t)(evNT / 32) * (L2E_RING / 2) + (size_t)lp.sLimit + 4 + L2E_BUCKETS + 4 + 2) + 8 * ((size_t)lp.sLimit + 4) + 16;
  const size_t shmS = (size_t)L2S_WARPS * lp.warpBytes;
  if (shmE > (size_t)L2_SHM_BUDGET || shmS > (size_t)L2_SHM_BUDGET) fail(BANI_ERR_INTERNAL, "L2 shared-memory budget exceeded");
  if (ctx->first_time((const void *)l2_seq_kernel)) {
    BANI_CUDA(cudaFuncSetAttribute(l2_events_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, L2_SHM_BUDGET));
    BANI_CUDA(cudaFuncSetAttribute(l2_events_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, L2_SHM_BUDGET));
    BANI_CUDA(cudaFuncSetAttribute(l2_events_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, L2_SHM_BUDGET));
    BANI_CUDA(cudaFuncSetAttribute(l2_seq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L2_SHM_BUDGET));
    BANI_CUDA(cudaFuncSetAttribute(l2_seq_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  }
  sgb.stop();
  { Stage sg(ctx, "l2_events"); sc.idEv = sg.id(); sc.evBytes = 32.0 * (double)totalSteps;
    if (evNT == 256) l2_events_kernel<256><<<F, 256, shmE, st>>>(lp);
    else if (evNT == 128) l2_events_kernel<128><<<F, 128, shmE, st>>>(lp);
    else l2_events_kernel<64><<<F, 64, shmE, st>>>(lp);
    ctx->launches++; }
  { Stage sg(ctx, "l2_seq", sc.evBytes + 16.0 * C);       // the event codes in, {position, shared} out
    l2_seq_kernel<<<nblk(C, L2S_WARPS * 32), L2S_WARPS * 32, shmS, st>>>(lp); ctx->launches++; }
  return P_PIECE_MAPPED;
}

// F: L2.  Bounds of every candidate, the fast path where the index has the window links for it, the exact kernel for
// what is left.  Returns P_PIECE_SPLIT_EVENTS when the piece's window events would not fit.
static PathId l2_candidates(Ctx *ctx, const Index *ix, const QPiece &pc, const Cands &cd, uint64_t *pp, Scores &sc)
{
  cudaStream_t st = ctx->stream;
  const int32_t F = pc.F; const uint32_t C = cd.C; const int smax = pc.smax;
  const int k = ctx->prm.kmer_size, w = ctx->prm.window_size, fragLen = ctx->prm.frag_len;
  const int cmw = fragLen - (w - 1) - (k - 1);         // computeMap.hpp:427
  const bool countPaths = ctx->flags.countPaths != 0;
  BANI_SCRATCH(int32_t, cPos, C);
  BANI_SCRATCH(int32_t, cBest, C);
  sc.pos = cPos; sc.best = cBest;
  L2Args l2; l2.cFrag = cd.frag.p; l2.cSeq = cd.seq.p; l2.cStart = cd.start.p; l2.cEnd = cd.end.p; l2.C = C;
  l2.fragHash = pc.fragHash.p; l2.segStart = pc.segStart.p; l2.sCount = pc.sCount.p;
  l2.recHash = ix->hash.p; l2.recWpos = ix->wpos.p; l2.recLink = ix->link.p; l2.contigRecOff = ix->contigRecOff.p;
  l2.fragLen = fragLen; l2.cmw = cmw; l2.smax = smax;
  l2.stride = ((size_t)2 * (smax + 2) + smax + 15) / 16 * 16;
  const unsigned blocks = (unsigned)std::min<uint64_t>((C + 63) / 64, (uint64_t)ctx->smCount * 16);
  BANI_SCRATCH(uint8_t, scratch, (size_t)blocks * 64 * l2.stride);
  BANI_SCRATCH(unsigned long long, d_n2, 1);
  sc.n2 = d_n2;
  BANI_CUDA(cudaMemsetAsync(d_n2.p, 0, 8, st));
  l2.scratch = scratch.p; l2.cPos = cPos.p; l2.cBest = cBest.p; l2.onlyFlagged = 1;
  Stage sgb(ctx, "l2_bounds", 12.0 * C);
  BANI_SCRATCH(uint32_t, fragCandOff, (size_t)F + 1);
  frag_cand_off_kernel<<<nblk((uint64_t)F + 1), 256, 0, st>>>(cd.frag.p, C, F, fragCandOff.p);
  ctx->launches++;
  L2PArgs lp; lp.cFrag = cd.frag.p; lp.cSeq = cd.seq.p; lp.cStart = cd.start.p; lp.cEnd = cd.end.p; lp.C = C;
  lp.fragCandOff = fragCandOff.p; lp.fragHash = pc.fragHash.p; lp.segStart = pc.segStart.p; lp.sCount = pc.sCount.p;
  lp.rec = ix->rec.p; lp.recWposSoA = ix->wpos.p; lp.contigRecOff = ix->contigRecOff.p; lp.fragLen = fragLen; lp.cmw = cmw;
  lp.rec8 = ix->rec8.p; lp.recLink = ix->link.p; lp.blkMax = ix->blkMax.p; lp.stage = ctx->flags.l2Stage;
  // fast path: needs the window links of the index (cmw >= 2) and ranks that fit the event code
  // (and whose per-warp state fits the shared-memory budget of l2_seq_kernel: larger sketches take l2_kernel)
  // (the switch l2_fast = 0 sends every candidate to l2_kernel)
  lp.sLimit = (ctx->flags.l2Fast && cmw >= 2 && ix->cmw == cmw && ix->rec8.p) ? std::min(std::min(smax, L2_SMAX), L2_SHM_BUDGET / (L2S_WARPS * 32) - 2) : 0;
  // bucket width near 0 ~ 2^32 / (s * w): minimizer hashes are minima of w hashes, density w/2^32 at 0
  lp.nBuckets = ((uint64_t)C >= 8ull * (uint64_t)F) ? L2E_BUCKETS : 1024;      // few candidates per fragment: building a big directory is not worth it
  { const int forced = ctx->flags.l2eBuckets;
    if (forced == 1024 || forced == L2E_BUCKETS) lp.nBuckets = forced; }
  { int sh = lp.nBuckets == L2E_BUCKETS ? 20 : 22; while (sh > 8 && ((uint64_t)std::max(smax, 1) * (uint64_t)w << sh) > ((1ull << 32) * (uint64_t)(L2E_BUCKETS / lp.nBuckets))) sh--; lp.shiftA = sh; }
  lp.warpBytes = (uint32_t)(std::max(lp.sLimit, 1) + 1) * 32u;      // one state byte per rank 0..s and lane
  BANI_SCRATCH(uint32_t, cB0, C);          // (one scratch slot per source line)
  BANI_SCRATCH(uint32_t, cE0, C);
  BANI_SCRATCH(uint32_t, cLast, C);
  BANI_SCRATCH(uint32_t, cNEv, C);
  BANI_SCRATCH(uint32_t, cChunks, (size_t)C + 1);
  BANI_SCRATCH(uint32_t, cOff, (size_t)C + 1);
  BANI_SCRATCH(uint16_t, cMB, (size_t)C + 1);
  lp.cMB = cMB.p;
  lp.cB0 = cB0.p; lp.cE0 = cE0.p; lp.cLast = cLast.p; lp.cNEv = cNEv.p; lp.cChunks = cChunks.p; lp.cOff = cOff.p;
  lp.cPos = cPos.p; lp.cBest = cBest.p; lp.ctr_n2 = d_n2.p; lp.events = nullptr; lp.perm = nullptr;
  l2_bounds_kernel<<<nblk((uint64_t)C + 1), 256, 0, st>>>(lp); ctx->launches++;
  if (countPaths) pp[P_L2_EXACT_AT_BOUNDS] += count_exact(ctx, cBest.p, C);
  if (lp.sLimit > 0 && l2_fast(ctx, pc, lp, cOff.p, sgb, pp, sc) == P_PIECE_SPLIT_EVENTS) return P_PIECE_SPLIT_EVENTS;
  sgb.stop();
  if (countPaths) pp[P_L2_EXACT_TOTAL] += count_exact(ctx, cBest.p, C);
  // exact slow path for whatever the fast path flagged (counter overflow, very large sketches)
  Stage sgs(ctx, "l2_exact");
  l2_kernel<<<blocks, 64, 0, st>>>(l2); ctx->launches++;
  return P_PIECE_MAPPED;
}

// G: report.  R and n2 come back behind one synchronisation; the rows go to *hostRows when it is given.
static void report(Ctx *ctx, const QPiece &pc, const Cands &cd, const Scores &sc, bani_map_counters &ctr,
                   std::vector<bani_mapping> *hostRows, Rows &rw)
{
  cudaStream_t st = ctx->stream;
  const uint32_t C = cd.C;
  RepArgs ra; ra.cFrag = cd.frag.p; ra.cSeq = cd.seq.p; ra.cPos = sc.pos.p; ra.cBest = sc.best.p; ra.C = C;
  ra.sCount = pc.sCount.p; ra.fragSeqId = pc.fragSeqId.p; ra.rowOff = ctx->d_rowOff.p; ra.ident = ctx->d_ident.p;
  ra.upper = ctx->d_upper.p; ra.pid = ctx->prm.perc_identity; ra.fragLen = ctx->prm.frag_len;
  BANI_SCRATCH(uint32_t, keep, C + 1);
  BANI_SCRATCH(uint32_t, keepScan, C + 1);
  keep_flag_kernel<<<nblk(C + 1), 256, 0, st>>>(ra, keep.p);
  ctx->launches++;
  ctx->scan(keep.p, keepScan.p, C + 1);
  unsigned long long n2 = 0;
  BANI_CUDA(cudaMemcpyAsync(&rw.R, keepScan.p + C, 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaMemcpyAsync(&n2, sc.n2.p, 8, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  ctr.n2 += n2; ctr.mappings += rw.R;
  ctx->mark("piece: L1 + L2 done");
  Stage::set_bytes(ctx, sc.idEv, 16.0 * (double)n2 + sc.evBytes);   // 16-byte records in, 2-byte event codes out
  if (rw.R == 0) return;
  const uint32_t R = rw.R;
  BANI_SCRATCH(bani_mapping, rows, R);
  rw.rows = rows; rw.frag.alloc(R, st);
  { Stage sg(ctx, "report", 44.0 * R);
    rows_kernel<<<nblk(C), 256, 0, st>>>(ra, keep.p, keepScan.p, rows.p, rw.frag.p); ctx->launches++; }
  if (hostRows) {
    size_t old = hostRows->size(); hostRows->resize(old + R);
    BANI_CUDA(cudaMemcpyAsync(hostRows->data() + old, rows.p, sizeof(bani_mapping) * (size_t)R, cudaMemcpyDeviceToHost, st));
    BANI_CUDA(cudaStreamSynchronize(st));
  }
}

// Stages C..H of one piece.  Returns P_PIECE_MAPPED, or the reason to map the piece in halves instead; the piece's
// counters and results reach `out` (query slots mapped to query ids) only when it is mapped.
static PathId map_piece(Ctx *ctx, const Index *ix, const QSketch &qs, const QPiece &pc, CgiState *cgi, bool wantRows, MapOutput &out)
{
  bani_map_counters ctr{};
  uint64_t pp[NPATH] = {};
  CgiResult res;
  ctx->mark("piece: begin");
  if (pc.F > 0 && ix->M > 0) {
    ctx->upload_lut(pc.smax, pc.sCount.p, pc.F);
    if (pc.T > 0 && pc.smax > 0) {
      Hits h; Cands cd; Scores sc; Rows rw;
      lookup(ctx, ix, pc, pp, h);
      const unsigned long long maxHits = (unsigned long long)std::max(1ll, ctx->flags.maxHitsPerPiece);    // 1.6 G hits per pass by default
      if (h.N > maxHits && pc.nq > 1) return P_PIECE_SPLIT_HITS;                      // too many hits for one pass
      if (h.N > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "one query genome gathers more than 2^32 index hits");
      ctr.hits = h.N;
      if (h.N > 0) l1_candidates(ctx, ix, pc, h, pp, cd);
      ctr.candidates = cd.C;
      if (cd.C > 0) {
        if (l2_candidates(ctx, ix, pc, cd, pp, sc) == P_PIECE_SPLIT_EVENTS) return P_PIECE_SPLIT_EVENTS;
        report(ctx, pc, cd, sc, ctr, wantRows ? &out.rows : nullptr, rw);
      }
      // H: the identity reduction (cgi.cu)
      if (rw.R > 0 && cgi) cgi_piece(ctx, *cgi, rw.rows.p, rw.frag.p, rw.R, pc.fragQuery.p, pc.nq, pp, res);
    }
    ctr.sum_s = pc.T;
  }
  ctr.fragments = pc.F;
  out.ctr.hits += ctr.hits; out.ctr.candidates += ctr.candidates; out.ctr.n2 += ctr.n2; out.ctr.mappings += ctr.mappings;
  out.ctr.fragments += ctr.fragments; out.ctr.sum_s += ctr.sum_s;
  if (ctx->flags.countPaths) {
    pp[P_PIECE_MAPPED]++;
    for (int i = 0; i < NPATH; i++) ctx->paths[i] += pp[i];
  }
  const int32_t *queryId = qs.queryId.data() + pc.q0;
  const uint64_t *totalFragments = qs.totalFragments.data() + pc.q0;
  if (!res.count.empty()) append_cgi_rows(res.count.data(), res.ident.data(), pc.nq, ix->nGenomes, queryId, totalFragments, out.cgi);
  for (bani_cgi_result r : res.pairs) {
    if (r.countSeq <= 0) continue;
    const int slot = r.qryGenomeId;
    r.qryGenomeId = queryId[slot]; r.totalQueryFragments = (int32_t)totalFragments[slot];
    out.cgi.push_back(r);
  }
  for (bani_frag_mapping &m : res.frags) m.qryGenomeId = queryId[m.qryGenomeId];
  out.frags.insert(out.frags.end(), res.frags.begin(), res.frags.end());
  return P_PIECE_MAPPED;
}

void qsketch_map(Ctx *ctx, const Index *ix, const QSketch *const *sketches, int32_t nSketches,
                 bool wantRows, bool wantCgi, MapOutput &out, bool wantFrags)
{
  cudaStream_t st = ctx->stream;
  wantCgi = wantCgi || wantFrags;
  const int k = ctx->prm.kmer_size, w = ctx->prm.window_size, fragLen = ctx->prm.frag_len;
  if (ix->device != ctx->device) fail(BANI_ERR_ARG, "index lives on another device");
  if (ix->k != k || ix->w != w || ix->fragLen != fragLen)
    fail(BANI_ERR_ARG, "index was built with other parameters (k %d w %d fragLen %d)", ix->k, ix->w, ix->fragLen);
  if (wantCgi && fragLen <= 20) fail(BANI_ERR_ARG, "fragment length must exceed 20 for the identity reduction");
  out.ctr = bani_map_counters{};
  std::unique_ptr<CgiState> cgi;
  if (wantCgi) cgi = std::make_unique<CgiState>(ctx, ix, wantFrags);

  for (int32_t si = 0; si < nSketches; si++) {
    const QSketch *qs = sketches[si];
    if (!qs) fail(BANI_ERR_ARG, "null query sketch");
    if (qs->device != ctx->device) fail(BANI_ERR_ARG, "query sketch lives on another device");
    if (qs->k != k || qs->w != w || qs->fragLen != fragLen) fail(BANI_ERR_ARG, "query sketch was built with other parameters");
    std::deque<const QPiece *> work;
    std::vector<std::unique_ptr<QPiece>> slices;
    for (const auto &pcp : qs->pieces) work.push_back(pcp.get());
    while (!work.empty()) {
      const QPiece &pc = *work.front();
      work.pop_front();
      const PathId r = map_piece(ctx, ix, *qs, pc, cgi.get(), wantRows, out);
      if (r != P_PIECE_MAPPED) {
        // halve the piece at a query boundary (by fragments) and do the halves instead
        if (ctx->flags.countPaths) ctx->paths[r]++;
        int qm = 1;
        while (qm < pc.nq - 1 && pc.qFragOff[qm] < pc.F / 2) qm++;
        slices.push_back(slice_piece(ctx, pc, qm, pc.nq)); work.push_front(slices.back().get());
        slices.push_back(slice_piece(ctx, pc, 0, qm)); work.push_front(slices.back().get());
      }
      if (pc.F > 0 && ix->M > 0) {
        BANI_CUDA(cudaGetLastError());
        BANI_CUDA(cudaStreamSynchronize(st));        // the piece's scratch is reused by the next one
      }
      ctx->mark("piece: rows assembled");
    }
  }
  ctx->mark("qsketch_map: pieces done");
}

} // namespace bani
