// index.cu -- HP1: reference index build.
//
// Replaces skch::Sketch::build + Sketch::index (src/map/include/winSketch.hpp:124-193):
//   build : every contig of every reference genome -> windowed minimizers (sketch.cu), written
//           already ordered by (seqId, wpos) == Sketch::minimizerIndex (winSketch.hpp:94)
//   index : the unordered_map<hash, vector<(seqId,wpos)>> (winSketch.hpp:84) becomes a stable
//           radix sort of (hash -> record index), a run-length compaction into unique keys +
//           offsets, and a bucket directory over the top bits of the hash.
// computeFreqHist (winSketch.hpp:199-248) has no effect at percentageThreshold = 0 (no
// minimizer is ever ignored) and is not reproduced.
//
// Extra, not in the reference: per record the distance (in records) to the previous / next
// record with the same hash.  The L2 stage uses it to keep SET semantics in a sliding window
// without an ordered map (slidingMap.hpp:137-200): a record entering the window adds a new
// distinct hash iff its previous twin is outside, a record leaving removes it iff its next twin
// is outside.
#include "common.cuh"
#include <algorithm>
#include <cstring>
#include <sys/stat.h>

namespace bani {

__global__ void iota_kernel(uint32_t *v, uint64_t n)
{
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = (uint32_t)i;
}

__global__ void head_flags_kernel(const uint32_t *sh, uint64_t n, uint32_t *head)
{
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || sh[i] != sh[i - 1]) ? 1u : 0u;
}

__global__ void unique_scatter_kernel(const uint32_t *sh, const uint32_t *head, const uint32_t *scan, uint64_t n,
                                      uint32_t *ukeys, uint32_t *uoff, unsigned long long *o_U)
{
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (head[i]) { ukeys[scan[i]] = sh[i]; uoff[scan[i]] = (uint32_t)i; }
  if (i == n - 1) { uint32_t U = scan[i] + head[i]; *o_U = U; }
}

// Twin links.  Only a few percent of the records share their hash with another record, so the link array is
// pre-filled with "no twin" (memset 0xFF) and only records that have a NEAR one are written (a 4-byte scatter).
__global__ void links_kernel(const uint32_t *sh, const uint32_t *posIdx, uint64_t n, uint32_t *link)
{
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = sh[i];
  const bool hasPrev = i > 0 && sh[i - 1] == h, hasNext = i + 1 < n && sh[i + 1] == h;
  if (!hasPrev && !hasNext) return;
  const uint32_t r = posIdx[i];
  uint32_t pd = 0xFFFFu, nd = 0xFFFFu;
  if (hasPrev) pd = min(r - posIdx[i - 1], 0xFFFFu);       // stable sort: twins ascend by record index
  if (hasNext) nd = min(posIdx[i + 1] - r, 0xFFFFu);
  // a twin 65535 or more records away reads as "no twin" (no window is that long): in collections of related
  // genomes almost every hash recurs in a sister genome millions of records away, and none of those needs a write
  if (pd != 0xFFFFu || nd != 0xFFFFu) link[r] = (pd << 16) | nd;
}

// One 16-byte record per minimizer for the L2 stream: x = hash, y = wpos | tie << 31, z = twin link,
// w = back | fwd << 16.  back / fwd / tie describe the L2 super-window geometry of computeL2MappedRegions
// (computeMap.hpp:418-497) around this record, which does not depend on the candidate (cmw is fixed):
//   back : records strictly after the window start when this record ENTERS the window, i.e.
//          x - (UB(w_x - cmw + 1) - 1), UB = first record of the contig with wpos > v
//   fwd  : LB(w_{x+1} + cmw - 1) - x, the window end (exclusive) when this record LEAVES the window
//          (0xFFFF for the last record of a contig: it never leaves inside a scored window)
//   tie  : the record at x + fwd enters in the same step in which x leaves (wpos equal to w_{x+1} + cmw - 1)
// so the event schedule of a candidate needs no search (map.cu, l2_events_kernel).
__global__ void zip_records_kernel(const uint32_t *hash, const int32_t *wpos, const uint32_t *link, const int32_t *seqId,
                                   const uint32_t *contigRecOff, int cmw, uint64_t n, uint4 *rec, int2 *pos8, uint2 *rec8)
{
  uint64_t i64 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i64 >= n) return;
  const uint32_t i = (uint32_t)i64;
  const int32_t wx = wpos[i];
  const int seq = seqId[i];
  const uint32_t lo = contigRecOff[seq], hi = contigRecOff[seq + 1];
  uint32_t back = 0, fwd = 0xFFFFu, tie = 0;
  if (cmw >= 2) {
    { // UB(wx - cmw + 1) over [lo, i]: the answer is within cmw records of i
      const int32_t v = wx - cmw + 1;
      uint32_t l = (i - lo > (uint32_t)cmw) ? i - (uint32_t)cmw : lo, h = i;
      while (l < h) { uint32_t m = (l + h) >> 1; if (wpos[m] <= v) l = m + 1; else h = m; }
      back = min(i - l + 1, 0xFFFFu);
    }
    if (i + 1 < hi) {
      const int32_t v = wpos[i + 1] + cmw - 1;
      uint32_t l = i + 1, h = (hi - i - 1 > (uint32_t)cmw + 1) ? i + 1 + (uint32_t)cmw + 1 : hi;
      while (l < h) { uint32_t m = (l + h) >> 1; if (wpos[m] < v) l = m + 1; else h = m; }
      fwd = min(l - i, 0xFFFEu);
      tie = (l < hi && wpos[l] == v) ? 1u : 0u;
    }
  }
  rec[i] = make_uint4(hash[i], (uint32_t)wx | (tie << 31), link[i], back | (fwd << 16));
  pos8[i] = make_int2(wx, seq);
  // compact form for the staged L2 path: the two twin tests do not depend on the candidate once the record is past the
  // first window -- new distinct hash on entering iff the previous twin is further than `back`, distinct hash gone on
  // leaving iff the next twin is at least `fwd` ahead -- so two bits replace the twin distances
  const uint32_t pd = link[i] >> 16, nd = link[i] & 0xFFFFu;
  const uint32_t f14 = fwd == 0xFFFFu ? 0x3FFFu : min(fwd, 0x3FFEu);
  rec8[i] = make_uint2(hash[i], (back & 0x3FFFu) | (f14 << 14) | (tie << 28) | ((pd > back ? 1u : 0u) << 29) | ((nd >= fwd ? 1u : 0u) << 30));
}

// Per block of 1024 records: the largest `back` and the largest `fwd` (last records of a contig, which never leave, aside).
// l2_bounds_kernel takes the maximum over the blocks a candidate touches to decide whether its events fit the
// shared-memory ring of l2_events_kernel; 0xFFFF marks a block with a link that does not fit the 14-bit fields of rec8.
__global__ void block_link_max_kernel(const uint4 *rec, uint64_t n, uint32_t *blkMax)
{
  __shared__ uint32_t s_b, s_f;
  if (threadIdx.x == 0) { s_b = 0; s_f = 0; }
  __syncthreads();
  uint32_t mb = 0, mf = 0;
  for (int j = 0; j < 4; j++) {
    const uint64_t i = (uint64_t)blockIdx.x * 1024 + (uint64_t)j * 256 + threadIdx.x;
    if (i < n) {
      const uint32_t w = rec[i].w, back = w & 0xFFFFu, fwd = w >> 16;
      if (back >= 0x3FFFu || (fwd != 0xFFFFu && fwd >= 0x3FFFu)) { mb = 0xFFFFu; mf = 0xFFFFu; }
      else { mb = max(mb, back); if (fwd != 0xFFFFu) mf = max(mf, fwd); }
    }
  }
  atomicMax(&s_b, mb); atomicMax(&s_f, mf);
  __syncthreads();
  if (threadIdx.x == 0) blkMax[blockIdx.x] = min(s_b, 0xFFFFu) | (min(s_f, 0xFFFFu) << 16);
}

__global__ void dir_fill_kernel(const uint32_t *ukeys, uint32_t U, int dirBits, uint32_t *dir)
{
  // dir[b] = lower_bound(ukeys, b << (32 - dirBits)); minimizer hashes are minima of w hashes, hence heavily
  // skewed towards small values: most high buckets are empty, so every bucket searches for itself
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > (1u << dirBits)) return;
  uint32_t lo = 0, hi = U;
  if (b == (1u << dirBits)) lo = U;
  else { const uint32_t v = b << (32 - dirBits); while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (ukeys[mid] < v) lo = mid + 1; else hi = mid; } }
  dir[b] = lo;
}

// Probe table of the lookup stage (Index::tab): every unique hash claims one of the 4 slots of bucket (hash & mask) with
// a 64-bit compare-and-swap; keys that find their bucket full stay reachable through the sorted key array.  Which 4 keys
// of an overfull bucket get in depends on the order of the atomics, the result of a lookup does not.
__global__ void table_fill_kernel(const uint32_t *ukeys, const uint32_t *uoff, uint32_t U, uint32_t mask, uint2 *tab,
                                  uint32_t *filt, uint32_t filtMask)
{
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= U) return;
  const uint32_t h = ukeys[u], o = uoff[u], cnt = uoff[u + 1] - o;
  if (filt) atomicOr(&filt[(h & filtMask) >> 5], 1u << (h & 31u));
  const unsigned long long e = ((unsigned long long)o << 32) | (unsigned long long)((h & 0xFFFFFF00u) | min(cnt, 255u));
  unsigned long long *bp = reinterpret_cast<unsigned long long *>(tab + 4 * (size_t)(h & mask));
#pragma unroll
  for (int sl = 0; sl < 4; sl++) if (atomicCAS(bp + sl, 0ull, e) == 0ull) return;
}

__global__ void fill_u32(uint32_t *p, uint32_t v, uint64_t n)
{
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---- host-side contig tables shared by index_build and index_load: position bins (CGI), validity-bitmap bases
static unsigned long long index_contig_tables(Ctx *ctx, Index *ix, const std::vector<int32_t> &contigGenome)
{
  cudaStream_t st = ctx->stream;
  const int fragLen = ix->fragLen;
  const int32_t nC = (int32_t)ix->contigLen.size();
  std::vector<uint32_t> binOff(1, 0);
  std::vector<unsigned long long> bitBase;
  unsigned long long totalBits = 0;
  ix->totalLen = 0;
  for (int32_t c = 0; c < nC; c++) {
    const int32_t L = ix->contigLen[c];
    bitBase.push_back(totalBits); totalBits += ((unsigned long long)L + 31) & ~31ull;
    const uint64_t bins = (fragLen > 20) ? (uint64_t)L / (uint64_t)(fragLen - 20) + 1 : 1;
    if (binOff.back() + bins > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "reference too large for 32-bit position bins");
    binOff.push_back((uint32_t)(binOff.back() + bins));
    ix->totalLen += (uint64_t)L;
  }
  ix->nContigs = nC;
  ix->totalBins = binOff.back();
  ix->contigRecOff.alloc((size_t)nC + 1, st);
  ix->contigGenome.alloc(std::max(nC, 1), st);
  ix->contigBinOff.alloc((size_t)nC + 1, st);
  BANI_CUDA(cudaMemcpyAsync(ix->contigBinOff.p, binOff.data(), 4 * (size_t)(nC + 1), cudaMemcpyHostToDevice, st));
  if (nC) BANI_CUDA(cudaMemcpyAsync(ix->contigGenome.p, contigGenome.data(), 4 * (size_t)nC, cudaMemcpyHostToDevice, st));
  if (nC) {
    ix->contigBitBase.alloc(nC, st);
    BANI_CUDA(cudaMemcpyAsync(ix->contigBitBase.p, bitBase.data(), 8 * (size_t)nC, cudaMemcpyHostToDevice, st));
  }
  BANI_CUDA(cudaStreamSynchronize(st));          // the host vectors go out of scope
  return totalBits;
}

static void index_make_empty(Ctx *ctx, Index *ix)
{
  cudaStream_t st = ctx->stream;
  // empty index: every lookup misses (a shard with no references, computeCoreIdentity.hpp:468-471)
  fill_u32<<<nblk(ix->nContigs + 1), 256, 0, st>>>(ix->contigRecOff.p, 0, (uint64_t)ix->nContigs + 1);
  ctx->launches++;
  ix->M = 0; ix->U = 0;
  ix->dirBits = 8;
  ix->dir.alloc((1u << ix->dirBits) + 1, st);
  BANI_CUDA(cudaMemsetAsync(ix->dir.p, 0, 4 * ((1u << ix->dirBits) + 1), st));
  ix->ukeys.alloc(1, st); ix->uoff.alloc(2, st); ix->posIdx.alloc(1, st);
  BANI_CUDA(cudaMemsetAsync(ix->uoff.p, 0, 8, st));
  ix->tabBits = 8; ix->tab.alloc((size_t)4 << ix->tabBits, st);
  BANI_CUDA(cudaMemsetAsync(ix->tab.p, 0, ix->tab.bytes(), st));
  ix->hash.alloc(1, st); ix->wpos.alloc(1, st); ix->seqId.alloc(1, st); ix->link.alloc(1, st);
  BANI_CUDA(cudaStreamSynchronize(st));
}

// ---- Sketch::index (winSketch.hpp:181-193): the hash-ordered side and the per-record links from the position-ordered
//      records (ix->hash / wpos / seqId / contigRecOff filled, ix->M > 0)
static void index_finish(Ctx *ctx, Index *ix)
{
  cudaStream_t st = ctx->stream;
  const uint64_t M = ix->M;
  ix->link.alloc(M, st);
  ix->posIdx.alloc(M, st);
  DevBuf<uint32_t> sortedHash(M, st), iota(M, st), head(M, st), scan(M, st);
  DevBuf<unsigned long long> d_U(1, st);
  {
    Stage sg(ctx, "index_sort", 24.0 * M);
    iota_kernel<<<nblk(M), 256, 0, st>>>(iota.p, M);
    ctx->launches++;
    size_t tb = cub_sort_pairs_u32_temp(M);
    DevBuf<uint8_t> tmp(tb, st);
    cub_sort_pairs_u32(tmp.p, tb, ix->hash.p, sortedHash.p, iota.p, ix->posIdx.p, M, 32, st);
  }
  Stage sgc(ctx, "index_compact", 16.0 * M);
  head_flags_kernel<<<nblk(M), 256, 0, st>>>(sortedHash.p, M, head.p);
  ctx->launches++;
  {
    size_t tb = cub_scan_u32_temp(M);
    DevBuf<uint8_t> tmp(tb, st);
    cub_exclusive_sum_u32(tmp.p, tb, head.p, scan.p, M, st);
  }
  // U is needed to size ukeys: read scan[M-1] + head[M-1]
  uint32_t lastScan = 0, lastHead = 0;
  BANI_CUDA(cudaMemcpyAsync(&lastScan, scan.p + (M - 1), 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaMemcpyAsync(&lastHead, head.p + (M - 1), 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  const uint64_t U = (uint64_t)lastScan + lastHead;
  ix->U = U;
  ix->ukeys.alloc(U, st); ix->uoff.alloc(U + 1, st);
  unique_scatter_kernel<<<nblk(M), 256, 0, st>>>(sortedHash.p, head.p, scan.p, M, ix->ukeys.p, ix->uoff.p, d_U.p);
  ctx->launches++;
  { uint32_t Mu = (uint32_t)M; BANI_CUDA(cudaMemcpyAsync(ix->uoff.p + U, &Mu, 4, cudaMemcpyHostToDevice, st)); }
  BANI_CUDA(cudaMemsetAsync(ix->link.p, 0xFF, 4 * (size_t)M, st));
  links_kernel<<<nblk(M), 256, 0, st>>>(sortedHash.p, ix->posIdx.p, M, ix->link.p);
  ctx->launches++;
  const int bits = index_dir_bits(U);       // <= 32 MB: the directory stays L2-resident (50 MB) during a lookup launch
  ix->dirBits = bits;
  ix->dir.alloc((1u << bits) + 1, st);
  dir_fill_kernel<<<nblk((1ull << bits) + 1), 256, 0, st>>>(ix->ukeys.p, (uint32_t)U, bits, ix->dir.p);
  ctx->launches++;
  {   // probe table: 2^tabBits >= U buckets (load <= 1 key per 4-slot bucket: ~2 % of the buckets are full), at most 2^28 (8.6 GB)
    const int tb = index_tab_bits(U);
    ix->tabBits = tb;
    ix->tab.alloc((size_t)4 << tb, st);
    BANI_CUDA(cudaMemsetAsync(ix->tab.p, 0, ix->tab.bytes(), st));
    const int fb = index_filt_bits(U);      // <= 32 MB of bits
    ix->filtBits = fb;
    if (fb) { ix->filt.alloc((size_t)1 << (fb - 5), st); BANI_CUDA(cudaMemsetAsync(ix->filt.p, 0, ix->filt.bytes(), st)); }
    table_fill_kernel<<<nblk(U), 256, 0, st>>>(ix->ukeys.p, ix->uoff.p, (uint32_t)U, (1u << tb) - 1u, ix->tab.p,
                                               ix->filt.p, fb ? (uint32_t)((1ull << fb) - 1ull) : 0u);
    ctx->launches++;
  }
  ix->rec.alloc(M, st);
  ix->cmw = ix->fragLen - (ix->w - 1) - (ix->k - 1);       // computeMap.hpp:427
  ix->pos8.alloc(M, st); ix->rec8.alloc(M, st);
  zip_records_kernel<<<nblk(M), 256, 0, st>>>(ix->hash.p, ix->wpos.p, ix->link.p, ix->seqId.p, ix->contigRecOff.p, ix->cmw, M, ix->rec.p, ix->pos8.p, ix->rec8.p);
  ctx->launches++;
  ix->blkMax.alloc((size_t)((M + 1023) / 1024), st);
  block_link_max_kernel<<<(unsigned)((M + 1023) / 1024), 256, 0, st>>>(ix->rec.p, M, ix->blkMax.p);
  ctx->launches++;
  sgc.stop();
  BANI_CUDA(cudaGetLastError());
  BANI_CUDA(cudaStreamSynchronize(st));
}

// Host sizes of genome g's part of an index: contigs, hashed positions (contigs of at least k bases) and validity bits.
struct GenomeSpan { uint64_t nC = 0, pos = 0, bits = 0; };
static GenomeSpan genome_span(const Genome *G, int k)
{
  GenomeSpan s;
  s.nC = (uint64_t)G->nContigs;
  for (int c = 0; c < G->nContigs; c++) {
    if (G->len[c] >= k) s.pos += (uint64_t)(G->len[c] - k + 1);
    s.bits += ((uint64_t)G->len[c] + 31) & ~31ull;
  }
  return s;
}

// Budgeted build, after the sketch launch over genomes [0, n): keeps the longest prefix whose records were all stored (<=
// `stored`) and whose exact build (index_footprint with U <= M, the staging capacity that was used and the tables of all
// launched genomes, which are alive until the cut) fits maxBytes, and
// shrinks the contig tables, the genome table and the validity bitmap to it.  Returns the prefix's record count.
static uint64_t index_cut(Ctx *ctx, Index *ix, Genome *const *refs, std::vector<int32_t> &contigGenome, const std::vector<GenomeSpan> &span,
                          uint64_t stored, uint64_t cap, uint64_t maxBytes, int32_t *nTaken)
{
  cudaStream_t st = ctx->stream;
  const int32_t n = (int32_t)ix->seqsByFile.size();
  std::vector<uint32_t> recOff((size_t)ix->nContigs + 1);
  BANI_CUDA(cudaMemcpyAsync(recOff.data(), ix->contigRecOff.p, 4 * recOff.size(), cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  // the contig tables and the bitmap of every launched genome stay alive until the cut: they are charged in full
  uint64_t launchedBits = 0;
  for (int32_t g = 0; g < n; g++) launchedBits += span[g].bits;
  const uint64_t launchedC = (uint64_t)ix->nContigs;
  int32_t t = 0;
  uint64_t nC = 0, M = 0;
  for (; t < n; t++) {
    const uint64_t c2 = (uint64_t)ix->seqsByFile[t], m2 = recOff[c2];
    if (m2 > stored || index_footprint(m2, m2, launchedC, launchedBits, cap).peak > maxBytes) break;
    nC = c2; M = m2;
  }
  if (t == 0)
    fail(BANI_ERR_LIMIT, "reference genome 0 of this chunk (%llu minimizers) does not fit the index budget of %llu bytes: its "
         "index needs %llu", (unsigned long long)recOff[ix->seqsByFile[0]], (unsigned long long)maxBytes,
         (unsigned long long)index_footprint(recOff[ix->seqsByFile[0]], recOff[ix->seqsByFile[0]], launchedC, launchedBits, cap).peak);
  *nTaken = t;
  if (t == n) return M;
  // the prefix's tables, as index_build would have made them from exactly these genomes
  ix->members.clear();
  for (int32_t g = 0, c = 0; g < t; c += refs[g]->nContigs, g++) ix->members.emplace(refs[g]->uid, c);
  ix->nGenomes = t;
  ix->seqsByFile.resize(t);
  ix->contigLen.resize(nC);
  contigGenome.resize(nC);
  DevBuf<uint32_t> oldRecOff = std::move(ix->contigRecOff);
  DevBuf<uint32_t> oldBits = std::move(ix->validBits);
  const unsigned long long totalBits = index_contig_tables(ctx, ix, contigGenome);     // totalBits == bits: whole words
  BANI_CUDA(cudaMemcpyAsync(ix->contigRecOff.p, oldRecOff.p, 4 * (nC + 1), cudaMemcpyDeviceToDevice, st));
  ix->validBits.alloc((size_t)(totalBits / 32) + 1, st);
  BANI_CUDA(cudaMemsetAsync(ix->validBits.p, 0, ix->validBits.bytes(), st));
  if (totalBits) BANI_CUDA(cudaMemcpyAsync(ix->validBits.p, oldBits.p, totalBits / 8, cudaMemcpyDeviceToDevice, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  return M;
}

// maxBytes = 0: the whole list.  maxBytes > 0 (index_build_budget): the longest prefix whose build fits (*nTaken).
//   Before the sketch launch only the expected record count is known: the launch takes the longest prefix whose expected
//   build fits (at least one genome, whose staging and tables alone must fit).  After it, contigRecOff holds the exact
//   record count of every genome; records are in (seqId, wpos) order, so a prefix of genomes is a prefix of the records,
//   of the validity bitmap and of the contig tables, and the index is cut there before anything that grows with M or U
//   is allocated.
static Index *index_build_impl(Ctx *ctx, Genome *const *refs, int32_t nRefs, uint64_t maxBytes, int32_t *nTaken)
{
  cudaStream_t st = ctx->stream;
  const int k = ctx->prm.kmer_size, w = ctx->prm.window_size, fragLen = ctx->prm.frag_len;
  const bool budget = maxBytes > 0;
  std::vector<GenomeSpan> span;
  if (budget) {
    for (int g = 0; g < nRefs; g++) {
      if (!refs[g]) fail(BANI_ERR_ARG, "null genome handle");
      span.push_back(genome_span(refs[g], k));
    }
    GenomeSpan p;
    int32_t n = 0;
    for (; n < nRefs; n++) {
      GenomeSpan q = p; q.nC += span[n].nC; q.pos += span[n].pos; q.bits += span[n].bits;
      const uint64_t cap = index_staging_cap(q.pos, w), Mexp = (uint64_t)(2.0 * (double)q.pos / (w + 1));
      // genome 0: its staging and tables must fit (its records are counted after the launch); later genomes: the whole
      // expected build
      const uint64_t need = n == 0 ? index_footprint(0, 0, q.nC, q.bits, cap).peak : index_footprint(Mexp, Mexp, q.nC, q.bits, cap).peak;
      if (need > maxBytes || (n > 0 && cap > 0xfffffff0ull)) break;
      p = q;
    }
    if (n == 0)
      fail(BANI_ERR_LIMIT, "reference genome 0 of this chunk (%llu bases) does not fit the index budget of %llu bytes: its sketch "
           "staging alone needs %llu", (unsigned long long)span[0].pos, (unsigned long long)maxBytes,
           (unsigned long long)index_footprint(0, 0, span[0].nC, span[0].bits, index_staging_cap(span[0].pos, w)).peak);
    nRefs = n;
  }
  *nTaken = nRefs;
  auto ix = std::make_unique<Index>();
  ix->device = ctx->device;
  ix->nGenomes = nRefs;
  ix->k = k; ix->w = w; ix->fragLen = fragLen;

  // ---- contig table over all genomes (every contig consumes a seqId: winSketch.hpp:150,164)
  std::vector<SeqDesc> desc;
  std::vector<int32_t> contigGenome;
  uint64_t totalPos = 0;
  for (int g = 0; g < nRefs; g++) {
    const Genome *G = refs[g];
    if (!G) fail(BANI_ERR_ARG, "null genome handle");
    if (G->device != ctx->device) fail(BANI_ERR_ARG, "genome lives on another device");
    ix->members.emplace(G->uid, (int32_t)desc.size());          // first occurrence wins if a genome is listed twice
    for (int c = 0; c < G->nContigs; c++) {
      SeqDesc d;
      d.packed = G->packedBase() + G->wordOff[c];
      d.nExc = (int32_t)(G->excOff[c + 1] - G->excOff[c]);
      d.excPos = d.nExc ? G->excPosBase() + G->excOff[c] : nullptr;
      d.excByte = d.nExc ? G->excByteBase() + G->excOff[c] : nullptr;
      d.startBase = 0; d.len = G->len[c]; d.seqId = (int32_t)desc.size();
      desc.push_back(d);
      ix->contigLen.push_back(G->len[c]);
      contigGenome.push_back(g);
      if (G->len[c] >= k) totalPos += G->len[c] - k + 1;
    }
    ix->seqsByFile.push_back((int32_t)desc.size());
  }
  const int32_t nC = (int32_t)desc.size();
  ctx->mark("index_build: enter + contig loop");
  const unsigned long long totalBits = index_contig_tables(ctx, ix.get(), contigGenome);
  ctx->mark("index_build: contig tables");

  if (nC == 0 || totalPos == 0) { index_make_empty(ctx, ix.get()); return ix.release(); }

  ix->validBits.alloc((size_t)(totalBits / 32) + 1, st);
  BANI_CUDA(cudaMemsetAsync(ix->validBits.p, 0, ix->validBits.bytes(), st));
  DevBuf<SeqDesc> d_desc(nC, st);
  BANI_CUDA(cudaMemcpyAsync(d_desc.p, desc.data(), sizeof(SeqDesc) * (size_t)nC, cudaMemcpyHostToDevice, st));

  // ---- build: minimizers in (seqId, wpos) order.  Expected density 2/(w+1); capacity 1.5x that,
  //      exact retry if a repetitive reference exceeds it (worst case one record per position).
  uint64_t cap = index_staging_cap(totalPos, w);
  uint64_t M = 0;
  {
    DevBuf<uint32_t> th; DevBuf<int32_t> tw, ts;
    // genomes that share an upload block (host-packed ingest) form a group: one sketch launch per group, issued as
    // soon as the group's H2D copies have landed, so the upload of group g+1 overlaps the hashing of group g
    std::vector<std::pair<int32_t, int32_t>> groups;              // [first contig, end contig)
    std::vector<const Genome *> groupHead;
    {
      int32_t c = 0;
      for (int g = 0; g < nRefs; g++) {
        const Genome *G = refs[g];
        const bool newGroup = groups.empty() || G->blk != groupHead.back()->blk;       // genomes with their own buffers (no block) share one group
        if (newGroup) { groups.push_back({c, c}); groupHead.push_back(G); }
        c += G->nContigs; groups.back().second = c;
      }
    }
    for (int attempt = 0; attempt < 2; attempt++) {
      if (cap > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "more than 2^32 minimizers in one index shard");
      th.alloc(cap, st); tw.alloc(cap, st); ts.alloc(cap, st);
      Stage sg(ctx, "ref_sketch", (double)ix->totalLen / 4.0);
      M = 0;
      for (size_t gi = 0; gi < groups.size(); gi++) {
        const int32_t ca = groups[gi].first, cb = groups[gi].second;
        groupHead[gi]->wait_ready(st);
        M += sketch_sequences(ctx, d_desc.p + ca, cb - ca, ix->contigLen.data() + ca, 0, th.p, tw.p, ts.p, cap, ix->contigRecOff.p + ca,
                              ix->validBits.p, ix->contigBitBase.p + ca, M);
        if (M > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "more than 2^32 minimizers in one index shard");
      }
      sg.bytes((double)ix->totalLen / 4.0 + 12.0 * (double)M);       // packed bases in, 12-byte records out
      ctx->mark("index_build: sketched");
      if (M <= cap) break;
      if (budget) {
        // only the genomes whose records were all stored can be kept: retry with an exact staging for genome 0 if even it
        // overflowed the expected capacity
        uint32_t r1 = 0;
        BANI_CUDA(cudaMemcpyAsync(&r1, ix->contigRecOff.p + ix->seqsByFile[0], 4, cudaMemcpyDeviceToHost, st));
        BANI_CUDA(cudaStreamSynchronize(st));
        if (r1 <= cap) break;
        if (index_footprint(r1, r1, (uint64_t)nC, totalBits, r1).peak > maxBytes)
          fail(BANI_ERR_LIMIT, "reference genome 0 of this chunk (%llu minimizers) does not fit the index budget of %llu bytes",
               (unsigned long long)r1, (unsigned long long)maxBytes);
        cap = r1;
        continue;
      }
      cap = M;
    }
    d_desc.release();                                             // the descriptors are only read by the sketch launch
    if (budget) M = index_cut(ctx, ix.get(), refs, contigGenome, span, std::min(M, cap), cap, maxBytes, nTaken);
    if (M > 0xfffffff0ull) fail(BANI_ERR_LIMIT, "more than 2^32 minimizers in one index shard");
    ix->M = M;
    if (M == 0) { index_make_empty(ctx, ix.get()); return ix.release(); }
    ix->hash.alloc(M, st); ix->wpos.alloc(M, st); ix->seqId.alloc(M, st);
    BANI_CUDA(cudaMemcpyAsync(ix->hash.p, th.p, 4 * M, cudaMemcpyDeviceToDevice, st));
    BANI_CUDA(cudaMemcpyAsync(ix->wpos.p, tw.p, 4 * M, cudaMemcpyDeviceToDevice, st));
    BANI_CUDA(cudaMemcpyAsync(ix->seqId.p, ts.p, 4 * M, cudaMemcpyDeviceToDevice, st));
  }
  index_finish(ctx, ix.get());
  ctx->mark("index_build: finished");
  return ix.release();
}

Index *index_build(Ctx *ctx, Genome *const *refs, int32_t nRefs)
{
  int32_t n = 0;
  return index_build_impl(ctx, refs, nRefs, 0, &n);
}

// make(): *peakBytes = the most device memory held during the call above what was held on entry
template <typename F>
static Index *with_peak(Ctx *ctx, uint64_t *peakBytes, F &&make)
{
  size_t live0 = 0, peak0 = 0, peak = 0;
  dev_mem_stats(ctx->device, &live0, nullptr, &peak0);
  dev_mem_peak_set(ctx->device, 0);                        // high-water mark from here on
  Index *ix = nullptr;
  try { ix = make(); }
  catch (...) { dev_mem_stats(ctx->device, nullptr, nullptr, &peak); dev_mem_peak_set(ctx->device, std::max(peak0, peak)); throw; }
  dev_mem_stats(ctx->device, nullptr, nullptr, &peak);
  dev_mem_peak_set(ctx->device, std::max(peak0, peak));
  *peakBytes = peak > live0 ? peak - live0 : 0;
  return ix;
}

Index *index_build_budget(Ctx *ctx, Genome *const *refs, int32_t nRefs, uint64_t maxBytes, int32_t *nTaken, uint64_t *peakBytes)
{
  if (nRefs < 1) fail(BANI_ERR_ARG, "a budgeted index build needs at least one genome");
  if (maxBytes == 0) fail(BANI_ERR_ARG, "the index budget must be positive");
  return with_peak(ctx, peakBytes, [&] { return index_build_impl(ctx, refs, nRefs, maxBytes, nTaken); });
}


// ---------------------------------------------------------------------------------------- on-disk sketch cache (SURVEY 8 f-4)
// The reference has no cache (only scripts/splitDatabase.sh + README.md:104-106: "divide the database, run as parallel
// processes"), so every run reads and sketches every reference again.  A saved index holds what only the sketch launch
// can produce -- the position-ordered (hash, wpos) records, the contig table and the validity bitmap -- as one flat
// little-endian file; the hash-ordered side, the links and the L2 records are rebuilt on the GPU at load time (a sort
// and a few passes: cheaper than reading them from disk).  A loaded index also serves as the QUERY side of its own
// genomes (qsketch_from_index): an all-vs-all run against a cache reads no FASTA at all.
//   u64 x 16 : magic, version, k, w, fragLen, M, nContigs, nGenomes, validWords, 0...
//   i32 contigLen[nContigs] | i32 seqsByFile[nGenomes] | u32 contigRecOff[nContigs+1] | u32 hash[M] | i32 wpos[M] |
//   u32 validBits[validWords] |
//   version 3 only: u64 tableSum | u64 genomeSum[nGenomes] |
//   u64 checksum (sum of all preceding 32-bit words)
// A sum is the 64-bit sum of the 32-bit words it covers.  tableSum covers the header, contigLen, seqsByFile and
// contigRecOff; genomeSum[g] covers genome g's records -- its slices of hash and of wpos -- and its validity bitmap words
// (every contig's bits start on a word, so a genome's bits are whole words).  The last bitmap word lies past every contig
// and is zero.  So a run of genomes can be read and checked without reading the rest of the file (index_load_budget,
// qsketch_from_index_file).  Version 2 files have the whole-file checksum only and are loaded whole.
static constexpr uint64_t IX_MAGIC = 0x32584449494e4142ull;
static constexpr uint64_t IX_HEADER_BYTES = 128;

__global__ void seqid_fill_kernel(const uint32_t *contigRecOff, int32_t nC, int32_t *seqId)
{
  const int c = blockIdx.x;
  if (c >= nC) return;
  const uint32_t a = contigRecOff[c], b = contigRecOff[c + 1];
  for (uint32_t i = a + threadIdx.x; i < b; i += blockDim.x) seqId[i] = c;
}

static uint64_t word_sum(const void *p, size_t bytes)
{
  const uint32_t *w = (const uint32_t *)p;
  uint64_t s = 0;
  for (size_t i = 0; i < bytes / 4; i++) s += w[i];
  return s;
}

namespace {
struct File {
  FILE *f = nullptr; std::string path; uint64_t sum = 0;
  File(const char *p, const char *mode) : f(fopen(p, mode)), path(p) { if (!f) fail(BANI_ERR_ARG, "cannot open %s", p); }
  ~File() { if (f) fclose(f); }
  void write(const void *p, size_t n) { put(p, n); sum += word_sum(p, n); }
  void read(void *p, size_t n) { get(p, n); sum += word_sum(p, n); }
  // the same without adding to `sum`: for callers that sum the words themselves
  void put(const void *p, size_t n) { if (n && fwrite(p, 1, n, f) != n) fail(BANI_ERR_INTERNAL, "write error on %s", path.c_str()); }
  void get(void *p, size_t n) { if (n && fread(p, 1, n, f) != n) fail(BANI_ERR_ARG, "%s is truncated", path.c_str()); }
  void seek(uint64_t off) { if (fseeko(f, (off_t)off, SEEK_SET) != 0) fail(BANI_ERR_ARG, "%s: cannot seek to byte %llu", path.c_str(), (unsigned long long)off); }
};

// Disk -> device through two pinned buffers: the disk read of a piece overlaps the copy of the previous one.
struct Upload {
  static constexpr size_t CH = (size_t)64 << 20;
  cudaStream_t st; File &f;
  void *stage[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  int cur = 0; bool used[2] = {false, false};
  Upload(Ctx *ctx, File &file) : st(ctx->stream), f(file)
  {
    try {
      BANI_CUDA(cudaHostAlloc(&stage[0], CH, cudaHostAllocDefault));
      BANI_CUDA(cudaHostAlloc(&stage[1], CH, cudaHostAllocDefault));
      BANI_CUDA(cudaEventCreate(&ev[0])); BANI_CUDA(cudaEventCreate(&ev[1]));
    } catch (...) { release(); throw; }
  }
  ~Upload() { release(); }
  void release()
  {
    cudaStreamSynchronize(st);
    for (int i = 0; i < 2; i++) {
      if (stage[i]) cudaFreeHost(stage[i]);
      if (ev[i]) cudaEventDestroy(ev[i]);
      stage[i] = nullptr; ev[i] = nullptr;
    }
  }
  // `bytes` from the file's current position to device address dp; *sum (optional) += their word sum
  void copy(void *dp, uint64_t bytes, uint64_t *sum = nullptr)
  {
    for (uint64_t o = 0; o < bytes; o += CH) {
      const size_t n = (size_t)std::min<uint64_t>(CH, bytes - o);
      if (used[cur]) BANI_CUDA(cudaEventSynchronize(ev[cur]));
      f.read(stage[cur], n);
      if (sum) *sum += word_sum(stage[cur], n);
      BANI_CUDA(cudaMemcpyAsync((uint8_t *)dp + o, stage[cur], n, cudaMemcpyHostToDevice, st));
      BANI_CUDA(cudaEventRecord(ev[cur], st));
      used[cur] = true; cur ^= 1;
    }
  }
  void finish() { BANI_CUDA(cudaStreamSynchronize(st)); }
};
}

uint64_t IndexFileInfo::off_hash() const { return IX_HEADER_BYTES + 4 * nContigs + 4 * nGenomes + 4 * (nContigs + 1); }
uint64_t IndexFileInfo::off_sums() const { return off_bits() + 4 * validWords; }
uint64_t IndexFileInfo::file_bytes() const { return off_sums() + (version >= 3 ? 8 + 8 * nGenomes : 0) + 8; }

// Header and tables of a saved index, checked as a whole load checks them and, version 3, against tableSum first (a
// corrupt table is reported as such).  The file is left after contigRecOff, with f.sum the sum of everything read so far.
static IndexFileInfo index_file_tables(File &f)
{
  const char *path = f.path.c_str();
  IndexFileInfo x;
  uint64_t h[16];
  f.read(h, sizeof h);
  if (h[0] != IX_MAGIC || (h[1] != 2 && h[1] != 3)) fail(BANI_ERR_ARG, "%s is not a fastani_b200 index file (version 2 or 3)", path);
  x.version = (int)h[1]; x.k = (int)h[2]; x.w = (int)h[3]; x.fragLen = (int)h[4];
  const uint64_t M = h[5], nC = h[6], nG = h[7];
  x.M = M; x.nContigs = nC; x.nGenomes = nG; x.validWords = h[8];
  if (M > 0xfffffff0ull || nC > 0x7ffffff0ull || nG > nC + 1 || nG > 0x7ffffff0ull || x.validWords > (1ull << 40))
    fail(BANI_ERR_ARG, "%s: corrupt header", path);
  {   // the sizes in the header must match the file before anything is allocated
    if (fseeko(f.f, 0, SEEK_END) != 0) fail(BANI_ERR_ARG, "%s: cannot seek", path);
    const uint64_t fileBytes = (uint64_t)ftello(f.f);
    f.seek(sizeof h);
    if (fileBytes != x.file_bytes())
      fail(BANI_ERR_ARG, "%s: %llu bytes, header says %llu (truncated or corrupt)", path, (unsigned long long)fileBytes, (unsigned long long)x.file_bytes());
  }
  x.contigLen.resize(nC); x.seqsByFile.resize(nG); x.recOff.resize(nC + 1);
  f.read(x.contigLen.data(), 4 * nC);
  f.read(x.seqsByFile.data(), 4 * nG);
  f.read(x.recOff.data(), 4 * (nC + 1));
  if (x.version >= 3) {
    uint64_t tableSum = 0;
    const uint64_t pos = (uint64_t)ftello(f.f);
    f.seek(x.off_sums());
    if (fread(&tableSum, 1, 8, f.f) != 8) fail(BANI_ERR_ARG, "%s is truncated", path);
    f.seek(pos);
    if (tableSum != f.sum) fail(BANI_ERR_ARG, "%s: table checksum mismatch (header or contig tables corrupt)", path);
  }
  int32_t prev = 0;
  for (uint64_t g = 0; g < nG; g++) {
    const int32_t e = x.seqsByFile[g];
    if (e < prev || (uint64_t)e > nC) fail(BANI_ERR_ARG, "%s: corrupt genome table", path);
    prev = e;
  }
  if ((uint64_t)prev != nC) fail(BANI_ERR_ARG, "%s: corrupt genome table (it ends at contig %d of %llu)", path, prev, (unsigned long long)nC);
  x.bitOff.assign(nC + 1, 0);
  for (uint64_t c = 0; c < nC; c++) {
    if (x.contigLen[c] < 0) fail(BANI_ERR_ARG, "%s: corrupt contig table", path);
    x.bitOff[c + 1] = x.bitOff[c] + (((uint64_t)x.contigLen[c] + 31) & ~31ull);
  }
  for (uint64_t c = 0; c < nC; c++) if (x.recOff[c] > x.recOff[c + 1]) fail(BANI_ERR_ARG, "%s: corrupt record offsets", path);
  if (x.recOff[0] != 0 || x.recOff[nC] != M) fail(BANI_ERR_ARG, "%s: corrupt record offsets", path);
  if (M ? x.validWords != x.bitOff[nC] / 32 + 1 : x.validWords != 0)
    fail(BANI_ERR_ARG, "%s: validity bitmap size does not match the contig table", path);
  return x;
}

IndexFileInfo index_file_info(const char *path)
{
  File f(path, "rb");
  return index_file_tables(f);
}

static void check_file_params(const Ctx *ctx, const IndexFileInfo &x, const char *path)
{
  const int k = ctx->prm.kmer_size, w = ctx->prm.window_size, fragLen = ctx->prm.frag_len;
  if (x.k != k || x.w != w || x.fragLen != fragLen)
    fail(BANI_ERR_ARG, "%s was built with other parameters (k %d w %d fragLen %d), this context has k %d w %d fragLen %d",
         path, x.k, x.w, x.fragLen, k, w, fragLen);
}

namespace {
// Writes a version-3 file: the header and tables on construction, then the three sections -- hash, wpos, validity bitmap --
// in order, each given in one or more pieces (device arrays, host words, zeros), then the sums (finish).  Every word of a
// section is added to the sum of the genome it belongs to on the way (words past the last genome, the trailing bitmap word,
// count for none) and to the checksum.  A writer destroyed before finish() removes its partial file.  The one place that
// knows the layout beyond the header: index_save and index_file_extend both write through it.
class IndexWriter {
 public:
  static constexpr size_t CHW = (size_t)16 << 20;          // words per piece of the pinned staging buffer
  IndexWriter(Ctx *ctx, const char *path, int k, int w, int fragLen, const std::vector<int32_t> &contigLen,
              const std::vector<int32_t> &seqsByFile, const std::vector<uint32_t> &recOff, uint64_t validWords)
    : st_(ctx->stream), f_(path, "wb")
  {
    try { begin(k, w, fragLen, contigLen, seqsByFile, recOff, validWords); }
    catch (...) { discard(); throw; }
  }
  ~IndexWriter() { if (stage_) cudaFreeHost(stage_); if (!done_) discard(); }
  IndexWriter(const IndexWriter &) = delete; IndexWriter &operator=(const IndexWriter &) = delete;
  // the pinned buffer, free between calls: a caller may read host words into it and hand them to host()
  uint32_t *buffer() { return stage_; }
  void next_section()
  {
    if (sec_ >= 2 || at_ != want_[sec_]) fail(BANI_ERR_INTERNAL, "%s: index section %d written incompletely", f_.path.c_str(), sec_);
    sec_++; at_ = 0; g_ = 0;
  }
  void host(const uint32_t *p, uint64_t n)
  {
    f_.put(p, 4 * n);
    // one pass over the words: each range goes to its genome's sum and to the checksum
    const std::vector<uint64_t> &ends = sec_ < 2 ? recEnd_ : bitEnd_;
    for (uint64_t i = 0; i < n;) {
      while (g_ < ends.size() && ends[g_] <= at_ + i) g_++;
      const uint64_t e = g_ == ends.size() ? n : std::min<uint64_t>(n, ends[g_] - at_);
      const uint64_t s = word_sum(p + i, 4 * (e - i));
      if (g_ < ends.size()) genomeSum_[g_] += s;
      f_.sum += s;
      i = e;
    }
    at_ += n;
  }
  void device(const void *dp, uint64_t n)
  {
    for (uint64_t o = 0; o < n; o += CHW) {
      const uint64_t m = std::min<uint64_t>(CHW, n - o);
      BANI_CUDA(cudaMemcpyAsync(stage_, (const uint32_t *)dp + o, 4 * m, cudaMemcpyDeviceToHost, st_));
      BANI_CUDA(cudaStreamSynchronize(st_));
      host(stage_, m);
    }
  }
  void zeros(uint64_t n)
  {
    memset(stage_, 0, 4 * std::min<uint64_t>(CHW, n));
    for (uint64_t o = 0; o < n; o += CHW) host(stage_, std::min<uint64_t>(CHW, n - o));
  }
  const std::vector<uint64_t> &genome_sums() const { return genomeSum_; }
  void finish()
  {
    if (sec_ != 2 || at_ != want_[2]) fail(BANI_ERR_INTERNAL, "%s: index section %d written incompletely", f_.path.c_str(), sec_);
    f_.write(&tableSum_, 8);
    f_.write(genomeSum_.data(), 8 * genomeSum_.size());
    const uint64_t sum = f_.sum;
    f_.write(&sum, 8);
    if (fflush(f_.f) != 0) fail(BANI_ERR_INTERNAL, "write error on %s", f_.path.c_str());
    done_ = true;
  }
 private:
  void begin(int k, int w, int fragLen, const std::vector<int32_t> &contigLen, const std::vector<int32_t> &seqsByFile,
             const std::vector<uint32_t> &recOff, uint64_t validWords)
  {
    const uint64_t nC = contigLen.size(), nG = seqsByFile.size(), M = recOff[nC];
    const uint64_t h[16] = {IX_MAGIC, 3, (uint64_t)k, (uint64_t)w, (uint64_t)fragLen, M, nC, nG, validWords};
    f_.write(h, sizeof h);
    f_.write(contigLen.data(), 4 * nC);
    f_.write(seqsByFile.data(), 4 * nG);
    f_.write(recOff.data(), 4 * (nC + 1));
    tableSum_ = f_.sum;
    // where every genome's records and bitmap words end (in 32-bit words of the hash / wpos and bitmap sections)
    recEnd_.resize(nG); bitEnd_.resize(nG);
    uint64_t bits = 0;
    for (uint64_t g = 0, c = 0; g < nG; g++) {
      for (; c < (uint64_t)seqsByFile[g]; c++) bits += ((uint64_t)contigLen[c] + 31) & ~31ull;
      recEnd_[g] = recOff[seqsByFile[g]];
      bitEnd_[g] = bits / 32;
    }
    want_[0] = want_[1] = M; want_[2] = validWords;
    genomeSum_.assign(nG, 0);
    BANI_CUDA(cudaHostAlloc(&stage_, 4 * CHW, cudaHostAllocDefault));
  }
  void discard()
  {
    if (f_.f) { fclose(f_.f); f_.f = nullptr; }
    remove(f_.path.c_str());
  }
  cudaStream_t st_; File f_;
  uint32_t *stage_ = nullptr;
  uint64_t tableSum_ = 0, want_[3] = {0, 0, 0}, at_ = 0;
  int sec_ = 0; size_t g_ = 0; bool done_ = false;
  std::vector<uint64_t> recEnd_, bitEnd_, genomeSum_;
};
}

void index_save(Ctx *ctx, const Index *ix, const char *path)
{
  cudaStream_t st = ctx->stream;
  if (ix->device != ctx->device) fail(BANI_ERR_ARG, "index lives on another device");
  const uint64_t M = ix->M, nC = (uint64_t)ix->nContigs;
  std::vector<uint32_t> recOff(nC + 1);
  BANI_CUDA(cudaMemcpyAsync(recOff.data(), ix->contigRecOff.p, 4 * (nC + 1), cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  const uint64_t validWords = M ? ix->validBits.n : 0;
  IndexWriter wr(ctx, path, ix->k, ix->w, ix->fragLen, ix->contigLen, ix->seqsByFile, recOff, validWords);
  wr.device(ix->hash.p, M);
  wr.next_section(); wr.device(ix->wpos.p, M);
  wr.next_section(); wr.device(ix->validBits.p, validWords);
  wr.finish();
}

// rebuilds the hash-ordered side of an index whose position-ordered side was read from a file
static void index_finish_loaded(Ctx *ctx, Index *ix)
{
  if (ix->M == 0) { index_make_empty(ctx, ix); return; }
  ix->seqId.alloc(ix->M, ctx->stream);
  seqid_fill_kernel<<<(unsigned)ix->nContigs, 128, 0, ctx->stream>>>(ix->contigRecOff.p, ix->nContigs, ix->seqId.p);
  ctx->launches++;
  index_finish(ctx, ix);
}

Index *index_load(Ctx *ctx, const char *path)
{
  cudaStream_t st = ctx->stream;
  File f(path, "rb");
  const IndexFileInfo x = index_file_tables(f);
  check_file_params(ctx, x, path);
  const uint64_t M = x.M, nC = x.contigLen.size(), nG = x.seqsByFile.size();
  auto ix = std::make_unique<Index>();
  ix->device = ctx->device; ix->k = x.k; ix->w = x.w; ix->fragLen = x.fragLen; ix->nGenomes = (int32_t)nG;
  ix->contigLen = x.contigLen; ix->seqsByFile = x.seqsByFile;
  std::vector<int32_t> contigGenome(nC);
  for (uint64_t g = 0, c = 0; g < nG; g++) for (; c < (uint64_t)x.seqsByFile[g]; c++) contigGenome[c] = (int32_t)g;
  index_contig_tables(ctx, ix.get(), contigGenome);
  BANI_CUDA(cudaMemcpyAsync(ix->contigRecOff.p, x.recOff.data(), 4 * (nC + 1), cudaMemcpyHostToDevice, st));
  ix->M = M;
  {
    Upload up(ctx, f);
    if (M) {
      ix->hash.alloc(M, st); ix->wpos.alloc(M, st);
      ix->validBits.alloc(x.validWords, st);
      up.copy(ix->hash.p, 4 * M); up.copy(ix->wpos.p, 4 * M); up.copy(ix->validBits.p, 4 * x.validWords);
    }
    up.finish();
  }
  if (x.version >= 3) { std::vector<uint64_t> sums(1 + nG); f.read(sums.data(), 8 * sums.size()); }
  const uint64_t sum = f.sum;
  uint64_t got = 0;
  if (fread(&got, 1, 8, f.f) != 8 || got != sum) fail(BANI_ERR_ARG, "%s: checksum mismatch", path);
  index_finish_loaded(ctx, ix.get());
  return ix.release();
}

// Genomes `gs` (ascending, distinct) of a version-3 file as the position-ordered side of one index, as index_build would
// have made it from exactly those genomes: contig tables, contigRecOff rebased to the genomes' records, hash, wpos and the
// validity bitmap.  Every slice read is checked against its genome's sum before the index is returned.
static std::unique_ptr<Index> index_read_genomes(Ctx *ctx, File &f, const IndexFileInfo &x, const std::vector<int32_t> &gs)
{
  cudaStream_t st = ctx->stream;
  const char *path = f.path.c_str();
  const uint64_t nG = x.seqsByFile.size();
  auto ix = std::make_unique<Index>();
  ix->device = ctx->device; ix->k = x.k; ix->w = x.w; ix->fragLen = x.fragLen; ix->nGenomes = (int32_t)gs.size();
  std::vector<int32_t> contigGenome;
  std::vector<uint32_t> recOff(1, 0);
  for (size_t i = 0; i < gs.size(); i++) {
    const int32_t g = gs[i];
    const uint64_t c0 = x.contig_begin(g), c1 = x.seqsByFile[g], base = recOff.back();
    for (uint64_t c = c0; c < c1; c++) {
      ix->contigLen.push_back(x.contigLen[c]);
      contigGenome.push_back((int32_t)i);
      recOff.push_back((uint32_t)(base + x.recOff[c + 1] - x.recOff[c0]));
    }
    ix->seqsByFile.push_back((int32_t)ix->contigLen.size());
  }
  const uint64_t M = recOff.back(), nC = ix->contigLen.size();
  const unsigned long long totalBits = index_contig_tables(ctx, ix.get(), contigGenome);
  BANI_CUDA(cudaMemcpyAsync(ix->contigRecOff.p, recOff.data(), 4 * (nC + 1), cudaMemcpyHostToDevice, st));
  ix->M = M;
  std::vector<uint64_t> want(nG);
  f.seek(x.off_sums() + 8);
  f.read(want.data(), 8 * nG);
  if (M) {
    ix->hash.alloc(M, st); ix->wpos.alloc(M, st);
    ix->validBits.alloc((size_t)(totalBits / 32) + 1, st);
    BANI_CUDA(cudaMemsetAsync(ix->validBits.p, 0, ix->validBits.bytes(), st));
    std::vector<uint64_t> got(gs.size(), 0);
    Upload up(ctx, f);
    uint64_t r = 0, b = 0;
    for (size_t i = 0; i < gs.size(); i++) {
      const int32_t g = gs[i];
      const uint64_t r0 = x.recOff[x.contig_begin(g)], n = x.recOff[x.seqsByFile[g]] - r0;
      f.seek(x.off_hash() + 4 * r0); up.copy(ix->hash.p + r, 4 * n, &got[i]);
      f.seek(x.off_wpos() + 4 * r0); up.copy(ix->wpos.p + r, 4 * n, &got[i]);
      const uint64_t w0 = x.bitOff[x.contig_begin(g)] / 32, nw = x.bitOff[x.seqsByFile[g]] / 32 - w0;
      f.seek(x.off_bits() + 4 * w0); up.copy(ix->validBits.p + b, 4 * nw, &got[i]);
      r += n; b += nw;
    }
    up.finish();
    for (size_t i = 0; i < gs.size(); i++)
      if (got[i] != want[gs[i]]) fail(BANI_ERR_ARG, "%s: checksum mismatch in genome %d", path, gs[i]);
    if (gs.back() == (int32_t)nG - 1) {            // the trailing bitmap word belongs to no genome: it must be zero
      uint32_t last = 1;
      f.seek(x.off_bits() + 4 * (x.validWords - 1));
      f.read(&last, 4);
      if (last != 0) fail(BANI_ERR_ARG, "%s: corrupt validity bitmap (the word past the last contig is not zero)", path);
    }
  }
  return ix;
}

static void require_ranges(const IndexFileInfo &x, const char *path)
{
  if (x.version < 3)
    fail(BANI_ERR_ARG, "%s was saved in version 2, which has no per-genome checksums: load it whole, or save it again to load "
         "it in ranges", path);
}

Index *index_load_budget(Ctx *ctx, const char *path, int32_t first, uint64_t maxBytes, int32_t *nTaken, uint64_t *peakBytes)
{
  if (maxBytes == 0) fail(BANI_ERR_ARG, "the index budget must be positive");
  File f(path, "rb");
  const IndexFileInfo x = index_file_tables(f);
  check_file_params(ctx, x, path);
  require_ranges(x, path);
  const int32_t nG = (int32_t)x.seqsByFile.size();
  if (first < 0 || first >= nG) fail(BANI_ERR_ARG, "genome %d outside %s (%d genomes)", first, path, nG);
  // the longest run [first, first + t) whose load fits: the footprint of an index build without sketch staging
  int32_t t = 0;
  const uint64_t c0 = x.contig_begin(first);
  auto need = [&](int32_t e) {
    const uint64_t c1 = x.seqsByFile[e - 1], m = x.recOff[c1] - x.recOff[c0];
    return index_footprint(m, m, c1 - c0, x.bitOff[c1] - x.bitOff[c0], 0).peak;
  };
  while (first + t < nG && need(first + t + 1) <= maxBytes) t++;
  if (t == 0)
    fail(BANI_ERR_LIMIT, "genome %d of %s (%llu minimizers) does not fit the index budget of %llu bytes: its index needs %llu", first, path,
         (unsigned long long)(x.recOff[x.seqsByFile[first]] - x.recOff[c0]), (unsigned long long)maxBytes, (unsigned long long)need(first + 1));
  *nTaken = t;
  std::vector<int32_t> gs(t);
  for (int32_t i = 0; i < t; i++) gs[i] = first + i;
  return with_peak(ctx, peakBytes, [&] {
    std::unique_ptr<Index> ix = index_read_genomes(ctx, f, x, gs);
    index_finish_loaded(ctx, ix.get());
    return ix.release();
  });
}

// Records are in (seqId, wpos) order and every contig's bits start on a word, so the index of "old genomes, then added
// genomes" has each section of the old file followed by the added index's: the tables are joined with the added offsets
// moved past the old ones, the old records and bitmap words are streamed from the file through the writer's buffer (each
// genome checked against its sum on the way), the added ones come from the device.  The bitmap of an added index without
// records is read too: contigs shorter than k + w - 1 have valid positions but no window.  Only an index of contigs that
// are all shorter than k has no bitmap at all; its words are zero, as the sketch launch of a fresh build leaves them.
void index_file_extend(Ctx *ctx, const char *inPath, const Index *add, const char *outPath)
{
  cudaStream_t st = ctx->stream;
  if (add->device != ctx->device) fail(BANI_ERR_ARG, "index lives on another device");
  {
    struct stat a, b;
    if (strcmp(inPath, outPath) == 0 || (stat(inPath, &a) == 0 && stat(outPath, &b) == 0 && a.st_dev == b.st_dev && a.st_ino == b.st_ino))
      fail(BANI_ERR_ARG, "%s is the file being extended: write the extended index to another path", outPath);
  }
  File f(inPath, "rb");
  const IndexFileInfo x = index_file_tables(f);
  check_file_params(ctx, x, inPath);
  if (add->k != x.k || add->w != x.w || add->fragLen != x.fragLen)
    fail(BANI_ERR_ARG, "the added index was built with other parameters (k %d w %d fragLen %d) than %s (k %d w %d fragLen %d)",
         add->k, add->w, add->fragLen, inPath, x.k, x.w, x.fragLen);
  if (x.version < 3)
    fail(BANI_ERR_ARG, "%s was saved in version 2, which has no per-genome checksums: save it again to add genomes to it", inPath);
  if (x.M == 0)
    fail(BANI_ERR_ARG, "%s holds no minimizers, so it saved no validity bitmap: build it again with the new genomes", inPath);
  const uint64_t nC0 = x.nContigs, M0 = x.M, nC1 = (uint64_t)add->nContigs, M1 = add->M;
  if (M0 + M1 > 0xfffffff0ull)
    fail(BANI_ERR_LIMIT, "%s (%llu minimizers) and the added genomes (%llu) exceed the 2^32 minimizers of one index file", inPath,
         (unsigned long long)M0, (unsigned long long)M1);
  if (nC0 + nC1 > 0x7ffffff0ull) fail(BANI_ERR_LIMIT, "%s and the added genomes exceed the 2^31 contigs of one index file", inPath);
  // the joined tables
  std::vector<int32_t> contigLen = x.contigLen, seqsByFile = x.seqsByFile;
  std::vector<uint32_t> recOff = x.recOff, addRecOff(nC1 + 1);
  BANI_CUDA(cudaMemcpyAsync(addRecOff.data(), add->contigRecOff.p, 4 * (nC1 + 1), cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  uint64_t addBits = 0;
  for (uint64_t c = 0; c < nC1; c++) {
    contigLen.push_back(add->contigLen[c]);
    recOff.push_back((uint32_t)(M0 + addRecOff[c + 1]));
    addBits += ((uint64_t)add->contigLen[c] + 31) & ~31ull;
  }
  for (int32_t e : add->seqsByFile) seqsByFile.push_back((int32_t)(nC0 + e));
  const uint64_t addWords = addBits / 32;
  if (add->validBits.n && add->validBits.n < addWords) fail(BANI_ERR_INTERNAL, "added index: validity bitmap shorter than its contigs");

  IndexWriter wr(ctx, outPath, x.k, x.w, x.fragLen, contigLen, seqsByFile, recOff, (x.bitOff[nC0] + addBits) / 32 + 1);
  auto copy = [&](uint64_t words) {                    // old file -> new file through the writer's buffer
    for (uint64_t o = 0; o < words; o += IndexWriter::CHW) {
      const uint64_t n = std::min<uint64_t>(IndexWriter::CHW, words - o);
      f.get(wr.buffer(), 4 * n);                      // summed once, by the writer: see the checksum below
      wr.host(wr.buffer(), n);
    }
  };
  copy(M0); wr.device(add->hash.p, M1);
  wr.next_section(); copy(M0); wr.device(add->wpos.p, M1);
  wr.next_section(); copy(x.validWords - 1);
  uint32_t last = 1;
  f.read(&last, 4);
  if (last != 0) fail(BANI_ERR_ARG, "%s: corrupt validity bitmap (the word past the last contig is not zero)", inPath);
  if (add->validBits.n) wr.device(add->validBits.p, addWords); else wr.zeros(addWords);
  wr.zeros(1);
  std::vector<uint64_t> want(1 + x.nGenomes);                 // tableSum (checked by index_file_tables), genomeSum[]
  f.read(want.data(), 8 * want.size());
  for (uint64_t g = 0; g < x.nGenomes; g++) {
    if (wr.genome_sums()[g] != want[1 + g]) fail(BANI_ERR_ARG, "%s: checksum mismatch in genome %llu", inPath, (unsigned long long)g);
    f.sum += want[1 + g];             // every old record and bitmap word but the zero trailing word belongs to a genome
  }
  const uint64_t sum = f.sum;
  uint64_t got = 0;
  if (fread(&got, 1, 8, f.f) != 8 || got != sum) fail(BANI_ERR_ARG, "%s: checksum mismatch", inPath);
  wr.finish();
}

QSketch *qsketch_from_index_file(Ctx *ctx, const char *path, const int32_t *ordinals, int32_t nq, const int32_t *queryIds)
{
  File f(path, "rb");
  const IndexFileInfo x = index_file_tables(f);
  check_file_params(ctx, x, path);
  require_ranges(x, path);
  const int32_t nG = (int32_t)x.seqsByFile.size();
  for (int32_t i = 0; i < nq; i++)
    if (ordinals[i] < 0 || ordinals[i] >= nG) fail(BANI_ERR_ARG, "genome ordinal %d outside %s (%d genomes)", ordinals[i], path, nG);
  if (x.M == 0) fail(BANI_ERR_ARG, "%s holds no minimizers: query sketches cannot be derived from it", path);
  // only the genomes asked for are read, each once, in file order; the queries keep their order
  std::vector<int32_t> gs(ordinals, ordinals + nq);
  std::sort(gs.begin(), gs.end());
  gs.erase(std::unique(gs.begin(), gs.end()), gs.end());
  std::vector<int32_t> local(nq);
  for (int32_t i = 0; i < nq; i++) local[i] = (int32_t)(std::lower_bound(gs.begin(), gs.end(), ordinals[i]) - gs.begin());
  std::unique_ptr<Index> part = index_read_genomes(ctx, f, x, gs);
  return qsketch_from_records(ctx, part.get(), local.data(), nq, queryIds);
}

} // namespace bani
