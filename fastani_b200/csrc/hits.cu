// hits.cu -- HP2 stages D+E fused per query fragment: gather the index hits of a fragment, sort them by
// (seqId, wpos) and apply the L1 candidate-region rule, all inside one CTA.
//
// Replaces the hit loop and std::sort of Map::doL1Mapping / computeL1CandidateRegions
// (src/map/include/computeMap.hpp:283-299, :320) and the region scan + merge of :322-352.
//
// The record index of a minimizer is monotone in (seqId, wpos), so sorting a fragment's hits by record index
// is the sort of :320.  A fragment has a few hundred to a few thousand hits: they fit in shared memory, so the
// device-wide 64-bit sort of (fragment, record) keys and the three passes over it (flags, scan, write) collapse
// into one kernel that reads each hit once:
//   1  gather   the position lists of the fragment's s query hashes -> shared memory
//   2  sort     block-wide radix sort (own: 8-bit digits, warp-match stable ranking) on the significant bits of the record index
//   3  fetch    (seqId, wpos) of every sorted hit -> shared memory (neighbouring ranks = neighbouring records)
//   4  L1       hit i opens a raw region iff hit i+minHits-1 is on the same contig less than fragLen ahead
//               (:324-336); overlapping raw regions merge (:342-350), which is a LOCAL rule on sorted hits:
//               i is the head of a merged region unless i-1 qualifies and reaches i's start, the tail unless
//               i+1 qualifies and starts at or before i's position
//   5  emit     block scan of head flags -> candidate ordinals; {seqId, start, end} written to a staging
//               area addressed by the fragment's global hit offset (a fragment never has more regions than hits)
// Fragments are binned by hit count into 13 size classes (256 ... 8192 hits per CTA, frag_class_items); larger
// ones (many near-identical references) stay on the device-wide sort path in map.cu.
#include "common.cuh"

namespace bani {

__global__ void frag_classify_kernel(const uint32_t *segStart, const unsigned long long *hitOff, int32_t F,
                                     uint32_t *candCount, uint32_t *fragClass, uint32_t *classCount, uint32_t *classList, unsigned long long maxFast)
{
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const unsigned long long n = hitOff[segStart[f + 1]] - hitOff[segStart[f]];
  candCount[f] = 0;
  uint32_t cls = FRAG_NCLASS + 1;                      // no hits
  if (n > maxFast) cls = FRAG_NCLASS;                  // device-wide path
  else if (n > 0) { cls = 0; while (n > 256ull * (unsigned long long)frag_class_items(cls)) cls++; }
  fragClass[f] = cls;
  if (cls <= FRAG_NCLASS) { const uint32_t o = atomicAdd(&classCount[cls], 1u); if (cls < FRAG_NCLASS) classList[(size_t)cls * F + o] = (uint32_t)f; }
}

// Block-wide stable LSD radix sort of CAP = 256 * ITEMS 32-bit keys held in shared memory, DB bits per pass (8 for the
// classes up to 2048 hits, 10 for the larger ones: a 29-bit record index then takes 3 passes instead of 4).
// Warp w owns the keys [w * 32 * ITEMS, (w+1) * 32 * ITEMS) of the current order and ranks them round by round
// (32 consecutive keys per round): lanes with the same digit find each other with match.any, the lowest of them
// bumps the warp's digit counter once for the whole group, the others take their place from the lane order --
// which keeps equal digits in input order, the property LSD needs.  Then every thread turns the per-warp counts of
// its 2^DB / 256 consecutive digits into offsets (prefix over warps, block scan over digits) and the keys are scattered
// to the other buffer.  Returns the buffer that holds the sorted keys.
template <int ITEMS, int DB>
__device__ __forceinline__ uint32_t *block_radix_sort(uint32_t *in, uint32_t *out, uint16_t *hist /* [8][2^DB] */,
                                                       uint32_t *digitBase /* [2^DB] */, uint32_t *wsum /* [8] */, int keyBits)
{
  constexpr int ND = 1 << DB, DPT = ND / 256;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const uint32_t ltMask = (1u << lane) - 1u;
  for (int shift = 0; shift < keyBits; shift += DB) {
    for (int i = tid; i < 8 * ND / 2; i += 256) reinterpret_cast<uint32_t *>(hist)[i] = 0;
    __syncthreads();
    uint32_t key[ITEMS]; uint32_t lr[ITEMS];
    uint16_t *myHist = hist + w * ND;
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
      key[r] = in[w * 32 * ITEMS + r * 32 + lane];
      const uint32_t d = (key[r] >> shift) & (uint32_t)(ND - 1);
      const uint32_t m = __match_any_sync(0xffffffffu, d);
      const int leader = __ffs(m) - 1;
      uint32_t old = 0;
      if (lane == leader) { old = myHist[d]; myHist[d] = (uint16_t)(old + __popc(m)); }
      old = __shfl_sync(0xffffffffu, old, leader);
      lr[r] = old + __popc(m & ltMask);
      __syncwarp();                                   // the counter update must be visible to the next round's leaders
    }
    __syncthreads();
    {
      // thread = DPT consecutive digits: counts of the 8 warps -> exclusive prefix over warps; totals -> exclusive scan over digits
      uint32_t tot[DPT], sum = 0;
#pragma unroll
      for (int j = 0; j < DPT; j++) {
        const int d = tid * DPT + j;
        uint32_t acc = 0;
#pragma unroll
        for (int ww = 0; ww < 8; ww++) { const uint32_t c = hist[ww * ND + d]; hist[ww * ND + d] = (uint16_t)acc; acc += c; }
        tot[j] = acc; sum += acc;
      }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      if (lane == 31) wsum[w] = incl;
      __syncthreads();
      uint32_t base = incl - sum;
      for (int ww = 0; ww < w; ww++) base += wsum[ww];
#pragma unroll
      for (int j = 0; j < DPT; j++) { digitBase[tid * DPT + j] = base; base += tot[j]; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < ITEMS; r++) {
      const uint32_t d = (key[r] >> shift) & (uint32_t)(ND - 1);
      out[digitBase[d] + myHist[d] + lr[r]] = key[r];
    }
    __syncthreads();
    uint32_t *t = in; in = out; out = t;
  }
  return in;
}

// 10-bit digits save a pass (3 instead of 4 for a 29-bit record index) but quadruple the per-pass fixed cost (zeroing and
// scanning 8 per-warp histograms): measured break-even at ~8 keys per thread
template <int ITEMS> struct FragSortBits { static constexpr int DB = ITEMS >= 10 ? 10 : 8; };

template <int ITEMS>
__global__ void __launch_bounds__(256)
frag_l1_kernel(const FragL1Args a, const uint32_t *list, uint32_t count)
{
  constexpr int CAP = 256 * ITEMS;
  constexpr int DB = FragSortBits<ITEMS>::DB, ND = 1 << DB;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint32_t *bufA = reinterpret_cast<uint32_t *>(smem_raw);                  // CAP
  uint32_t *bufB = bufA + CAP;                                              // CAP
  uint16_t *hist = reinterpret_cast<uint16_t *>(bufB + CAP);                // 8 * ND
  uint32_t *digitBase = reinterpret_cast<uint32_t *>(hist + 8 * ND);        // ND
  uint32_t *wsum = digitBase + ND;                                          // 8
  if (blockIdx.x >= count) return;
  const int f = (int)list[blockIdx.x], tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t t0 = a.segStart[f];
  const int s = a.sCount[f];
  const unsigned long long base = a.hitOff[t0];
  const int n = (int)(a.hitOff[a.segStart[f + 1]] - base);

  // ---- 1: gather.  Lane per position list: a warp copies 32 lists side by side, element j of every list in step j (lists
  //         are short -- one entry per related reference that holds the minimizer -- so a warp is done after max(count)
  //         steps; the j-th and (j+1)-th element of a list share a sector, which stays in L1 between the steps)
  for (int q = tid; q < ((s + 31) & ~31); q += 256) {
    uint32_t lo = 0, cnt = 0, o = 0;
    if (q < s) { lo = a.hitLo[t0 + q]; cnt = a.hitCnt[t0 + q]; o = (uint32_t)(a.hitOff[t0 + q] - base); }
    uint32_t mx = cnt;
#pragma unroll
    for (int sh = 16; sh; sh >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, sh));
    for (uint32_t j = 0; j < mx; j++) if (j < cnt) bufA[o + j] = __ldg(&a.posIdx[lo + j]);
  }
  for (int i = n + tid; i < CAP; i += 256) bufA[i] = 0xFFFFFFFFu;
  __syncthreads();
  // ---- 2: sort by record index
  const uint32_t *sorted = block_radix_sort<ITEMS, DB>(bufA, bufB, hist, digitBase, wsum, a.keyBits);
  // ---- 3: (wpos, seqId) of the sorted hits, one 8-byte load each; rank r = i*256 + tid (neighbouring lanes = neighbouring records)
  uint32_t keys[ITEMS];
#pragma unroll
  for (int i = 0; i < ITEMS; i++) keys[i] = sorted[i * 256 + tid];
  __syncthreads();
  int32_t *s_w = reinterpret_cast<int32_t *>(bufA), *s_seq = reinterpret_cast<int32_t *>(bufB);
#pragma unroll
  for (int i = 0; i < ITEMS; i++) {
    const int r = i * 256 + tid;
    if (r < n) { const int2 p = __ldg(&a.recPos[keys[i]]); s_w[r] = p.x; s_seq[r] = p.y; }
  }
  __syncthreads();
  // ---- 4: L1 flags.  Item i of lane `lane` in warp `wid` is rank i*256 + wid*32 + lane: consecutive lanes read
  //         consecutive words (no bank conflicts).  Pass 1: does hit r open a raw region (:324-336)?  One evaluation per
  //         hit; a ballot packs the answers of 32 consecutive ranks into one word of qualW.  Pass 2: head / tail of the
  //         merged regions from the neighbours' answers (:342-350).
  const int mh = a.minHits[s];
  uint32_t *qualW = reinterpret_cast<uint32_t *>(hist);              // [ITEMS][8] words, rank r -> word r >> 5
  uint16_t *slice = reinterpret_cast<uint16_t *>(qualW + ITEMS * 8); // [ITEMS][8] head counts per 32 consecutive ranks
  int32_t starts[ITEMS];
  uint32_t qualMask = 0;
#pragma unroll
  for (int i = 0; i < ITEMS; i++) {
    const int r = i * 256 + tid, rb = r + mh - 1;
    bool q = false;
    starts[i] = 0;
    if (rb < n && s_seq[rb] == s_seq[r]) {
      const int32_t wb = s_w[rb];
      if (wb - s_w[r] < a.fragLen) { q = true; starts[i] = max(0, wb - a.fragLen + 1); }
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, q);
    if (lane == 0) qualW[i * 8 + wid] = bal;
    if (q) qualMask |= 1u << i;
  }
  __syncthreads();
  auto qual_at = [&](int r) -> bool { return (qualW[r >> 5] >> (r & 31)) & 1u; };
  auto start_at = [&](int r) -> int32_t { return max(0, s_w[r + mh - 1] - a.fragLen + 1); };
  uint32_t headMask = 0, tailMask = 0;           // bit i: item i of this thread
  uint32_t headBallot[ITEMS];                    // heads of the 32 ranks of this warp's slice of item i
#pragma unroll
  for (int i = 0; i < ITEMS; i++) {
    const int r = i * 256 + tid;
    bool hd = false;
    if ((qualMask >> i) & 1u) {
      const int32_t st = starts[i];
      const bool merged = r > 0 && s_seq[r - 1] == s_seq[r] && qual_at(r - 1) && s_w[r - 1] >= st;
      const bool nextMerges = r + 1 < n && s_seq[r + 1] == s_seq[r] && qual_at(r + 1) && s_w[r] >= start_at(r + 1);
      hd = !merged;
      if (hd) headMask |= 1u << i;
      if (!nextMerges) tailMask |= 1u << i;
    }
    headBallot[i] = __ballot_sync(0xffffffffu, hd);
    if (lane == 0) slice[i * 8 + wid] = (uint16_t)__popc(headBallot[i]);
  }
  __syncthreads();
  // ---- 5: ordinals = exclusive prefix over the (item, warp) slices in rank order + position inside the slice
  uint32_t total = 0;
  {
    // every thread scans the <= 256 slice counts it needs (ITEMS * 8 entries, broadcast reads)
    uint32_t run = 0;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
      uint32_t before = run;
#pragma unroll
      for (int ww = 0; ww < 8; ww++) { const uint32_t c = slice[i * 8 + ww]; if (ww < wid) before += c; run += c; }
      const uint32_t hb = headBallot[i];
      const uint32_t upto = before + __popc(hb & ((2u << lane) - 1u));     // heads at ranks <= mine
      const int r = i * 256 + tid;
      if ((headMask >> i) & 1u) { a.stSeq[base + upto - 1] = s_seq[r]; a.stStart[base + upto - 1] = starts[i]; }
      if ((tailMask >> i) & 1u) a.stEnd[base + upto - 1] = s_w[r];
    }
    total = run;
  }
  if (tid == 0) a.candCount[f] = total;
}

// Fragments with few hits (shards of a multi-GPU run see a few hundred hits per fragment): one WARP per fragment instead
// of a CTA -- no block barriers, a bitonic network on <= CAPW keys in a slice of shared memory instead of four radix
// passes with their per-pass histogram work.  Same five steps, same outputs as frag_l1_kernel.
template <int CAPW>
__global__ void __launch_bounds__(128)
frag_l1_warp_kernel(const FragL1Args a, const uint32_t *list, uint32_t count)
{
  __shared__ uint32_t sm[4][3 * CAPW];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t slot = blockIdx.x * 4 + wid;
  if (slot >= count) return;
  const int f = (int)list[slot];
  uint32_t *keys = sm[wid];
  int32_t *s_w = reinterpret_cast<int32_t *>(keys + CAPW), *s_seq = s_w + CAPW;
  const uint32_t t0 = a.segStart[f];
  const int s = a.sCount[f];
  const unsigned long long base = a.hitOff[t0];
  const int n = (int)(a.hitOff[a.segStart[f + 1]] - base);
  int n2 = 32; while (n2 < n) n2 <<= 1;
  // ---- 1: gather, lane per position list (lists are short: about one hit per query hash here)
  for (int q = lane; q < s; q += 32) {
    const uint32_t cnt = a.hitCnt[t0 + q];
    if (cnt) {
      const uint32_t lo = a.hitLo[t0 + q], o = (uint32_t)(a.hitOff[t0 + q] - base);
      for (uint32_t j = 0; j < cnt; j++) keys[o + j] = __ldg(&a.posIdx[lo + j]);
    }
  }
  for (int i = n + lane; i < n2; i += 32) keys[i] = 0xFFFFFFFFu;
  __syncwarp();
  // ---- 2: sort by record index (bitonic, warp-synchronous)
  for (int k2 = 2; k2 <= n2; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int t = lane; t < (n2 >> 1); t += 32) {
        const int i = 2 * t - (t & (j - 1)), p = i + j;
        const uint32_t x = keys[i], y = keys[p];
        const bool asc = (i & k2) == 0;
        if ((x > y) == asc) { keys[i] = y; keys[p] = x; }
      }
      __syncwarp();
    }
  // ---- 3: (wpos, seqId) of the sorted hits
  for (int r = lane; r < n; r += 32) { const int2 p = __ldg(&a.recPos[keys[r]]); s_w[r] = p.x; s_seq[r] = p.y; }
  __syncwarp();
  // ---- 4 + 5: region rule on 32 consecutive ranks at a time; a ballot of the raw-region flags of the NEXT 32 ranks is
  //             needed for the right neighbour of lane 31, so the flags of every block are computed one block ahead
  const int mh = a.minHits[s];
  auto qual = [&](int r) -> bool {
    const int rb = r + mh - 1;
    return r < n && rb < n && s_seq[rb] == s_seq[r] && s_w[rb] - s_w[r] < a.fragLen;
  };
  auto start_of = [&](int r) -> int32_t { return max(0, s_w[r + mh - 1] - a.fragLen + 1); };
  uint32_t run = 0;
  uint32_t qPrev = 0, qCur = __ballot_sync(0xffffffffu, qual(lane));
  for (int r0 = 0; r0 < n; r0 += 32) {
    const uint32_t qNext = __ballot_sync(0xffffffffu, qual(r0 + 32 + lane));
    const int r = r0 + lane;
    bool hd = false, tl = false;
    int32_t st = 0;
    if ((qCur >> lane) & 1u) {
      st = start_of(r);
      const bool qL = lane ? ((qCur >> (lane - 1)) & 1u) : ((qPrev >> 31) & 1u);
      const bool qR = lane < 31 ? ((qCur >> (lane + 1)) & 1u) : (qNext & 1u);
      const bool merged = r > 0 && qL && s_seq[r - 1] == s_seq[r] && s_w[r - 1] >= st;
      const bool nextMerges = r + 1 < n && qR && s_seq[r + 1] == s_seq[r] && s_w[r] >= start_of(r + 1);
      hd = !merged; tl = !nextMerges;
    }
    const uint32_t hb = __ballot_sync(0xffffffffu, hd);
    const uint32_t upto = run + __popc(hb & ((2u << lane) - 1u));           // heads at ranks <= mine
    if (hd) { a.stSeq[base + upto - 1] = s_seq[r]; a.stStart[base + upto - 1] = st; }
    if (tl) a.stEnd[base + upto - 1] = s_w[r];
    run += __popc(hb);
    qPrev = qCur; qCur = qNext;
  }
  if (lane == 0) a.candCount[f] = run;
}

template <int ITEMS>
static void launch_class(Ctx *ctx, const FragL1Args &a, const uint32_t *list, uint32_t count, cudaStream_t st)
{
  if (count == 0) return;
  constexpr int ND = 1 << FragSortBits<ITEMS>::DB;
  const size_t shm = sizeof(uint32_t) * 2 * 256 * ITEMS + 2 * 8 * ND + 4 * ND + 64;
  if (ctx->first_time((const void *)frag_l1_kernel<ITEMS>))
    BANI_CUDA(cudaFuncSetAttribute(frag_l1_kernel<ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
  frag_l1_kernel<ITEMS><<<count, 256, shm, st>>>(a, list, count);
}

void frag_classify(Ctx *ctx, const uint32_t *segStart, const unsigned long long *hitOff, int32_t F,
                   uint32_t *candCount, uint32_t *fragClass, uint32_t *classCount /* 8, zeroed here */, uint32_t *classList /* 4*F */,
                   unsigned long long maxFast)
{
  BANI_CUDA(cudaMemsetAsync(classCount, 0, (FRAG_NCLASS + 2) * sizeof(uint32_t), ctx->stream));
  frag_classify_kernel<<<nblk(F), 256, 0, ctx->stream>>>(segStart, hitOff, F, candCount, fragClass, classCount, classList, maxFast);
  ctx->launches++;
}

void frag_l1_fast(Ctx *ctx, const FragL1Args &a, const uint32_t *classList, const uint32_t *classCount)
{
  cudaStream_t st = ctx->stream;
  const size_t F = (size_t)a.F;
  // one instantiation per size class (frag_class_items): the sort works on 256 * ITEMS slots, so narrow classes
  // keep the padding of a fragment's hit list small
  // up to 512 hits: warp per fragment
  if (classCount[0]) frag_l1_warp_kernel<256><<<(classCount[0] + 3) / 4, 128, 0, st>>>(a, classList + 0 * F, classCount[0]);
  if (classCount[1]) frag_l1_warp_kernel<512><<<(classCount[1] + 3) / 4, 128, 0, st>>>(a, classList + 1 * F, classCount[1]);
  launch_class<3>(ctx, a, classList + 2 * F, classCount[2], st);
  launch_class<4>(ctx, a, classList + 3 * F, classCount[3], st);
  launch_class<5>(ctx, a, classList + 4 * F, classCount[4], st);
  launch_class<6>(ctx, a, classList + 5 * F, classCount[5], st);
  launch_class<7>(ctx, a, classList + 6 * F, classCount[6], st);
  launch_class<8>(ctx, a, classList + 7 * F, classCount[7], st);
  launch_class<10>(ctx, a, classList + 8 * F, classCount[8], st);
  launch_class<12>(ctx, a, classList + 9 * F, classCount[9], st);
  launch_class<16>(ctx, a, classList + 10 * F, classCount[10], st);
  launch_class<24>(ctx, a, classList + 11 * F, classCount[11], st);
  launch_class<32>(ctx, a, classList + 12 * F, classCount[12], st);
  for (int i = 0; i < FRAG_NCLASS; i++) if (classCount[i]) ctx->launches++;
  BANI_CUDA(cudaGetLastError());
}

// ---- candidates of the device-wide path -> the same staging area (candidate c of fragment f lands at
//      hitOff[segStart[f]] + its ordinal inside the fragment)
__global__ void cand_stage_kernel(const int32_t *cFrag, const int32_t *cSeq, const int32_t *cStart, const int32_t *cEnd, uint32_t C,
                                  const uint32_t *segStart, const unsigned long long *hitOff,
                                  int32_t *stSeq, int32_t *stStart, int32_t *stEnd, uint32_t *candCount)
{
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int f = cFrag[c];
  uint32_t lo = 0, hi = c;                       // first candidate of fragment f
  while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (cFrag[mid] < f) lo = mid + 1; else hi = mid; }
  const unsigned long long o = hitOff[segStart[f]] + (c - lo);
  stSeq[o] = cSeq[c]; stStart[o] = cStart[c]; stEnd[o] = cEnd[c];
  atomicAdd(&candCount[f], 1u);
}

void cand_stage(Ctx *ctx, const int32_t *cFrag, const int32_t *cSeq, const int32_t *cStart, const int32_t *cEnd, uint32_t C,
                const uint32_t *segStart, const unsigned long long *hitOff, int32_t *stSeq, int32_t *stStart, int32_t *stEnd,
                uint32_t *candCount)
{
  if (!C) return;
  cand_stage_kernel<<<nblk(C), 256, 0, ctx->stream>>>(cFrag, cSeq, cStart, cEnd, C, segStart, hitOff, stSeq, stStart, stEnd, candCount);
  ctx->launches++;
}

// ---- staging -> dense candidate arrays in (fragment, position) order; one warp per fragment
__global__ void cand_compact_kernel(const uint32_t *segStart, const unsigned long long *hitOff, int32_t F,
                                    const uint32_t *candCount, const uint32_t *candOff,
                                    const int32_t *stSeq, const int32_t *stStart, const int32_t *stEnd,
                                    int32_t *cFrag, int32_t *cSeq, int32_t *cStart, int32_t *cEnd)
{
  const int f = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (f >= F) return;
  const uint32_t n = candCount[f];
  if (!n) return;
  const unsigned long long src = hitOff[segStart[f]];
  const uint32_t dst = candOff[f];
  for (uint32_t i = lane; i < n; i += 32) {
    cFrag[dst + i] = f; cSeq[dst + i] = stSeq[src + i]; cStart[dst + i] = stStart[src + i]; cEnd[dst + i] = stEnd[src + i];
  }
}

void cand_compact(Ctx *ctx, const uint32_t *segStart, const unsigned long long *hitOff, int32_t F,
                  const uint32_t *candCount, const uint32_t *candOff, const int32_t *stSeq, const int32_t *stStart,
                  const int32_t *stEnd, int32_t *cFrag, int32_t *cSeq, int32_t *cStart, int32_t *cEnd)
{
  cand_compact_kernel<<<nblk((uint64_t)F * 32), 256, 0, ctx->stream>>>(segStart, hitOff, F, candCount, candOff, stSeq, stStart, stEnd,
                                                                         cFrag, cSeq, cStart, cEnd);
  ctx->launches++;
}

} // namespace bani
