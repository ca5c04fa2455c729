// cgi.cu -- HP2 stage H: the per-pair identity reduction of the mapping rows of a piece.
//
// Replaces cgi::computeCGI (src/cgi/include/computeCoreIdentity.hpp:166-298): 1-way best per (fragment, genome);
// 2-way best per (ref contig, position bin) via atomicMax on a dense bin table; ordered float32 sum per genome pair.
// Pieces whose dense (query, genome) output would dwarf their rows take a sparse path that sorts the rows instead.
#include "common.cuh"
#include <algorithm>

namespace bani {

struct CgiArgs {
  const bani_mapping *rows; const int32_t *rFrag; uint32_t R;
  const int32_t *fragQuery;            // chunk-local query slot of a fragment
  const int32_t *contigGenome; const uint32_t *contigBinOff;
  int fragLen; unsigned long long totalBins; int nGenomes;
  uint32_t *table;                     // [querySlot - qLo][totalBins] float bits, 0 = empty
  uint8_t *touched;                    // [querySlot - qLo][nGenomes]
  int qLo, qHi;                        // query slots of the piece handled by this pass
};

// 1-way: best row of each (fragment, genome) by (identity, refSeqId, refStartPos) (cgid_types.hpp:31-39,
// computeCoreIdentity.hpp:214-231): true if no other row of fragment f (row i, identity id) on genome g beats row i
__device__ __forceinline__ bool cgi_one_way_winner(const CgiArgs &a, uint32_t i, int f, int g, float id)
{
  // rows of a fragment are contiguous and ordered by (refSeqId, refStartPos): a later row wins ties
  for (uint32_t j = i + 1; j < a.R && a.rFrag[j] == f && a.contigGenome[a.rows[j].refSeqId] == g; j++)
    if (a.rows[j].nucIdentity >= id) return false;
  for (uint32_t j = i; j-- > 0 && a.rFrag[j] == f && a.contigGenome[a.rows[j].refSeqId] == g;)
    if (a.rows[j].nucIdentity > id) return false;
  return true;
}

__device__ __forceinline__ unsigned long long cgi_bin(const CgiArgs &a, const bani_mapping &r)
{
  return a.contigBinOff[r.refSeqId] + (uint32_t)(r.refStartPos / (a.fragLen - 20));
}

// 2-way: best identity per (ref contig, position bin) (:237-254)
__global__ void cgi_scatter_kernel(const CgiArgs a)
{
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.R) return;
  const int f = a.rFrag[i];
  const int q = a.fragQuery[f];
  if (q < a.qLo || q >= a.qHi) return;
  const bani_mapping r = a.rows[i];
  const int g = a.contigGenome[r.refSeqId];
  if (!cgi_one_way_winner(a, i, f, g, r.nucIdentity)) return;
  atomicMax(a.table + (unsigned long long)(q - a.qLo) * a.totalBins + cgi_bin(a, r), __float_as_uint(r.nucIdentity));
  a.touched[(size_t)(q - a.qLo) * a.nGenomes + g] = 1;
}

// Fragment-row mode of stage H (bani_map_cgi_sketch_frags): each bin holds the 64-bit key (identity bits << 32 | querySeqId)
// of its winner.  Every row of one table row and bin has the same query and genome, and positive floats order as their
// bits, so the 64-bit maximum is the best identity and, among equal identities, the largest querySeqId: the last element
// of computeCGI's stable sort over the 1-way list, which is ordered by (genome, querySeqId) (computeCoreIdentity.hpp:237-254).
struct CgiFragArgs {
  unsigned long long *table;           // [querySlot - qLo][totalBins] keys, 0 = empty
  uint8_t *win;                        // per row: 1-way winner of this pass
  unsigned long long *key; uint32_t *row; uint32_t *count;   // emitted 2-way winners: (query slot << 32 | global bin), row
};

__device__ __forceinline__ unsigned long long cgi_frag_key(const bani_mapping &r)
{
  return ((unsigned long long)__float_as_uint(r.nucIdentity) << 32) | (uint32_t)r.querySeqId;
}

__global__ void cgi_scatter_frag_kernel(const CgiArgs a, const CgiFragArgs f)
{
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.R) return;
  const int fr = a.rFrag[i];
  const int q = a.fragQuery[fr];
  const bani_mapping r = a.rows[i];
  const int g = a.contigGenome[r.refSeqId];
  const bool w = q >= a.qLo && q < a.qHi && cgi_one_way_winner(a, i, fr, g, r.nucIdentity);
  f.win[i] = w;
  if (!w) return;
  atomicMax(f.table + (unsigned long long)(q - a.qLo) * a.totalBins + cgi_bin(a, r), cgi_frag_key(r));
  a.touched[(size_t)(q - a.qLo) * a.nGenomes + g] = 1;
}

// the 1-way winners that hold their bin's key: one per non-empty bin, appended in any order (sorted afterwards)
__global__ void cgi_emit_kernel(const CgiArgs a, const CgiFragArgs f)
{
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.R || !f.win[i]) return;
  const bani_mapping r = a.rows[i];
  const int q = a.fragQuery[a.rFrag[i]];
  const unsigned long long bin = cgi_bin(a, r);
  if (f.table[(unsigned long long)(q - a.qLo) * a.totalBins + bin] != cgi_frag_key(r)) return;
  const uint32_t o = atomicAdd(f.count, 1u);
  f.key[o] = ((unsigned long long)q << 32) | bin;
  f.row[o] = i;
}

// sorted (query slot, bin) keys -> records; qryGenomeId holds the piece-local query slot until the host maps it
__global__ void cgi_frag_gather_kernel(const bani_mapping *rows, const unsigned long long *key, const uint32_t *row, uint32_t n,
                                       bani_frag_mapping *out)
{
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const bani_mapping r = rows[row[j]];
  bani_frag_mapping m;
  m.qryGenomeId = (int32_t)(key[j] >> 32); m.querySeqId = r.querySeqId; m.refSeqId = r.refSeqId; m.refStartPos = r.refStartPos;
  m.identity = r.nucIdentity;
  out[j] = m;
}

// ordered float32 sum over the bins of one (query, genome) pair (computeCoreIdentity.hpp:267-297);
// clears what it read so the table is all-zero again for the next chunk.  The identity is the high word of a 64-bit key.
template <typename T>
__device__ __forceinline__ void cgi_sum_pair(T *table, uint8_t *touched, const uint32_t *contigBinOff, const int32_t *genomeContigEnd,
                                             unsigned long long totalBins, int nGenomes, int nQ, int32_t *oCount, float *oIdent)
{
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (uint32_t)nQ * (uint32_t)nGenomes) return;
  const int q = i / nGenomes, g = i % nGenomes;
  int32_t cnt = 0; float sum = 0.0f;
  if (touched[i]) {
    touched[i] = 0;
    const uint32_t b0 = contigBinOff[g ? genomeContigEnd[g - 1] : 0], b1 = contigBinOff[genomeContigEnd[g]];
    T *row = table + (unsigned long long)q * totalBins;
    for (uint32_t b = b0; b < b1; b++) {
      const T v = row[b];
      if (v) { sum += __uint_as_float((uint32_t)(v >> (8 * sizeof(T) - 32))); cnt++; row[b] = 0; }
    }
  }
  oCount[i] = cnt; oIdent[i] = cnt ? sum / cnt : 0.0f;
}

__global__ void cgi_sum_kernel(uint32_t *table, uint8_t *touched, const uint32_t *contigBinOff, const int32_t *genomeContigEnd,
                               unsigned long long totalBins, int nGenomes, int nQ, int32_t *oCount, float *oIdent)
{
  cgi_sum_pair(table, touched, contigBinOff, genomeContigEnd, totalBins, nGenomes, nQ, oCount, oIdent);
}

__global__ void cgi_sum_frag_kernel(unsigned long long *table, uint8_t *touched, const uint32_t *contigBinOff, const int32_t *genomeContigEnd,
                                    unsigned long long totalBins, int nGenomes, int nQ, int32_t *oCount, float *oIdent)
{
  cgi_sum_pair(table, touched, contigBinOff, genomeContigEnd, totalBins, nGenomes, nQ, oCount, oIdent);
}

// Sparse stage H: the same reduction from the rows of a piece, with no table over (query, bin) or (query, genome).  Used
// for pieces whose dense output would dwarf their rows (many small genomes).  Every row gets a key: 1-way winners
// (query slot << binBits | global bin), the others the sentinel (nQ << binBits), which sorts after every real key.  So a
// radix sort over the significant bits of all R rows compacts the winners to the front without a host-side count.
__global__ void cgi_sparse_key_kernel(const CgiArgs a, int binBits, int nQ, unsigned long long *key, uint32_t *row)
{
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.R) return;
  const int f = a.rFrag[i];
  const int q = a.fragQuery[f];
  const bani_mapping r = a.rows[i];
  const int g = a.contigGenome[r.refSeqId];
  const bool w = cgi_one_way_winner(a, i, f, g, r.nucIdentity);
  key[i] = w ? ((unsigned long long)q << binBits) | cgi_bin(a, r) : (unsigned long long)nQ << binBits;
  row[i] = i;
}

// 1 where a run of equal winner keys -- one (query slot, bin) -- starts; n + 1 flags, the last 0 (exclusive scan -> count)
__global__ void cgi_sparse_bin_head_kernel(const unsigned long long *key, uint32_t n, unsigned long long sentinel, uint32_t *head)
{
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > n) return;
  head[j] = j < n && key[j] < sentinel && (j == 0 || key[j] != key[j - 1]);
}

// One thread per bin: its 2-way winner is the row with the largest 64-bit key (identity bits << 32 | querySeqId) -- what
// the dense path's atomicMax keeps; the pair is unique within a bin, so the winning row is deterministic.  Writes the bin
// as (query slot << 32 | global bin) with its row, and flags the bins that start a (query slot, genome) pair: bins of a
// genome are contiguous in the global bin order, so the pairs are runs of the sorted bins.
__global__ void cgi_sparse_bin_max_kernel(const CgiArgs a, const unsigned long long *key, const uint32_t *row, uint32_t n, int binBits,
                                          const uint32_t *head, const uint32_t *binIdx,
                                          unsigned long long *binKey, uint32_t *binRow, uint32_t *pairHead)
{
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || !head[j]) return;
  const unsigned long long k = key[j];
  uint32_t best = row[j];
  unsigned long long bestV = cgi_frag_key(a.rows[best]);
  for (uint32_t t = j + 1; t < n && key[t] == k; t++) {
    const unsigned long long v = cgi_frag_key(a.rows[row[t]]);
    if (v > bestV) { bestV = v; best = row[t]; }
  }
  const unsigned long long q = k >> binBits, bin = k & ((1ull << binBits) - 1);
  const uint32_t b = binIdx[j];
  binKey[b] = (q << 32) | bin;
  binRow[b] = best;
  const int g = a.contigGenome[a.rows[best].refSeqId];
  pairHead[b] = j == 0 || (key[j - 1] >> binBits) != q || a.contigGenome[a.rows[row[j - 1]].refSeqId] != g;
}

// One thread per (query slot, genome) pair: the float32 sum of its bin winners' identities in ascending bin order, divided
// by the count -- cgi_sum_pair's order and arithmetic, including its skipping of a bin whose value is 0.  Writes the pair
// as a bani_cgi_result with the query slot in qryGenomeId (the host maps it), in (query slot, genome) order.
__global__ void cgi_sparse_pair_kernel(const CgiArgs a, const unsigned long long *binKey, const uint32_t *binRow, const uint32_t *nBinsP,
                                       const uint32_t *pairHead, const uint32_t *pairIdx, bool fragKeys, bani_cgi_result *out)
{
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nBins = *nBinsP;
  if (b >= nBins || !pairHead[b]) return;
  int32_t cnt = 0; float sum = 0.0f;
  for (uint32_t t = b; t < nBins && (t == b || !pairHead[t]); t++) {
    const bani_mapping &r = a.rows[binRow[t]];
    const unsigned long long v = fragKeys ? cgi_frag_key(r) : (unsigned long long)__float_as_uint(r.nucIdentity);
    if (v) { sum += r.nucIdentity; cnt++; }
  }
  bani_cgi_result o;
  o.refGenomeId = a.contigGenome[a.rows[binRow[b]].refSeqId]; o.qryGenomeId = (int32_t)(binKey[b] >> 32);
  o.countSeq = cnt; o.totalQueryFragments = 0; o.identity = cnt ? sum / cnt : 0.0f;
  out[pairIdx[b]] = o;
}

// stage H takes the sparse path when a piece's dense (query, genome) output exceeds both its rows and this many entries
// (32 MB of count + identity): below it the dense tables cost less than the sparse path's sort (DESIGN.md section 6)
static constexpr uint64_t CGI_SPARSE_MIN_PAIRS = 1u << 22;

// ------------------------------------------------------------------ host
CgiState::CgiState(Ctx *ctx, const Index *ix_, bool frags_) : ix(ix_), frags(frags_)
{
  // the 2-way table holds a bounded number of queries at a time (4-byte bins, 8-byte keys in the fragment-row mode)
  qMax = 1u << 30;
  if (ix->totalBins) qMax = std::max<uint64_t>(1, ((uint64_t)3 << 30) / (bin_bytes() * ix->totalBins));
  if (ctx->flags.cgiTableQueries > 0) qMax = std::min<uint64_t>(qMax, (uint64_t)ctx->flags.cgiTableQueries);
  const int nG = ix->nGenomes;
  gce.alloc(std::max(nG, 1), ctx->stream);
  if (nG) BANI_CUDA(cudaMemcpyAsync(gce.p, ix->seqsByFile.data(), 4 * (size_t)nG, cudaMemcpyHostToDevice, ctx->stream));
}

// the fragment rows of n 2-way winners (sorted by query slot, global bin) to the host; the copy lands at the next synchronisation
static void frag_rows(Ctx *ctx, const bani_mapping *rows, const unsigned long long *key, const uint32_t *row, uint32_t n,
                      std::vector<bani_frag_mapping> &out)
{
  BANI_SCRATCH(bani_frag_mapping, dFrags, n);
  cgi_frag_gather_kernel<<<nblk(n), 256, 0, ctx->stream>>>(rows, key, row, n, dFrags.p);
  ctx->launches++;
  out.resize(n);
  BANI_CUDA(cudaMemcpyAsync(out.data(), dFrags.p, sizeof(bani_frag_mapping) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
}

static void cgi_sparse(Ctx *ctx, const CgiState &cs, const CgiArgs &ca, int nQ, uint64_t *pp, CgiResult &res)
{
  cudaStream_t st = ctx->stream;
  const uint32_t R = ca.R;
  int qBits = 0; while ((1ull << qBits) <= (uint64_t)nQ) qBits++;                 // slots 0 .. nQ (the sentinel)
  int binBits = 1; while ((1ull << binBits) < cs.ix->totalBins) binBits++;
  if (qBits + binBits > 64) fail(BANI_ERR_LIMIT, "sparse identity reduction: %d query bits + %d bin bits exceed 64", qBits, binBits);
  BANI_SCRATCH(unsigned long long, spKey, R);
  BANI_SCRATCH(unsigned long long, spKeySorted, R);
  BANI_SCRATCH(uint32_t, spRow, R);
  BANI_SCRATCH(uint32_t, spRowSorted, R);
  BANI_SCRATCH(uint32_t, binHead, (size_t)R + 1);
  BANI_SCRATCH(uint32_t, binIdx, (size_t)R + 1);
  BANI_SCRATCH(unsigned long long, binKey, R);
  BANI_SCRATCH(uint32_t, binRow, R);
  BANI_SCRATCH(uint32_t, pairHead, (size_t)R + 1);
  BANI_SCRATCH(uint32_t, pairIdx, (size_t)R + 1);
  BANI_SCRATCH(bani_cgi_result, dPairs, R);
  Stage sg(ctx, "cgi_sparse", 150.0 * R);
  pp[P_CGI_SPARSE]++;
  cgi_sparse_key_kernel<<<nblk(R), 256, 0, st>>>(ca, binBits, nQ, spKey.p, spRow.p);
  ctx->launches++;
  ctx->sort_pairs(spKey.p, spKeySorted.p, spRow.p, spRowSorted.p, R, qBits + binBits);
  cgi_sparse_bin_head_kernel<<<nblk((uint64_t)R + 1), 256, 0, st>>>(spKeySorted.p, R, (unsigned long long)nQ << binBits, binHead.p);
  ctx->launches++;
  ctx->scan(binHead.p, binIdx.p, (size_t)R + 1);
  BANI_CUDA(cudaMemsetAsync(pairHead.p, 0, 4 * ((size_t)R + 1), st));
  cgi_sparse_bin_max_kernel<<<nblk(R), 256, 0, st>>>(ca, spKeySorted.p, spRowSorted.p, R, binBits, binHead.p, binIdx.p,
                                                     binKey.p, binRow.p, pairHead.p);
  ctx->launches++;
  ctx->scan(pairHead.p, pairIdx.p, (size_t)R + 1);
  cgi_sparse_pair_kernel<<<nblk(R), 256, 0, st>>>(ca, binKey.p, binRow.p, binIdx.p + R, pairHead.p, pairIdx.p, cs.frags, dPairs.p);
  ctx->launches++;
  uint32_t nBins = 0, nPairs = 0;
  BANI_CUDA(cudaMemcpyAsync(&nBins, binIdx.p + R, 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaMemcpyAsync(&nPairs, pairIdx.p + R, 4, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  // the bin winners are already in (query slot, global bin) order: the fragment rows need no second sort
  if (cs.frags && nBins > 0) frag_rows(ctx, ca.rows, binKey.p, binRow.p, nBins, res.frags);
  res.pairs.resize(nPairs);
  if (nPairs) BANI_CUDA(cudaMemcpyAsync(res.pairs.data(), dPairs.p, sizeof(bani_cgi_result) * (size_t)nPairs, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  ctx->mark("piece: sparse identity rows on host");
}

// at most tableQ queries of the piece per pass over the rows
static void cgi_dense(Ctx *ctx, CgiState &cs, CgiArgs ca, int nQ, uint64_t *pp, CgiResult &res)
{
  cudaStream_t st = ctx->stream;
  const uint32_t R = ca.R; const int nG = cs.ix->nGenomes;
  const bool fm = cs.frags;
  res.count.assign((size_t)nQ * nG, 0); res.ident.assign((size_t)nQ * nG, 0.f);
  const uint64_t needQ = std::min<uint64_t>(cs.qMax, std::max<uint64_t>(nQ, 1));
  if (needQ > cs.tableQ) {
    cs.tableQ = needQ;
    cs.table.alloc((size_t)cs.tableQ * cs.ix->totalBins * cs.bin_bytes(), st);
    cs.touched.alloc((size_t)cs.tableQ * std::max(nG, 1), st);
    BANI_CUDA(cudaMemsetAsync(cs.table.p, 0, cs.table.bytes(), st));
    BANI_CUDA(cudaMemsetAsync(cs.touched.p, 0, cs.touched.bytes(), st));
  }
  uint32_t *table = (uint32_t *)cs.table.p; unsigned long long *table64 = (unsigned long long *)cs.table.p;
  ca.table = fm ? nullptr : table; ca.touched = cs.touched.p;
  BANI_SCRATCH(int32_t, oCount, (size_t)nQ * nG);
  DevBuf<float> oIdent((size_t)nQ * nG, st);
  // fragment-row mode: scatter 64-bit keys, emit each bin's winning row before the sum clears the bin, then
  // sort the piece's winners by (query slot, global bin) -- unique keys, so the order is deterministic
  CgiFragArgs fa{}; View<unsigned long long> emKeySorted; View<uint32_t> emRowSorted;
  if (fm) {
    BANI_SCRATCH(uint8_t, win, R);
    BANI_SCRATCH(unsigned long long, emKey, R);
    emKeySorted = ctx->view<unsigned long long>(BANI_SLOT_ID, R);
    BANI_SCRATCH(uint32_t, emRow, R);
    emRowSorted = ctx->view<uint32_t>(BANI_SLOT_ID, R);
    BANI_SCRATCH(uint32_t, emCount, 1);
    BANI_CUDA(cudaMemsetAsync(emCount.p, 0, 4, st));
    fa.table = table64; fa.win = win.p; fa.key = emKey.p; fa.row = emRow.p; fa.count = emCount.p;
  }
  {
    Stage sg(ctx, fm ? "cgi_frags" : "cgi", (fm ? 64.0 : 48.0) * R);
    for (int qa = 0; qa < nQ; qa += (int)cs.tableQ) {
      const int nPass = std::min<int>((int)cs.tableQ, nQ - qa);
      ca.qLo = qa; ca.qHi = qa + nPass;
      if (fm) cgi_scatter_frag_kernel<<<nblk(R), 256, 0, st>>>(ca, fa);
      else cgi_scatter_kernel<<<nblk(R), 256, 0, st>>>(ca);
      ctx->launches++; pp[P_CGI_PASSES]++;
      if (fm) { cgi_emit_kernel<<<nblk(R), 256, 0, st>>>(ca, fa); ctx->launches++; }
      int32_t *oc = oCount.p + (size_t)qa * nG; float *oi = oIdent.p + (size_t)qa * nG;
      if (fm) cgi_sum_frag_kernel<<<nblk((uint64_t)nPass * nG), 256, 0, st>>>(table64, cs.touched.p, ca.contigBinOff, cs.gce.p, ca.totalBins, nG, nPass, oc, oi);
      else cgi_sum_kernel<<<nblk((uint64_t)nPass * nG), 256, 0, st>>>(table, cs.touched.p, ca.contigBinOff, cs.gce.p, ca.totalBins, nG, nPass, oc, oi);
      ctx->launches++;
    }
    uint32_t nEm = 0;
    if (fm) {
      BANI_CUDA(cudaMemcpyAsync(&nEm, fa.count, 4, cudaMemcpyDeviceToHost, st));
      BANI_CUDA(cudaStreamSynchronize(st));
    }
    if (nEm > 0) {
      int qBits = 0; while ((1 << qBits) < nQ) qBits++;
      ctx->sort_pairs(fa.key, emKeySorted.p, fa.row, emRowSorted.p, nEm, 32 + qBits);
      frag_rows(ctx, ca.rows, emKeySorted.p, emRowSorted.p, nEm, res.frags);
    }
  }
  ctx->mark("piece: cgi launched");
  BANI_CUDA(cudaMemcpyAsync(res.count.data(), oCount.p, 4 * (size_t)nQ * nG, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaMemcpyAsync(res.ident.data(), oIdent.p, 4 * (size_t)nQ * nG, cudaMemcpyDeviceToHost, st));
  BANI_CUDA(cudaStreamSynchronize(st));
  ctx->mark("piece: identity tables on host");
}

void cgi_piece(Ctx *ctx, CgiState &cs, const bani_mapping *rows, const int32_t *rFrag, uint32_t R, const int32_t *fragQuery, int nQ,
               uint64_t *pp, CgiResult &res)
{
  CgiArgs ca; ca.rows = rows; ca.rFrag = rFrag; ca.R = R; ca.fragQuery = fragQuery;
  ca.contigGenome = cs.ix->contigGenome.p; ca.contigBinOff = cs.ix->contigBinOff.p; ca.fragLen = cs.ix->fragLen;
  ca.totalBins = cs.ix->totalBins; ca.nGenomes = cs.ix->nGenomes; ca.table = nullptr; ca.touched = nullptr; ca.qLo = 0; ca.qHi = nQ;
  // sparse when the dense (query, genome) output of the piece would exceed both its rows and 2^22 entries (many small
  // genomes; DESIGN.md section 6), unless the cgi_sparse switch forces a path
  const bool sparse = ctx->flags.cgiSparse >= 0 ? ctx->flags.cgiSparse == 1
                                                : (uint64_t)nQ * cs.ix->nGenomes > std::max<uint64_t>(R, CGI_SPARSE_MIN_PAIRS);
  if (sparse) cgi_sparse(ctx, cs, ca, nQ, pp, res);
  else cgi_dense(ctx, cs, ca, nQ, pp, res);
}

} // namespace bani
