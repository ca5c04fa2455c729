// budget.cpp -- device-memory footprint of an index build, the index budget of a mapping run, and the cut of a reference
// list into chunks whose indexes fit it.  Host arithmetic only (no device call), so that a plan can be made and checked
// without a GPU; the budgeted build (index.cu), the chunk planner and the context helper (capi.cu) all count with
// index_footprint and nothing else.
#include "common.cuh"
#include <algorithm>

namespace bani {

// What index_build holds at once (index.cu), every buffer rounded as the caching allocator rounds it:
//   sketch stage : contig tables + validity bitmap + contig descriptors + th/tw/ts staging (3 x 4 B x stagingCap) + the
//                  sketch launch's tile state, then the hash/wpos/seqId copies (3 x 4 B x M) while the staging is alive.  A
//                  budgeted build that keeps a prefix also holds a second bitmap and contig table for the cut.
//   finish stage : hash/wpos/seqId + link/posIdx + the four sort/scan arrays (sortedHash, iota, head, scan) + either the CUB
//                  temp storage or ukeys/uoff, the directory, the power-of-two probe table and filter, rec/pos8/rec8/blkMax.
// The contig descriptors are freed when the sketch launch is done.  The resident index is what stays after the build:
// everything of the finish stage but the four sort/scan arrays and the CUB temp storage.
IndexFootprint index_footprint(uint64_t M, uint64_t Ub, uint64_t nC, uint64_t bits, uint64_t stagingCap)
{
  auto R = [](uint64_t b) { return (uint64_t)dev_round_size((size_t)b); };
  Ub = std::min(Ub, M);
  const uint64_t tables = R(4 * (nC + 1)) + R(4 * std::max<uint64_t>(nC, 1)) + R(4 * (nC + 1)) + (nC ? R(8 * nC) : 0);
  const uint64_t bitmap = R(4 * (bits / 32 + 1));
  const uint64_t desc = R(sizeof(SeqDesc) * std::max<uint64_t>(nC, 1));
  const uint64_t rec4 = R(4 * M);
  // sketch launch: a tile covers >= 2048 positions (sketch.cu), so its 8-byte tile state is below 2 bytes per staged record
  const uint64_t sketchTemp = R(4 * (nC + 1)) + R(2 * stagingCap + 8 * nC + 16);
  const uint64_t sketchStage = 2 * tables + 2 * bitmap + desc + 3 * R(4 * stagingCap) + sketchTemp + 3 * rec4;
  // CUB: the radix sort keeps an alternate key and value array (8 B per record) plus its digit tables; the scan only tile states
  const uint64_t cubSort = R(8 * M + M / 4 + ((uint64_t)64 << 20));
  const uint64_t cubScan = R(M / 64 + ((uint64_t)1 << 20));
  const int fb = index_filt_bits(Ub);
  const uint64_t lookup = R(4 * Ub) + R(4 * (Ub + 1)) + R(4 * ((1ull << index_dir_bits(Ub)) + 1)) + R(32ull << index_tab_bits(Ub)) +
                          (fb ? R(4ull << (fb - 5)) : 0);
  const uint64_t l2 = R(16 * M) + R(8 * M) + R(8 * M) + R(4 * ((M + 1023) / 1024));
  const uint64_t base = tables + bitmap + 3 * rec4 + 2 * rec4;                     // + link, posIdx
  const uint64_t finishStage = base + 4 * rec4 + R(8) + std::max(std::max(cubSort, cubScan), lookup + l2);
  IndexFootprint f;
  f.peak = std::max(sketchStage, finishStage);
  f.resident = base + lookup + l2;
  return f;
}

// The mapping working set, from the caps that bound it (map.cu): a piece gathers at most maxHitsPerPiece index hits with
// 12 bytes of L1 staging each, a piece's L2 event streams take at most eventBytesPerPiece (0 = a quarter of the device),
// and the identity reduction's bin table at most 3 GiB.
uint64_t map_working_set(uint64_t deviceBytes, long long maxHitsPerPiece, long long eventBytesPerPiece)
{
  const uint64_t hits = 12ull * (uint64_t)std::max(1ll, maxHitsPerPiece);
  const uint64_t events = eventBytesPerPiece > 0 ? (uint64_t)eventBytesPerPiece : deviceBytes / 4;
  return hits + events + (3ull << 30);
}

// The working set a run can reach, each term clamped by its cap above.  A query hash meets a reference genome about once
// (a minimizer recurs in a genome only in repeats), so a piece gathers at most about queryHashes x nRefs hits; a query
// fragment has about one L2 candidate per reference genome, whose window events take 32-byte slots of 16 events, two per
// record of a 2 x fragLen span at 2 / (w + 1) records per base (64 fragLen / (w + 1) bytes, twice that for slack); the bin
// table holds 4 bytes per position bin of the references and query; per fragment about 128 bytes of L1 tables.  A run of a
// few genomes thus needs megabytes, not the tens of gigabytes the caps allow, and a run of config 3's size reaches the caps.
uint64_t map_working_set_run(uint64_t deviceBytes, long long maxHitsPerPiece, long long eventBytesPerPiece, uint64_t queryHashes,
                             uint64_t queryFragments, uint64_t nQueries, uint64_t refBases, uint64_t nRefs, int w, int fragLen)
{
  const double wd = (double)std::max(w, 1), fl = (double)std::max(fragLen, 21);
  const double hitCap = (double)std::max(1ll, maxHitsPerPiece);
  const double evCap = eventBytesPerPiece > 0 ? (double)eventBytesPerPiece : (double)(deviceBytes / 4);
  const double hits = std::min(hitCap, (double)queryHashes * (double)nRefs);
  const double events = std::min(evCap, (double)queryFragments * (double)nRefs * 128.0 * fl / (wd + 1.0));
  const double bins = (double)refBases / (fl - 20.0) + (double)nRefs;
  const double table = std::min((double)(3ull << 30), 4.0 * bins * (double)std::max<uint64_t>(nQueries, 1));
  const double frag = 128.0 * std::min((double)queryFragments, (double)(1 << 18));
  return (uint64_t)(12.0 * hits + events + table + frag);
}

// Expected index of `pos` hashed positions: 2 / (w + 1) minimizers per position (the density index_build sizes its staging
// for, with 1.5x slack), every hash distinct (the bound on U).
static IndexFootprint expected_footprint(uint64_t pos, uint64_t nC, uint64_t bits, int w)
{
  const uint64_t M = (uint64_t)(2.0 * (double)pos / (w + 1));
  return index_footprint(M, M, nC, bits, index_staging_cap(pos, w));
}

// The index budget: the build peak of the largest index (at the expected density) whose build fits in the free bytes left
// by the query sketches AND whose resident part leaves room for the mapping working set.  The build's temporaries are gone
// when mapping starts, so the two are not summed: max(build peak, resident + working set) <= free - query sketches.
uint64_t index_budget(uint64_t freeBytes, uint64_t qsketchBytes, uint64_t workingSet, int w)
{
  if (freeBytes <= qsketchBytes) return 0;
  const uint64_t avail = freeBytes - qsketchBytes;
  auto fits = [&](uint64_t pos) {
    const IndexFootprint f = expected_footprint(pos, pos / 100000 + 1, pos + 32 * (pos / 100000 + 1), w);
    return f.peak <= avail && f.resident + workingSet <= avail;
  };
  if (!fits(0)) return 0;
  uint64_t lo = 0, hi = 1ull << 46;                // fits(lo), positions of far more than any device holds
  while (hi - lo > 1) { const uint64_t m = lo + (hi - lo) / 2; if (fits(m)) lo = m; else hi = m; }
  return expected_footprint(lo, lo / 100000 + 1, lo + 32 * (lo / 100000 + 1), w).peak;
}

// Cuts genomes [0, n) into consecutive chunks: each chunk is the longest run whose expected build peak fits the budget and
// whose staging stays below 2^32 records.  Returns the number of chunks (ends[c] = one past the last genome of chunk c),
// or -(g + 1) if genome g alone does not fit.
int32_t plan_chunks(const uint64_t *len, const int32_t *nContigs, int32_t n, int k, int w, uint64_t budget, int32_t *ends)
{
  int32_t nc = 0, g = 0;
  while (g < n) {
    uint64_t pos = 0, cont = 0, bits = 0;
    int32_t e = g;
    while (e < n) {
      const uint64_t p2 = pos + (len[e] >= (uint64_t)k ? len[e] - (uint64_t)k + 1 : 0);
      const uint64_t c2 = cont + (uint64_t)std::max(nContigs[e], 0);
      const uint64_t b2 = bits + len[e] + 32ull * (uint64_t)std::max(nContigs[e], 1);
      if (expected_footprint(p2, c2, b2, w).peak > budget || index_staging_cap(p2, w) > 0xfffffff0ull) break;
      pos = p2; cont = c2; bits = b2; e++;
    }
    if (e == g) return -(g + 1);
    ends[nc++] = e;
    g = e;
  }
  return nc;
}

// Bytes of the query sketch of a genome (bani_qsketch_info's export_bytes), estimated before it is built: the unique
// minimizer hashes of every fragment (about 2 / (w + 1) per base, 4 bytes each) plus 20 bytes of tables per fragment.
uint64_t qsketch_bytes_estimate(uint64_t len, int w, int fragLen)
{
  const uint64_t frags = fragLen > 0 ? len / (uint64_t)fragLen + 1 : 1;
  return (uint64_t)(8.0 * (double)len / (w + 1)) + 20 * frags + 256;
}

// The plan of one GPU's run: reference chunks and query blocks.  Query sketches above the query budget are mapped in
// blocks, unless that budget is derived and the whole run fits one index with every sketch resident.  The index budget
// leaves room for the largest block's sketches and the working set that block can reach.  A derived budget that cannot
// hold a genome does not refuse the run: it is mapped on one index, as it would be if it fitted (returns 1).  With a
// forced budget such a genome is an error: returns -(g + 1).  Otherwise returns the number of chunks.
int32_t plan_run(const RunSize &r, const uint64_t *refLen, const int32_t *refContigs, int32_t nRefs, const uint64_t *queryLen,
                 const uint64_t *qsBytes, int32_t nQ, int32_t *chunkEnd, int32_t *blockEnd, int32_t *nBlocks, uint64_t *indexBudget)
{
  const int w = r.w;
  if (nRefs == 0) {                                               // nothing to index: the run's one (empty) index
    if (nQ) blockEnd[0] = nQ;
    *nBlocks = nQ ? 1 : 0;
    *indexBudget = r.indexBudget;
    return 0;
  }
  uint64_t refBases = 0;
  for (int32_t g = 0; g < nRefs; g++) refBases += refLen[g];
  auto qbytes = [&](int32_t q) { return qsBytes ? qsBytes[q] : qsketch_bytes_estimate(queryLen[q], w, r.fragLen); };
  // index budget for queries [a, b) resident
  auto budgetFor = [&](int32_t a, int32_t b) {
    if (r.indexBudget) return r.indexBudget;
    uint64_t bytes = 0, len = 0, frags = 0;
    for (int32_t q = a; q < b; q++) { bytes += qbytes(q); len += queryLen[q]; frags += queryLen[q] / (uint64_t)std::max(r.fragLen, 1) + 1; }
    const uint64_t hashes = (uint64_t)(2.0 * (double)len / (w + 1));
    const uint64_t ws = map_working_set_run(r.deviceBytes, r.maxHitsPerPiece, r.eventBytesPerPiece, hashes, frags, (uint64_t)(b - a), refBases,
                                            (uint64_t)nRefs, w, r.fragLen);
    return index_budget(r.freeBytes, bytes, ws, w);
  };
  auto oneIndex = [&]() {
    chunkEnd[0] = nRefs;
    if (nQ) blockEnd[0] = nQ;
    *nBlocks = nQ ? 1 : 0;
    *indexBudget = budgetFor(0, nQ);
    return 1;
  };
  uint64_t qTotal = 0;
  for (int32_t q = 0; q < nQ; q++) qTotal += qbytes(q);
  const uint64_t qb = r.queryBudget ? r.queryBudget : r.freeBytes / 4;
  if (!r.queryBudget) {                                           // derived: every sketch resident if the run fits one index
    const uint64_t ib = budgetFor(0, nQ);
    if (ib && plan_chunks(refLen, refContigs, nRefs, r.k, w, ib, chunkEnd) == 1) return oneIndex();
  }
  int32_t nb = 0;
  {
    uint64_t acc = 0;
    for (int32_t q = 0, a = 0; q < nQ; q++) {                   // block [a, q): at least one query each
      if (q > a && acc + qbytes(q) > qb) { blockEnd[nb++] = q; a = q; acc = 0; }
      acc += qbytes(q);
    }
    if (nQ) blockEnd[nb++] = nQ;
  }
  uint64_t ib = ~0ull;
  for (int32_t b = 0, a = 0; b < nb; a = blockEnd[b], b++) ib = std::min(ib, budgetFor(a, blockEnd[b]));
  if (nb == 0) ib = budgetFor(0, 0);
  *nBlocks = nb;
  *indexBudget = ib;
  const int32_t nc = plan_chunks(refLen, refContigs, nRefs, r.k, w, ib, chunkEnd);
  if (nc < 0 && !r.indexBudget) return oneIndex();
  return nc;
}

// "123", "64M", "2G" (binary units) -> bytes; false for anything else
bool parse_byte_count(const char *s, uint64_t *out)
{
  if (!s || !*s) return false;
  uint64_t v = 0;
  const char *p = s;
  for (; *p >= '0' && *p <= '9'; p++) { if (v > (~0ull - 9) / 10) return false; v = v * 10 + (uint64_t)(*p - '0'); }
  if (p == s) return false;
  int sh = 0;
  if (*p == 'K' || *p == 'k') sh = 10; else if (*p == 'M' || *p == 'm') sh = 20; else if (*p == 'G' || *p == 'g') sh = 30;
  if (sh) p++;
  if (*p) return false;
  if (sh && v > (~0ull >> sh)) return false;
  *out = v << sh;
  return true;
}

} // namespace bani
