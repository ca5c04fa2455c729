// ani_host.hpp -- C++ host side above the C ABI (include/fastani_b200.h), mirroring the reference's interface for
// the hot path and the host glue around it, so that a FastANI maintainer finds the same names:
//
//   skch::Parameters        src/map/include/map_parameters.hpp:22-41
//   skch::Sketch            src/map/include/winSketch.hpp:43-343      (constructor = HP1, on the GPU)
//   skch::Map               src/map/include/computeMap.hpp:35-560     (constructor = HP2, on the GPU)
//   cgi::computeCGI ...     src/cgi/include/computeCoreIdentity.hpp   (host restatement, kept for comparison behind
//                                                                      BANI_CLI_HOST_CGI=1; the CLI uses the fused device reduction)
//   cgi::outputCGI / outputPhylip / outputVisualizationFile / splitReferenceGenomes / correctRefGenomeIds
//
// Nothing here computes minimizers, hashes or identities on the CPU: Sketch and Map only hold handles of the
// library; without a GPU their constructors throw (the library has no CPU fallback).
#pragma once
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>
#include <system_error>
#include <thread>
#include <tuple>
#include <unordered_map>
#include <vector>
#include "../../include/fastani_b200.h"
#include "kseq_reader.hpp"

namespace skch {

typedef int32_t seqno_t;
typedef int32_t offset_t;
typedef bani_mapping MappingResult;                       // base_types.hpp:89-102, same layout
typedef std::vector<MappingResult> MappingResultsVector_t;

struct Parameters {                                       // map_parameters.hpp:22-41
  int kmerSize = 16, windowSize = 0, minReadLength = 3000;
  float minFraction = 0.2f;
  int threads = 1, alphabetSize = 4;
  uint64_t referenceSize = 5000000;
  float percentageIdentity = 80;
  double p_value = 1e-03;
  std::vector<std::string> refSequences, querySequences;
  std::string outFileName;
  bool reportAll = true, visualize = false, matrixOutput = false;
  float maxRatioDiff = 100.0f;
  bool sanityCheck = false;
  int gpus = 0;                                           // extension: devices to shard the references over (0 = all visible)
  bool blockPartition = false;                            // extension: --partition block (contiguous reference shards instead of the round-robin deal)
  std::string saveIndex, loadIndex;                       // extension: on-disk sketch cache (prefix of <prefix>.meta + <prefix>.<g>of<N>.idx)
  bani_params c() const
  {
    bani_params p; bani_params_default(&p);
    p.kmer_size = kmerSize; p.window_size = windowSize; p.frag_len = minReadLength;
    p.perc_identity = percentageIdentity; p.p_value = p_value; p.reference_size = referenceSize;
    return p;
  }
};

struct ContigInfo { std::string name; offset_t len; };    // base_types.hpp:72-76

inline void check(int rc, const char *what)
{
  if (rc != BANI_OK) throw std::runtime_error(std::string(what) + ": " + bani_last_error());
}

// A genome resident on one device.
struct DeviceGenome {
  bani_genome *h = nullptr;
  const bani_host::HostGenome *host = nullptr;
  ~DeviceGenome() { if (h) bani_genome_destroy(h); }
};

// 2-bit packing on the host, in the reader thread that parsed the file (bani_pack_contig needs no GPU): the ASCII bytes
// are released, a quarter of them (+ 5 bytes per non-ACGT byte) stay for the upload.
inline void pack_genome(bani_host::HostGenome &g)
{
  if (g.packed) return;
  int64_t words = 0;
  g.wordOff.clear(); g.excOff.assign(1, 0);
  for (const auto &c : g.contigs) { g.wordOff.push_back(words); words += (((int64_t)c.len + 15) / 16 + 3) / 4 * 4; }
  g.words.assign((size_t)words + 8, 0u);
  for (size_t i = 0; i < g.contigs.size(); i++) {
    const auto &c = g.contigs[i];
    if (c.len > 0x7fffffffull) throw std::runtime_error("contig " + c.name + " exceeds the int32 offset_t of the reference");
    const size_t e0 = g.excPos.size();
    uint64_t cap = std::max<uint64_t>(c.len / 64, 256), n = 0;
    for (;;) {
      g.excPos.resize(e0 + cap); g.excByte.resize(e0 + cap);
      check(bani_pack_contig(g.seq.data() + c.off, (int64_t)c.len, g.words.data() + g.wordOff[i], g.excPos.data() + e0, g.excByte.data() + e0, cap, &n), "bani_pack_contig");
      if (n <= cap) break;
      cap = n;
    }
    g.excPos.resize(e0 + n); g.excByte.resize(e0 + n);
    g.excOff.push_back((int64_t)(e0 + n));
  }
  std::vector<uint8_t>().swap(g.seq);
  g.packed = true;
}

// One upload batch on the host: the packed genomes [i, j) back to back in one array per kind, with the offset tables
// bani_genome_create_packed_batch takes.  The copies are made by `threads` threads into uninitialised storage (first touch
// of 1 GB of fresh pages by one thread costs more than parsing the files did).
struct HostBatch {
  std::unique_ptr<uint32_t[]> w; size_t words = 0;
  std::vector<uint32_t> ep; std::vector<uint8_t> eb;
  std::vector<int32_t> genOff, clen; std::vector<int64_t> woff, eoff;
};

inline HostBatch assemble_batch(const std::vector<const bani_host::HostGenome *> &gs, size_t i, size_t j, int threads)
{
  HostBatch b;
  std::vector<size_t> wAt, eAt;
  size_t wp = 0, epos = 0;
  b.genOff.assign(1, 0); b.eoff.assign(1, 0);
  for (size_t g = i; g < j; g++) {
    const auto &G = *gs[g];
    if (!G.packed) throw std::runtime_error("upload_genomes: genome " + G.path + " has not been packed");
    wAt.push_back(wp); eAt.push_back(epos);
    for (size_t c = 0; c < G.contigs.size(); c++) {
      b.clen.push_back((int32_t)G.contigs[c].len); b.woff.push_back((int64_t)wp + G.wordOff[c]); b.eoff.push_back((int64_t)epos + G.excOff[c + 1]);
    }
    wp += G.words.size(); epos += G.excPos.size();
    b.genOff.push_back((int32_t)b.clen.size());
  }
  b.clen.push_back(0); b.woff.push_back((int64_t)wp);
  b.words = wp;
  b.w.reset(new uint32_t[wp + 8]);
  memset(b.w.get() + wp, 0, 8 * sizeof(uint32_t));
  b.ep.resize(epos + 1); b.eb.resize(epos + 1);
  const size_t n = j - i;
  const int nt = (int)std::max<size_t>(1, std::min<size_t>((size_t)std::max(threads, 1), n));
  std::atomic<size_t> next(0);
  auto work = [&]() {
    for (size_t k; (k = next++) < n;) {
      const auto &G = *gs[i + k];
      if (!G.words.empty()) memcpy(b.w.get() + wAt[k], G.words.data(), 4 * G.words.size());
      if (!G.excPos.empty()) { memcpy(b.ep.data() + eAt[k], G.excPos.data(), 4 * G.excPos.size()); memcpy(b.eb.data() + eAt[k], G.excByte.data(), G.excByte.size()); }
    }
  };
  std::vector<std::thread> th;
  try { for (int t = 1; t < nt; t++) th.emplace_back(work); }
  catch (const std::system_error &) {}                            // no more threads to be had: the ones that exist do the work
  work();
  for (auto &t : th) t.join();
  return b;
}

// Uploads host-packed genomes (bani_genome_create_packed_batch): the genomes of a batch are laid out back to back in one
// host array per kind; the library copies them in groups on its copy stream.
inline void upload_genomes(bani_ctx *ctx, const std::vector<const bani_host::HostGenome *> &gs,
                           std::vector<std::unique_ptr<DeviceGenome>> &out, size_t batchWords = (size_t)1 << 28, int threads = 8)
{
  size_t i = 0;
  while (i < gs.size()) {
    size_t j = i, words = 0;
    while (j < gs.size() && (j == i || words + gs[j]->words.size() <= batchWords)) { words += gs[j]->words.size(); j++; }
    HostBatch b = assemble_batch(gs, i, j, threads);
    std::vector<bani_genome *> hs(j - i, nullptr);
    check(bani_genome_create_packed_batch(ctx, (int32_t)(j - i), b.genOff.data(), b.clen.data(), b.woff.data(), b.w.get(), b.eoff.data(), b.ep.data(), b.eb.data(),
                                          /*async=*/0, hs.data()), "bani_genome_create_packed_batch");
    for (size_t g = i; g < j; g++) { auto d = std::make_unique<DeviceGenome>(); d->h = hs[g - i]; d->host = gs[g]; out.push_back(std::move(d)); }
    i = j;
  }
}

// The tables of a saved index file (bani_index_file_info; no device): per genome its contig count, length and cumulative
// contig count, and every contig's length -- what a run plans its chunks and filters by --minFraction with
struct IndexFileTables {
  std::vector<int32_t> genomeContigs, seqsByFile, contigLen;
  std::vector<uint64_t> genomeLen;
};
inline IndexFileTables indexFileTables(const std::string &path)
{
  int32_t nG = 0; uint64_t nC = 0;
  check(bani_index_file_info(path.c_str(), nullptr, nullptr, nullptr, nullptr, &nG, &nC, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0),
        "bani_index_file_info");
  IndexFileTables t;
  t.genomeContigs.resize(std::max(nG, 1)); t.genomeLen.resize(std::max(nG, 1)); t.contigLen.resize(std::max<uint64_t>(nC, 1));
  check(bani_index_file_info(path.c_str(), nullptr, nullptr, nullptr, nullptr, &nG, &nC, nullptr, t.genomeContigs.data(), t.genomeLen.data(),
                             nullptr, nullptr, t.genomeContigs.size(), t.contigLen.data(), t.contigLen.size()), "bani_index_file_info");
  t.genomeContigs.resize(nG); t.genomeLen.resize(nG); t.contigLen.resize(nC);
  for (int32_t g = 0, c = 0; g < nG; g++) { c += t.genomeContigs[g]; t.seqsByFile.push_back(c); }
  return t;
}

// ---------------------------------------------------------------------------------------- Sketch (HP1)
class Sketch {
 public:
  std::vector<ContigInfo> metadata;                       // winSketch.hpp:70: every contig, also the too short ones
  std::vector<int> sequencesByFileInfo;                   // winSketch.hpp:75: cumulative contig count per genome
  Sketch(bani_ctx *ctx, const Parameters &p, const std::vector<const DeviceGenome *> &refs) : ctx_(ctx), param_(p)
  {
    std::vector<bani_genome *> hs;
    for (auto *g : refs) {
      hs.push_back(g->h);
      for (const auto &c : g->host->contigs) metadata.push_back(ContigInfo{c.name, (offset_t)c.len});
      sequencesByFileInfo.push_back((int)metadata.size());
    }
    check(bani_index_build(ctx, hs.data(), (int32_t)hs.size(), &ix_), "bani_index_build");
  }
  // From the on-disk sketch cache (bani_index_load): lengths and the genome table come from the file, contig names from
  // the caller's metadata (one per contig; may be empty when no --visualize output is wanted)
  Sketch(bani_ctx *ctx, const Parameters &p, const std::string &indexFile, const std::vector<std::string> &contigNames) : ctx_(ctx), param_(p)
  {
    check(bani_index_load(ctx, indexFile.c_str(), &ix_), "bani_index_load");
    uint64_t nMin = 0, nUniq = 0, totalLen = 0, nc = 0, ng = 0;
    check(bani_index_stats(ix_, &nMin, &nUniq, &totalLen, &nc, &ng), "bani_index_stats");
    std::vector<int32_t> cl(std::max<uint64_t>(nc, 1)), sbf(std::max<uint64_t>(ng, 1));
    check(bani_index_contigs(ix_, cl.data(), cl.size(), sbf.data(), sbf.size()), "bani_index_contigs");
    for (uint64_t c = 0; c < nc; c++) metadata.push_back(ContigInfo{c < contigNames.size() ? contigNames[c] : std::string(), (offset_t)cl[c]});
    for (uint64_t g = 0; g < ng; g++) sequencesByFileInfo.push_back((int)sbf[g]);
  }
  void save(const std::string &indexFile) const { check(bani_index_save(ctx_, ix_, indexFile.c_str()), "bani_index_save"); }
  ~Sketch() { if (ix_) bani_index_destroy(ix_); }
  Sketch(const Sketch &) = delete; Sketch &operator=(const Sketch &) = delete;
  const bani_index *handle() const { return ix_; }
  // winSketch.hpp:298-318
  bool sanityCheck(float maxRatioDiff)
  {
    if (!param_.sanityCheck) return true;
    return indexSanityCheck(ix_, maxRatioDiff, ratioDifference_);
  }
  // the same for any index (a chunk of a reference shard): ratioDifference is set
  static bool indexSanityCheck(const bani_index *ix, float maxRatioDiff, float &ratioDifference)
  {
    uint64_t nMin = 0, nUniq = 0, totalLen = 0, nc = 0, ng = 0;
    check(bani_index_stats(ix, &nMin, &nUniq, &totalLen, &nc, &ng), "bani_index_stats");
    const float hashRatio = float(totalLen) / float(nMin), uniqHashRatio = float(totalLen) / float(nUniq);
    ratioDifference = std::abs(hashRatio - uniqHashRatio);
    return !(ratioDifference > maxRatioDiff);
  }
  float getRatioDifference() const { return ratioDifference_; }
 private:
  bani_ctx *ctx_; Parameters param_; bani_index *ix_ = nullptr;
  float ratioDifference_ = 1.0f;          // the reference leaves it uninitialised; it prints `true`
};

// ---------------------------------------------------------------------------------------- Map (HP2)
// computeMap.hpp:138-167: the Map::metadata lengths of one query contig (entry i of a genome belongs to querySeqId i): a
// contig too short to map is one entry; any other gives len / fragLen fragments, the last one extended by len % fragLen
inline void appendFragmentLengths(const Parameters &p, offset_t len, std::vector<offset_t> &out)
{
  if (len < p.windowSize || len < p.kmerSize || len < p.minReadLength) { out.push_back(len); return; }
  const int fc = len / p.minReadLength;
  for (int i = 0; i < fc; i++) out.push_back(i != fc - 1 ? p.minReadLength : p.minReadLength + (len % p.minReadLength));
}

class Map {
 public:
  std::vector<ContigInfo> metadata;                       // computeMap.hpp:84: filled only with --visualize
  typedef std::function<void(const MappingResult &)> PostProcessResultsFn_t;
  // computeMap.hpp:93-102: maps one query genome, calls f once per reported mapping in (fragment, candidate) order
  Map(bani_ctx *ctx, const Parameters &p, const Sketch &refsketch, const DeviceGenome &query,
      uint64_t &totalQueryFragments, PostProcessResultsFn_t f = nullptr)
  {
    bani_mapping *rows = nullptr; uint64_t n = 0, tq = 0; bani_map_counters ctr;
    check(bani_map_genome(ctx, refsketch.handle(), query.h, &rows, &n, &tq, &ctr), "bani_map_genome");
    totalQueryFragments += tq;
    if (f) for (uint64_t i = 0; i < n; i++) f(rows[i]);
    bani_free(rows);
    if (p.visualize) {                                    // computeMap.hpp:138-167
      std::vector<offset_t> lens;
      for (const auto &c : query.host->contigs) {
        lens.clear();
        appendFragmentLengths(p, (offset_t)c.len, lens);
        for (offset_t l : lens) metadata.push_back(ContigInfo{c.name, l});
      }
    }
  }
  static void insertL2ResultsToVec(MappingResultsVector_t &v, const MappingResult &reportedL2Result) { v.push_back(reportedL2Result); }
};

} // namespace skch

namespace cgi {

struct MappingResult_CGI {                                // cgid_types.hpp:18-28
  skch::seqno_t refSequenceId, genomeId, querySeqId;
  skch::offset_t refStartPos, queryStartPos, mapRefPosBin;
  float nucIdentity;
};

struct CGI_Results {                                      // cgid_types.hpp:68-80
  skch::seqno_t refGenomeId, qryGenomeId, countSeq, totalQueryFragments;
  float identity;
};

// computeCoreIdentity.hpp:57-61: sum over contigs >= fragLen of floor(len / fragLen) * fragLen; computed from the
// contig table of the ingest pass instead of a second read of every file
inline uint64_t genomeLength(const bani_host::HostGenome &g, int fragLen)
{
  uint64_t s = 0;
  for (const auto &c : g.contigs) if ((int64_t)c.len >= fragLen) s += (c.len / (uint64_t)fragLen) * (uint64_t)fragLen;
  return s;
}

// the same from a contig-length table (a reference genome known only through a saved index): contigs [c0, c1)
inline uint64_t genomeLength(const std::vector<int32_t> &contigLen, int c0, int c1, int fragLen)
{
  uint64_t s = 0;
  for (int c = c0; c < c1; c++) if ((int64_t)contigLen[c] >= fragLen) s += ((uint64_t)contigLen[c] / (uint64_t)fragLen) * (uint64_t)fragLen;
  return s;
}

// computeCoreIdentity.hpp:103-153
inline void outputVisualizationFile(const skch::Parameters &parameters, const std::vector<MappingResult_CGI> &mappings_2way,
                                    const skch::Map &mapper, const skch::Sketch &refSketch, const std::string &queryName,
                                    const std::vector<std::string> &shardRefNames, std::ostream &outstrm)
{
  std::vector<int64_t> queryOffsetAdder(mapper.metadata.size()), refOffsetAdder(refSketch.metadata.size());
  for (size_t i = 0; i < mapper.metadata.size(); i++) queryOffsetAdder[i] = i ? queryOffsetAdder[i - 1] + mapper.metadata[i - 1].len : 0;
  for (size_t i = 0; i < refSketch.metadata.size(); i++) refOffsetAdder[i] = i ? refOffsetAdder[i - 1] + refSketch.metadata[i - 1].len : 0;
  for (const auto &e : mappings_2way) {
    outstrm << queryName << "\t" << shardRefNames[e.genomeId] << "\t" << e.nucIdentity << "\tNA\tNA\tNA"
            << "\t" << e.queryStartPos + queryOffsetAdder[e.querySeqId]
            << "\t" << e.queryStartPos + parameters.minReadLength - 1 + queryOffsetAdder[e.querySeqId]
            << "\t" << e.refStartPos + refOffsetAdder[e.refSequenceId]
            << "\t" << e.refStartPos + parameters.minReadLength - 1 + refOffsetAdder[e.refSequenceId]
            << "\tNA\tNA\n";
  }
}

// prefix sums of lengths: offset of entry i in the concatenation of entries 0 .. i-1
inline std::vector<int64_t> offsetAdder(const std::vector<skch::offset_t> &lens)
{
  std::vector<int64_t> off(lens.size() + 1, 0);
  for (size_t i = 0; i < lens.size(); i++) off[i + 1] = off[i] + lens[i];
  return off;
}

// outputVisualizationFile for the 2-way mappings of one query from the device reduction (bani_map_cgi_sketch_frags).
// queryOffsetAdder: offsetAdder of the query's Map::metadata lengths; refOffsetAdder: that of refSketch.metadata.
inline void outputVisualizationFile(const skch::Parameters &parameters, const bani_frag_mapping *frags, size_t n,
                                    const std::vector<int64_t> &queryOffsetAdder, const std::vector<int64_t> &refOffsetAdder,
                                    const skch::Sketch &refSketch, const std::string &queryName,
                                    const std::vector<std::string> &shardRefNames, std::ostream &outstrm)
{
  const auto &sbf = refSketch.sequencesByFileInfo;
  for (size_t i = 0; i < n; i++) {
    const bani_frag_mapping &e = frags[i];
    const size_t g = std::upper_bound(sbf.begin(), sbf.end(), e.refSeqId) - sbf.begin();   // :29-41
    outstrm << queryName << "\t" << shardRefNames[g] << "\t" << e.identity << "\tNA\tNA\tNA"
            << "\t" << queryOffsetAdder[e.querySeqId]
            << "\t" << parameters.minReadLength - 1 + queryOffsetAdder[e.querySeqId]
            << "\t" << e.refStartPos + refOffsetAdder[e.refSeqId]
            << "\t" << e.refStartPos + parameters.minReadLength - 1 + refOffsetAdder[e.refSeqId]
            << "\tNA\tNA\n";
  }
}

// computeCoreIdentity.hpp:166-298 from the mapping rows (host; the batch path uses bani_map_cgi instead)
inline void computeCGI(const skch::Parameters &parameters, const skch::MappingResultsVector_t &results, const skch::Map &mapper,
                       const skch::Sketch &refSketch, uint64_t totalQueryFragments, uint64_t queryFileNo, const std::string &queryName,
                       const std::vector<std::string> &shardRefNames, std::ostream *visual, std::vector<CGI_Results> &out)
{
  std::vector<MappingResult_CGI> shortResults; shortResults.reserve(results.size());
  for (const auto &e : results) {
    const auto it = std::upper_bound(refSketch.sequencesByFileInfo.begin(), refSketch.sequencesByFileInfo.end(), e.refSeqId);   // :29-41
    shortResults.push_back(MappingResult_CGI{e.refSeqId, (skch::seqno_t)(it - refSketch.sequencesByFileInfo.begin()), e.querySeqId,
                                             e.refStartPos, e.queryStartPos, e.refStartPos / (parameters.minReadLength - 20), e.nucIdentity});
  }
  std::vector<MappingResult_CGI> one, two;
  std::sort(shortResults.begin(), shortResults.end(), [](const MappingResult_CGI &x, const MappingResult_CGI &y) {
    return std::tie(x.genomeId, x.querySeqId, x.nucIdentity, x.refSequenceId, x.refStartPos) <
           std::tie(y.genomeId, y.querySeqId, y.nucIdentity, y.refSequenceId, y.refStartPos); });
  for (const auto &e : shortResults) {
    if (one.empty() || !(e.genomeId == one.back().genomeId && e.querySeqId == one.back().querySeqId)) one.push_back(e);
    else one.back() = e;
  }
  // the reference's std::sort leaves the order of equal (contig, bin, identity) keys unspecified; a stable sort is one of
  // its possible outcomes and keeps this deterministic
  std::stable_sort(one.begin(), one.end(), [](const MappingResult_CGI &x, const MappingResult_CGI &y) {
    return std::tie(x.refSequenceId, x.mapRefPosBin, x.nucIdentity) < std::tie(y.refSequenceId, y.mapRefPosBin, y.nucIdentity); });
  for (const auto &e : one) {
    if (two.empty() || !(e.refSequenceId == two.back().refSequenceId && e.mapRefPosBin == two.back().mapRefPosBin)) two.push_back(e);
    else two.back() = e;
  }
  if (visual) outputVisualizationFile(parameters, two, mapper, refSketch, queryName, shardRefNames, *visual);
  for (auto it = two.begin(); it != two.end();) {
    const skch::seqno_t g = it->genomeId;
    auto end = std::find_if(it, two.end(), [&](const MappingResult_CGI &e) { return e.genomeId != g; });
    float sum = 0.0f;
    for (auto i2 = it; i2 != end; ++i2) sum += i2->nucIdentity;
    CGI_Results r; r.qryGenomeId = (skch::seqno_t)queryFileNo; r.refGenomeId = g; r.countSeq = (skch::seqno_t)(end - it);
    r.totalQueryFragments = (skch::seqno_t)totalQueryFragments; r.identity = sum / r.countSeq;
    out.push_back(r);
    it = end;
  }
}

// computeCoreIdentity.hpp:457-474: reference j goes to shard j % G
// (block = true: contiguous ranges of the list instead -- same results, list neighbours stay on one GPU)
inline std::vector<std::vector<int>> splitReferenceGenomes(int nRefs, int G, bool block = false)
{
  std::vector<std::vector<int>> s(G);
  if (block) { for (int g = 0; g < G; g++) for (int j = (int)((int64_t)nRefs * g / G); j < (int)((int64_t)nRefs * (g + 1) / G); j++) s[g].push_back(j); }
  else for (int j = 0; j < nRefs; j++) s[j % G].push_back(j);
  return s;
}
// the inverse of splitReferenceGenomes: list position j -> (shard, ordinal inside the shard)
inline std::pair<int, int> referenceShardOrdinal(int j, int nRefs, int G, bool block = false)
{
  if (!block) return {j % G, j / G};
  auto start = [&](int g) { return (int)((int64_t)nRefs * g / G); };
  int g = (int)((int64_t)j * G / nRefs);                  // start(g) <= j; shards before j's may be empty (nRefs < G)
  while (g + 1 < G && start(g + 1) <= j) g++;
  return {g, j - start(g)};
}
// computeCoreIdentity.hpp:480-487: shard-local reference id -> global id
inline void correctRefGenomeIds(std::vector<CGI_Results> &v, int shard, int G, int nRefs = 0, bool block = false)
{
  const int base = block ? (int)((int64_t)nRefs * shard / G) : 0;
  for (auto &e : v) e.refGenomeId = block ? base + e.refGenomeId : e.refGenomeId * G + shard;
}

inline bool passesMinFraction(const skch::Parameters &p, const CGI_Results &e, uint64_t qLen, uint64_t rLen)
{
  const uint64_t minGenomeLength = std::min(qLen, rLen);
  const uint64_t sharedLength = (uint64_t)((int64_t)e.countSeq * p.minReadLength);     // int * int in the reference (:323)
  return sharedLength >= minGenomeLength * p.minFraction;                               // uint64 * float -> float (:326)
}

// computeCoreIdentity.hpp:307-343.  The reference sorts with an operator< that orders by query ascending, identity
// descending and leaves ties to std::sort; ties are broken here by reference id so the output is reproducible.
inline void outputCGI(const skch::Parameters &p, const std::unordered_map<std::string, uint64_t> &genomeLengths,
                      std::vector<CGI_Results> &v, const std::string &fileName)
{
  std::sort(v.begin(), v.end(), [](const CGI_Results &a, const CGI_Results &b) {
    if (a.qryGenomeId != b.qryGenomeId) return a.qryGenomeId < b.qryGenomeId;
    if (a.identity != b.identity) return a.identity > b.identity;
    return a.refGenomeId < b.refGenomeId; });
  std::ofstream outstrm(fileName);
  for (const auto &e : v) {
    const std::string &q = p.querySequences[e.qryGenomeId], &r = p.refSequences[e.refGenomeId];
    if (passesMinFraction(p, e, genomeLengths.at(q), genomeLengths.at(r)))
      outstrm << q << "\t" << r << "\t" << e.identity << "\t" << e.countSeq << "\t" << e.totalQueryFragments << "\n";
  }
}

// computeCoreIdentity.hpp:352-448
inline void outputPhylip(const skch::Parameters &p, const std::unordered_map<std::string, uint64_t> &genomeLengths,
                         const std::vector<CGI_Results> &v, const std::string &fileName)
{
  std::unordered_map<std::string, int> genome2Int; std::vector<std::string> rev;
  for (const auto *lst : {&p.querySequences, &p.refSequences})
    for (const auto &e : *lst) if (!genome2Int.count(e)) { genome2Int[e] = (int)rev.size(); rev.push_back(e); }
  const int n = (int)rev.size();
  std::vector<std::vector<float>> m(n, std::vector<float>(n, 0.0f));
  for (const auto &e : v) {
    const std::string &q = p.querySequences[e.qryGenomeId], &r = p.refSequences[e.refGenomeId];
    if (!passesMinFraction(p, e, genomeLengths.at(q), genomeLengths.at(r))) continue;
    int a = genome2Int[q], b = genome2Int[r];
    if (a == b) continue;
    if (a < b) std::swap(a, b);
    m[a][b] = m[a][b] > 0 ? (m[a][b] + e.identity) / 2 : e.identity;
  }
  std::ofstream outstrm(fileName + ".matrix");
  outstrm << n << "\n";
  for (int i = 0; i < n; i++) {
    outstrm << rev[i];
    for (int j = 0; j < i; j++) outstrm << "\t" << (m[i][j] > 0.0 ? std::to_string(m[i][j]) : std::string("NA"));
    outstrm << "\n";
  }
}

} // namespace cgi
