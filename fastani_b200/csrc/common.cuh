// common.cuh -- internal types shared by the translation units of libfastani_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <memory>
#include <map>
#include <stdexcept>
#include <cstdio>
#include <cstdarg>
#include <chrono>
#include <type_traits>
#include "../../include/fastani_b200.h"

namespace bani {

// ---------------------------------------------------------------- errors
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

void set_last_error(const std::string &m);

[[noreturn]] inline void fail(int code, const char *fmt, ...)
{
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  throw Error(code, buf);
}

#define BANI_CUDA(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
  ::bani::fail(BANI_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// ---------------------------------------------------------------- device memory
// DevBuf owns a block from the caching allocator of alloc.cpp (freed blocks are reused on the same
// stream; the driver is only called on a miss).
void *dev_alloc(size_t bytes, cudaStream_t st, size_t *granted, int *dev);
void  dev_free(void *p, size_t granted, cudaStream_t st, int dev);      // dev = the device the block was allocated on
void  dev_cache_flush(int dev);
size_t dev_round_size(size_t bytes);                                    // what a request of `bytes` is rounded to
void  dev_mem_stats(int dev, size_t *live, size_t *cached, size_t *peakLive);
void  dev_mem_peak_set(int dev, size_t v);                              // peakLive = max(v, live)

template <typename T>
struct DevBuf {
  T *p = nullptr; size_t n = 0; cudaStream_t st = nullptr; size_t granted = 0; int dev = -1;
  DevBuf() {}
  DevBuf(size_t n_, cudaStream_t s) { alloc(n_, s); }
  DevBuf(const DevBuf &) = delete; DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), n(o.n), st(o.st), granted(o.granted), dev(o.dev) { o.p = nullptr; o.n = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept
  { if (this != &o) { release(); p = o.p; n = o.n; st = o.st; granted = o.granted; dev = o.dev; o.p = nullptr; o.n = 0; } return *this; }
  ~DevBuf() { release(); }
  void alloc(size_t n_, cudaStream_t s)
  {
    release(); n = n_; st = s;
    if (n == 0) return;
    p = (T *)dev_alloc(n * sizeof(T), s, &granted, &dev);
  }
  void release() { if (p) { dev_free(p, granted, st, dev); p = nullptr; } n = 0; }
  size_t bytes() const { return n * sizeof(T); }
};

// ---------------------------------------------------------------- statistics (host)
int   stat_recommended_window_size(double p_value, int k, float identity, int fragLen, uint64_t refSize);
int   stat_min_hits_relaxed(int s, int k, float identity);
void  stat_identity(int shared, int s, int k, float *id, float *ub);

// LUT rows consumed by the mapping kernels: for sketch size s,
//   minHits[s]            = max(1, estimateMinimumHitsRelaxed(s, k, pid))
//   rowOff[s] .. +s+1     : identity[x], upper[x] for x = 0..s
struct StatLut {
  int k = 0; float pid = 0;
  std::vector<int32_t> minHits;     // index s (0 unused)
  std::vector<uint32_t> rowOff;     // index s -> offset into ident/upper
  std::vector<float> ident, upper;
  int smax = 0;                     // rows 1 .. smax are all present (dense part)
  std::vector<char> have;           // beyond the dense part: rows computed on demand (index s)
  void ensure(int s_needed);        // extends the dense part up to s_needed (host)
  bool ensure_rows(const std::vector<int> &svals);   // makes the rows of these sketch sizes present; true if anything was added
};

// ---------------------------------------------------------------- genomes
// Per-contig descriptor consumed by the sketch kernel.  A query fragment is the
// same thing with a non-zero startBase and len = fragLen.
struct SeqDesc {
  const uint32_t *packed;   // first 2-bit word of the parent contig (16 bases / word)
  const uint32_t *excPos;   // sorted contig-relative positions of non-ACGT bytes (parent contig)
  const uint8_t  *excByte;  // their (upper-cased) bytes
  int32_t nExc;
  int32_t startBase;        // offset of this sequence inside the parent contig
  int32_t len;              // bases
  int32_t seqId;            // ordinal written to the records
};

uint64_t next_genome_uid();

// Device block shared by the genomes of one upload sub-batch of the host-packed path (bani_genome_create_packed_batch):
// one H2D copy per array on the context's copy stream; `ready` is recorded behind them and every consumer makes its
// stream wait for it, so uploads of later sub-batches overlap the sketch launches of earlier ones.
struct GenomeBlock {
  DevBuf<uint32_t> words; DevBuf<uint32_t> excPos; DevBuf<uint8_t> excByte;
  cudaEvent_t ready = nullptr; int device = 0;
  ~GenomeBlock() { if (ready) { cudaSetDevice(device); cudaEventDestroy(ready); } }
};

struct Genome {
  uint64_t uid = next_genome_uid();  // identity that survives address reuse (index membership, see Index::members)
  int device = 0;
  int32_t nContigs = 0;
  std::vector<int32_t> len;          // per contig
  std::vector<int64_t> wordOff;      // per contig, into packed (multiple of 4 words)
  std::vector<int64_t> excOff;       // per contig +1, into exc arrays
  uint64_t totalLen = 0, nExc = 0;
  DevBuf<uint32_t> packed;           // own buffers (ASCII ingest, pack.cu) ...
  DevBuf<uint32_t> excPos;
  DevBuf<uint8_t>  excByte;
  std::shared_ptr<GenomeBlock> blk;  // ... or a slice of a shared upload block (host-packed ingest)
  const uint32_t *blkWords = nullptr; const uint32_t *blkExcPos = nullptr; const uint8_t *blkExcByte = nullptr;
  const uint32_t *packedBase() const { return blk ? blkWords : packed.p; }
  const uint32_t *excPosBase() const { return blk ? blkExcPos : excPos.p; }
  const uint8_t  *excByteBase() const { return blk ? blkExcByte : excByte.p; }
  void wait_ready(cudaStream_t st) const { if (blk && blk->ready) cudaStreamWaitEvent(st, blk->ready, 0); }
};

struct Ctx;

// ---------------------------------------------------------------- query sketch (first half of HP2)
// Map::doL1Mapping, computeMap.hpp:252-276: per fragment the sorted unique minimizer hashes Q, s = |Q|.
// A piece holds at most 2^18 fragments of whole query genomes (map.cu: FRAG_MAX); arrays are packed back to back so that a
// sketch can be exported to one flat device buffer and moved between GPUs.
struct QPiece {
  uint64_t memberOf = 0;             // uid of the index the fragment sketches were derived from (stage A'), 0 = hashed / imported
  int q0 = 0, nq = 0;                // local query range [q0, q0 + nq) of the owning sketch
  int32_t F = 0; uint64_t T = 0; int smax = 0;
  DevBuf<uint32_t> fragHash;         // T  : sorted unique hashes of fragment f at [segStart[f], segStart[f+1])
  DevBuf<uint32_t> segStart;         // F+1
  DevBuf<int32_t>  sCount;           // F  : s
  DevBuf<int32_t>  fragQuery;        // F  : query slot inside the piece (0 .. nq)
  DevBuf<int32_t>  fragSeqId;        // F  : querySeqId of the mapping records (fragment ordinal inside its genome)
  std::vector<int32_t> qFragOff;     // nq+1 (host): first fragment of every query of the piece
};
struct QSketch {
  int device = 0; int k = 0, w = 0, fragLen = 0;
  std::vector<int32_t> queryId;          // id reported as qryGenomeId
  std::vector<uint64_t> totalFragments;  // Map's totalQueryFragments per query
  std::vector<std::unique_ptr<QPiece>> pieces;
  uint64_t F = 0, T = 0;
};

// ---------------------------------------------------------------- index (HP1 output)
struct Index {
  uint64_t uid = next_genome_uid();  // identity of this index (a query sketch remembers the index it was derived from)
  int device = 0;
  uint64_t M = 0, U = 0, totalLen = 0;
  int32_t nContigs = 0, nGenomes = 0;
  int dirBits = 0;
  // position-ordered records (== Sketch::minimizerIndex as SoA) + same-hash links
  DevBuf<uint32_t> hash; DevBuf<int32_t> wpos; DevBuf<int32_t> seqId; DevBuf<uint32_t> link;
  DevBuf<int2> pos8;                 // {wpos, seqId} per record: what the L1 stage fetches per sorted hit (one 8-byte load)
  DevBuf<uint2> rec8;                // 8-byte L2 record: x = hash, y = back:14 | fwd:14 | tie | new | gone (index.cu); valid where blkMax allows
  DevBuf<uint32_t> blkMax;           // per 1024 records: max back | max fwd << 16 (0xFFFF: a link does not fit 14 bits)
  DevBuf<uint4> rec;                 // 16-byte L2 record: x=hash, y=wpos|tie<<31, z=twin link, w=back|fwd<<16 (index.cu)
  int cmw = 0;                       // super-window width the back/fwd fields were computed for
  int k = 0, w = 0, fragLen = 0;     // parameters of the context the index was built with
  DevBuf<uint32_t> contigRecOff;     // nContigs+1: first record of each contig
  DevBuf<int32_t>  contigGenome;     // nContigs: genome ordinal of a contig (reviseRefIdToGenomeId)
  DevBuf<uint32_t> contigBinOff;     // nContigs+1: prefix of #position-bins per contig (CGI)
  // hash-ordered lookup side (== Sketch::minimizerPosLookupIndex)
  DevBuf<uint32_t> ukeys;            // U unique hashes ascending
  DevBuf<uint32_t> uoff;             // U+1 offsets into posIdx
  DevBuf<uint32_t> posIdx;           // M record indices, sorted by (hash, record index)
  DevBuf<uint32_t> dir;              // (1<<dirBits)+1 bucket directory over the top bits of the hash
  // one-sector probe table: 2^tabBits buckets of 4 entries {x = (hash & ~0xFF) | min(count, 255), y = offset into posIdx},
  // bucket = LOW bits of the hash (uniform, unlike the top bits of a minimizer hash); x == 0 = empty.  A full bucket or a
  // saturated count sends the probe to the sorted keys above (index.cu: table_fill_kernel, map.cu: lookup_kernel)
  DevBuf<uint2> tab; int tabBits = 0;
  // membership filter in front of the probe table for small shards (multi-GPU): one bit per value of the low filtBits bits
  // of the hash, sized 8x the unique hashes and at most 32 MB so that it stays L2-resident; a clear bit answers a miss
  // without touching DRAM (most probes of a shard are misses when the queries of other shards are mapped against it)
  DevBuf<uint32_t> filt; int filtBits = 0;
  std::vector<int32_t> contigLen;    // host copies
  std::vector<int32_t> seqsByFile;   // cumulative contig count per genome (sequencesByFileInfo)
  // Which genomes the index was built from (uid -> first contig ordinal) and, per hashed position, whether it was
  // VALID (forward hash != reverse-complement hash, commonFunc.hpp:131): together with the position-ordered records
  // this is enough to derive the fragment sketches of a member genome without hashing it again (map.cu, stage A').
  std::map<uint64_t, int32_t> members;
  DevBuf<uint32_t> validBits;        // bit contigBitBase[c] + p = position p of contig c is valid
  DevBuf<unsigned long long> contigBitBase;   // nContigs (multiples of 32)
  uint64_t totalBins = 0;
};

// A non-owning typed view of a persistent scratch slot.
template <typename T>
struct View {
  T *p = nullptr; size_t n = 0;
};

// Run-time switches of a context (bani_ctx_set_flag); the defaults can also be set through the environment
// (BANI_NO_SKETCH_REUSE, BANI_MAX_HITS_PER_PIECE, BANI_FRAG_L1_MAX, BANI_L2E_BUCKETS, BANI_L2_STAGE, BANI_TRACE, BANI_CGI_SPARSE),
// read when the context is created.
struct CtxFlags {
  int sketchReuse = 1;                        // stage A': fragment sketches of index members are read from the index
  long long maxHitsPerPiece = 3ll << 29;      // a piece that gathers more index hits is split at a query boundary
  long long fragL1Max = 8192;                 // hits per fragment handled inside one CTA (<= FRAG_L1_MAX)
  int l2eBuckets = 0;                         // 0 = adaptive; 1024 / 4096 force the size of the L2 rank directory
  int trace = 0;                              // BANI_TRACE: wall-clock marks of the host orchestration on stderr (diagnostic)
  int l2Stage = 1;                            // 1: l2_events_kernel stages event codes in shared memory where the window links allow it
                                              //    (more instructions for about half the DRAM traffic: the faster choice on H100, DESIGN.md
                                              //    section 6); 0: direct stores for every candidate, kept as a tested alternative
  long long uploadGroupWords = 16ll << 20;    // packed words (16 bases each) per upload group of the host-packed ingest
  // Test switches that bring branches of the mapping path, which otherwise need very large inputs, down to small ones.
  // Results never depend on them.
  long long fragsPerPiece = 1ll << 18;        // fragments per query piece (map.cu: FRAG_MAX is the default and the maximum)
  long long eventBytesPerPiece = 0;           // a piece whose L2 event streams take more is halved; 0 = a quarter of device memory
  long long cgiTableQueries = 0;              // queries per pass of the identity reduction; 0 = as many as 3 GiB of bin table hold
  int l2Fast = 1;                             // 0: every L2 candidate goes to the exact kernel (l2_kernel)
  int countPaths = 0;                         // 1: count which branch of the mapping path ran (bani_ctx_path_counts)
  int cgiSparse = -1;                         // stage H per piece: -1 chosen from the piece's size, 0 dense tables, 1 sparse rows
  // Budgets of a run that builds its references in chunks (bani_ctx_plan_run); results never depend on them.
  unsigned long long indexBytesBudget = 0;    // build peak of one chunk's index; 0 = derived from device memory
  unsigned long long querySketchBudget = 0;   // query sketches resident at once; 0 = derived from device memory
};

// Branches of the mapping path, counted when CtxFlags::countPaths is set (names: capi.cu, bani_ctx_path_counts).  What a
// counter counts: fragments per L1 size class; probes that walked the sorted keys; L2 candidates with window events per
// event-kernel variant; candidates left to the exact kernel after the bounds pass and in total; pieces and passes;
// pieces whose identity reduction took the sparse path (cgi.passes counts dense passes only).
// The per-piece counters (everything but piece.split_*) are those of the pieces that were mapped, not of those split.
enum PathId {
  P_L1_CLASS0 = 0, P_L1_DEVICE_WIDE = 13,                    // 13 == FRAG_NCLASS
  P_LOOKUP_WALK_SATURATED, P_LOOKUP_WALK_FULL_BUCKET,
  P_L2_EVENTS_NT64, P_L2_EVENTS_NT128, P_L2_EVENTS_NT256, P_L2_DIR1024, P_L2_DIR4096, P_L2_STAGED, P_L2_DIRECT,
  P_L2_EXACT_AT_BOUNDS, P_L2_EXACT_TOTAL,
  P_PIECE_MAPPED, P_PIECE_SPLIT_HITS, P_PIECE_SPLIT_EVENTS, P_CGI_PASSES, P_CGI_SPARSE,
  NPATH
};
extern const char *const PATH_NAMES[NPATH];

// CUB-backed primitives (cubops.cu; kept in one TU because CUB compiles slowly)
size_t cub_sort_pairs_u32_temp(size_t n);
void   cub_sort_pairs_u32(void *temp, size_t tempBytes, const uint32_t *kin, uint32_t *kout,
                          const uint32_t *vin, uint32_t *vout, size_t n, int endBit, cudaStream_t s);
size_t cub_sort_keys_u64_temp(size_t n);
void   cub_sort_keys_u64(void *temp, size_t tempBytes, const uint64_t *kin, uint64_t *kout, size_t n,
                         int beginBit, int endBit, cudaStream_t s);
size_t cub_sort_pairs_u64_u32_temp(size_t n);
void   cub_sort_pairs_u64_u32(void *temp, size_t tempBytes, const uint64_t *kin, uint64_t *kout,
                              const uint32_t *vin, uint32_t *vout, size_t n, int endBit, cudaStream_t s);
size_t cub_scan_u32_temp(size_t n);
void   cub_exclusive_sum_u32(void *temp, size_t tempBytes, const uint32_t *in, uint32_t *out, size_t n, cudaStream_t s);
size_t cub_scan_u64_temp(size_t n);
void   cub_exclusive_sum_u32_to_u64(void *temp, size_t tempBytes, const uint32_t *in, uint64_t *out, size_t n, cudaStream_t s);

struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copyStream = nullptr;   // H2D uploads of host-packed genomes (overlap with the sketch launches on `stream`)
  bani_params prm{};
  CtxFlags flags;
  int smCount = 0;
  size_t memTotal = 0;               // device memory: bounds the working set of a mapping piece (map.cu)
  StatLut lut;
  DevBuf<int32_t> d_minHits; DevBuf<uint32_t> d_rowOff; DevBuf<float> d_ident, d_upper;
  int lutUploaded = 0;
  void upload_lut(int smax, const int32_t *d_sCount = nullptr, int32_t F = 0);
  // optional per-stage device timing (CUDA events on `stream`), see bani_ctx_profile_*
  // diagnostic: microseconds of host wall clock since the previous mark (flags.trace)
  std::chrono::steady_clock::time_point traceT = std::chrono::steady_clock::now();
  void mark(const char *what)
  {
    if (!flags.trace) return;
    const auto t = std::chrono::steady_clock::now();
    fprintf(stderr, "[bani trace] %-28s +%8.1f us\n", what, std::chrono::duration<double, std::micro>(t - traceT).count());
    traceT = t;
  }
  uint64_t launches = 0;             // kernels of this library launched so far (CUB's not counted)
  uint64_t paths[NPATH] = {};        // branch counters since the last bani_ctx_path_counts (flags.countPaths)
  bool profiling = false;
  struct ProfEv { const char *name; cudaEvent_t a, b; double bytes; };
  std::vector<ProfEv> profEvents;
  // Grow-only scratch slots for the per-chunk working set of the mapping pipeline (hit keys, flags,
  // candidate arrays ...): after the first chunk nothing is allocated or freed inside the timed path.
  std::map<uint64_t, DevBuf<uint8_t>> slots;
  // Temp storage of the CUB calls of the mapping path: one grow-only buffer serves them all, because every such call is
  // enqueued on `stream` and its temp storage is dead once the call has run in stream order (a buffer that grows goes
  // back to the caching allocator on `stream`, which is stream-ordered too).
  DevBuf<uint8_t> cubTemp;
  // kernel function attributes (dynamic shared memory limit, carve-out) are per DEVICE: remember per context what has
  // been set, so that a process driving several GPUs (the C++ CLI: one thread + context per GPU) sets them on each
  std::map<const void *, bool> attrDone;
  bool first_time(const void *key) { bool &d = attrDone[key]; const bool f = !d; d = true; return f; }
  template <typename T> View<T> view(uint64_t id, size_t n)
  {
    DevBuf<uint8_t> &b = slots[id];
    const size_t bytes = (n ? n : 1) * sizeof(T);
    if (b.n < bytes) b.alloc(bytes + bytes / 8 + 256, stream);
    View<T> v; v.p = (T *)b.p; v.n = n; return v;
  }
  void *cub_temp(size_t bytes) { if (cubTemp.n < bytes) cubTemp.alloc(bytes + bytes / 8 + 256, stream); return cubTemp.p; }
  // exclusive sums and radix sorts on `stream`
  void scan(const uint32_t *in, uint32_t *out, size_t n) { size_t b = cub_scan_u32_temp(n); cub_exclusive_sum_u32(cub_temp(b), b, in, out, n, stream); }
  void scan(const uint32_t *in, unsigned long long *out, size_t n)
  { size_t b = cub_scan_u64_temp(n); cub_exclusive_sum_u32_to_u64(cub_temp(b), b, in, (uint64_t *)out, n, stream); }
  void sort_pairs(const uint32_t *kin, uint32_t *kout, const uint32_t *vin, uint32_t *vout, size_t n, int endBit)
  { size_t b = cub_sort_pairs_u32_temp(n); cub_sort_pairs_u32(cub_temp(b), b, kin, kout, vin, vout, n, endBit, stream); }
  void sort_pairs(const unsigned long long *kin, unsigned long long *kout, const uint32_t *vin, uint32_t *vout, size_t n, int endBit)
  { size_t b = cub_sort_pairs_u64_u32_temp(n); cub_sort_pairs_u64_u32(cub_temp(b), b, (const uint64_t *)kin, (uint64_t *)kout, vin, vout, n, endBit, stream); }
  void sort_keys(const unsigned long long *kin, unsigned long long *kout, size_t n, int endBit)
  { size_t b = cub_sort_keys_u64_temp(n); cub_sort_keys_u64(cub_temp(b), b, (const uint64_t *)kin, (uint64_t *)kout, n, 0, endBit, stream); }
};

constexpr uint64_t fnv1a(const char *s, uint64_t h = 0xcbf29ce484222325ull)
{ return *s ? fnv1a(s + 1, (h ^ (unsigned char)*s) * 0x100000001b3ull) : h; }
// one scratch slot per (source file, source line): never put two BANI_SCRATCH on one line
#define BANI_SLOT_ID (::std::integral_constant<uint64_t, ::bani::fnv1a(__FILE__) ^ (uint64_t)__LINE__>::value)
#define BANI_SCRATCH(T, name, count) ::bani::View<T> name = ctx->view<T>(BANI_SLOT_ID, (count))

// RAII stage timer: records an event pair around a stage when profiling is on.
struct Stage {
  Ctx *c; size_t idx = (size_t)-1;
  Stage(Ctx *ctx, const char *name, double algoBytes = 0) : c(ctx)
  {
    if (!c->profiling) return;
    Ctx::ProfEv e; e.name = name; e.bytes = algoBytes;
    cudaEventCreate(&e.a); cudaEventCreate(&e.b);
    cudaEventRecord(e.a, c->stream);
    idx = c->profEvents.size(); c->profEvents.push_back(e);
  }
  void bytes(double b) { if (idx != (size_t)-1) c->profEvents[idx].bytes = b; }
  size_t id() const { return idx; }                       // to set the bytes after the stage has been closed
  static void set_bytes(Ctx *c, size_t id, double b) { if (id != (size_t)-1 && id < c->profEvents.size()) c->profEvents[id].bytes = b; }
  void stop() { if (idx != (size_t)-1) { cudaEventRecord(c->profEvents[idx].b, c->stream); idx = (size_t)-1; } }
  ~Stage() { stop(); }
};

// ---------------------------------------------------------------- kernels' host entry points
// pack.cu
void genome_create_batch(Ctx *ctx, int32_t nGenomes, const int32_t *genOff, const int64_t *off,
                         const uint8_t *seq, Genome **out);
void genome_decode(Ctx *ctx, const Genome *g, int32_t contig, uint8_t *out, int64_t cap);
void genome_create_packed_batch(Ctx *ctx, int32_t nGenomes, const int32_t *genOff, const int32_t *contigLen, const int64_t *wordOff,
                                const uint32_t *words, const int64_t *excOff, const uint32_t *excPos, const uint8_t *excByte,
                                bool async, Genome **out);
uint64_t host_pack_contig(const uint8_t *seq, int64_t len, uint32_t *words, uint32_t *excPos, uint8_t *excByte, uint64_t excCap);

// sketch.cu : windowed minimizers of a list of sequences, records compacted in
// (sequence, wpos) order.  Outputs may be null (skipped).  Returns total records
// (which may exceed `cap`; only the first cap are stored).
// recBase: records already written by earlier launches into the same output arrays (index build in upload groups);
// outputs and segStart values are offset by it, `cap` is the capacity of the whole arrays.
uint64_t sketch_sequences(Ctx *ctx, const SeqDesc *d_desc, int32_t nSeq, const int32_t *h_len, int32_t uniformLen,
                          uint32_t *o_hash, int32_t *o_wpos, int32_t *o_seqId, uint64_t cap,
                          uint32_t *o_segStart /* nSeq+1 */,
                          uint32_t *o_validBits = nullptr, const unsigned long long *bitBase = nullptr, uint64_t recBase = 0);

// index.cu
Index *index_build(Ctx *ctx, Genome *const *refs, int32_t nRefs);
// The longest prefix of refs whose build peak (index_footprint) fits maxBytes, at least one genome (BANI_ERR_LIMIT if that
// one does not fit); the index equals index_build's of exactly that prefix.  *peakBytes: most bytes held above the entry.
Index *index_build_budget(Ctx *ctx, Genome *const *refs, int32_t nRefs, uint64_t maxBytes, int32_t *nTaken, uint64_t *peakBytes);

// budget.cpp (host arithmetic only): index footprint, mapping working set, index budget, chunk plan
inline int index_dir_bits(uint64_t U) { int b = 8; while (b < 23 && (1ull << b) < U) b++; return b; }    // <= 32 MB directory
inline int index_tab_bits(uint64_t U) { int b = 8; while (b < 28 && (1ull << b) < U) b++; return b; }    // >= U buckets, <= 2^28
inline int index_filt_bits(uint64_t U)                                                                  // 0 = no filter; <= 32 MB
{
  if (U > (1ull << 26)) return 0;
  int fb = 8; while ((1ull << fb) < U) fb++;
  return fb + 3 < 28 ? fb + 3 : 28;
}
// th/tw/ts capacity of index_build: 1.5x the expected 2 / (w + 1) minimizers per position
inline uint64_t index_staging_cap(uint64_t totalPos, int w)
{
  const uint64_t c = (uint64_t)(3.0 * totalPos / (w + 1)) + 65536;
  return c < totalPos ? c : totalPos;
}
struct IndexFootprint { uint64_t peak = 0, resident = 0; };
IndexFootprint index_footprint(uint64_t M, uint64_t Ubound, uint64_t nContigs, uint64_t bitmapBits, uint64_t stagingCap);
uint64_t map_working_set(uint64_t deviceBytes, long long maxHitsPerPiece, long long eventBytesPerPiece);
uint64_t map_working_set_run(uint64_t deviceBytes, long long maxHitsPerPiece, long long eventBytesPerPiece, uint64_t queryHashes,
                             uint64_t queryFragments, uint64_t nQueries, uint64_t refBases, uint64_t nRefs, int w, int fragLen);
uint64_t index_budget(uint64_t freeBytes, uint64_t qsketchBytes, uint64_t workingSet, int w);
int32_t  plan_chunks(const uint64_t *len, const int32_t *nContigs, int32_t n, int k, int w, uint64_t budget, int32_t *ends);
uint64_t qsketch_bytes_estimate(uint64_t len, int w, int fragLen);
// what a run plan depends on besides the genome sizes: free device bytes (free + cached), the device's size, the piece caps,
// the forced budgets (0 = derived) and the parameters
struct RunSize {
  uint64_t freeBytes = 0, deviceBytes = 0; long long maxHitsPerPiece = 0, eventBytesPerPiece = 0;
  uint64_t indexBudget = 0, queryBudget = 0; int k = 16, w = 1, fragLen = 3000;
};
int32_t plan_run(const RunSize &r, const uint64_t *refLen, const int32_t *refContigs, int32_t nRefs, const uint64_t *queryLen,
                 const uint64_t *qsBytes, int32_t nQ, int32_t *chunkEnd, int32_t *blockEnd, int32_t *nBlocks, uint64_t *indexBudget);
bool     parse_byte_count(const char *s, uint64_t *out);
void   index_save(Ctx *ctx, const Index *ix, const char *path);
Index *index_load(Ctx *ctx, const char *path);
// Header and tables of a saved index (host only, index.cu: file layout), checked as index_load checks them and, from
// version 3 on, against the table checksum.  Genome g owns contigs [contig_begin(g), seqsByFile[g]), records
// [recOff[c0], recOff[c1]) and validity bits [bitOff[c0], bitOff[c1]).
struct IndexFileInfo {
  int version = 0, k = 0, w = 0, fragLen = 0;
  uint64_t M = 0, nContigs = 0, nGenomes = 0, validWords = 0;
  std::vector<int32_t> contigLen, seqsByFile;
  std::vector<uint32_t> recOff;                 // nContigs + 1
  std::vector<uint64_t> bitOff;                 // nContigs + 1: first validity bit of every contig (multiples of 32)
  uint64_t contig_begin(int32_t g) const { return g ? (uint64_t)seqsByFile[g - 1] : 0; }
  uint64_t off_hash() const;                    // byte offsets of the file's sections
  uint64_t off_wpos() const { return off_hash() + 4 * M; }
  uint64_t off_bits() const { return off_wpos() + 4 * M; }
  uint64_t off_sums() const;
  uint64_t file_bytes() const;
};
IndexFileInfo index_file_info(const char *path);
// The version-3 file inPath followed by the genomes of `added`, written to outPath: equal byte for byte to index_save of the
// index built from inPath's genomes and then added's.  The old file is streamed through a host buffer and checked on the way.
void index_file_extend(Ctx *ctx, const char *inPath, const Index *added, const char *outPath);
// The longest run of genomes [first, first + *nTaken) of a version-3 file whose load (index_footprint of its exact record
// count, no sketch staging) fits maxBytes, at least one (BANI_ERR_LIMIT if that one does not fit); only that run is read.
// The index equals index_build's of exactly those genomes.  *peakBytes: most bytes held above the entry.
Index *index_load_budget(Ctx *ctx, const char *path, int32_t first, uint64_t maxBytes, int32_t *nTaken, uint64_t *peakBytes);
struct QSketch;
// qsketch_from_index over the genomes `ordinals` of a version-3 file, reading only their records
QSketch *qsketch_from_index_file(Ctx *ctx, const char *path, const int32_t *ordinals, int32_t nq, const int32_t *queryIds);

// map.cu
struct MapOutput {
  std::vector<bani_mapping> rows;               // when wantRows
  std::vector<bani_cgi_result> cgi;             // when wantCgi
  std::vector<bani_frag_mapping> frags;         // when wantFrags: the 2-way mappings behind cgi
  std::vector<uint64_t> totalQueryFragments;    // per query
  bani_map_counters ctr{};
};
void map_queries(Ctx *ctx, const Index *ix, const Genome *const *queries, int32_t nq,
                 bool wantRows, bool wantCgi, MapOutput &out);
QSketch *qsketch_create(Ctx *ctx, const Genome *const *queries, int32_t nq, const int32_t *queryIds, const Index *hint);
QSketch *qsketch_from_index(Ctx *ctx, const Index *ix, const int32_t *ordinals, int32_t nq, const int32_t *queryIds);
// the same without the check that the index holds records: stage A' reads only contigRecOff, wpos, hash, the validity
// bitmap and the contig tables, so `ix` may be a partial index read from a file (index.cu) without index_finish
QSketch *qsketch_from_records(Ctx *ctx, const Index *ix, const int32_t *ordinals, int32_t nq, const int32_t *queryIds);
uint64_t qsketch_export_bytes(const QSketch *qs);
void qsketch_export(Ctx *ctx, const QSketch *qs, void *devBuf, uint64_t cap);
QSketch *qsketch_import(Ctx *ctx, const void *devBuf, uint64_t bytes);
QSketch *qsketch_merge(Ctx *ctx, const QSketch *const *sketches, int32_t n);
// wantFrags (implies wantCgi): the identity reduction also records which fragment won each bin (out.frags)
void qsketch_map(Ctx *ctx, const Index *ix, const QSketch *const *sketches, int32_t nSketches,
                 bool wantRows, bool wantCgi, MapOutput &out, bool wantFrags = false);

// cgi.cu : stage H, the per-pair identity reduction of the mapping rows of a piece.  CgiState lives for one qsketch_map
// call: the 2-way bin table, its touched flags per (query, genome) and the last contig of every genome.
struct CgiState {
  const Index *ix; bool frags;                  // frags: 8-byte bins that also identify the winning fragment, else 4-byte
  uint64_t qMax = 0, tableQ = 0;                // queries the bin table may hold / holds (per pass over the rows)
  DevBuf<uint8_t> table; DevBuf<uint8_t> touched; DevBuf<int32_t> gce;
  CgiState(Ctx *ctx, const Index *ix, bool frags);
  uint64_t bin_bytes() const { return frags ? 8 : 4; }
};
// Results in query-slot space: dense (count, identity) tables [slot][genome] or sparse pairs (qryGenomeId = slot), and
// when CgiState::frags the 2-way winners (qryGenomeId = slot)
struct CgiResult {
  std::vector<int32_t> count; std::vector<float> ident; std::vector<bani_cgi_result> pairs; std::vector<bani_frag_mapping> frags;
};
// the R mapping rows of a piece in (fragment, candidate) order, the fragment of each row, the query slot (0 .. nQ) of each fragment
void cgi_piece(Ctx *ctx, CgiState &cs, const bani_mapping *rows, const int32_t *rFrag, uint32_t R, const int32_t *fragQuery, int nQ,
               uint64_t *pp, CgiResult &res);

// hits.cu : per-fragment gather + shared-memory sort + L1 candidate regions
static constexpr unsigned long long FRAG_L1_MAX = 8192;   // hits per fragment handled inside one CTA
static constexpr int FRAG_NCLASS = 13;                    // size classes: 256 * {1,2,3,4,5,6,7,8,10,12,16,24,32} hits
static_assert(P_L1_DEVICE_WIDE == FRAG_NCLASS, "one path counter per L1 size class");
__host__ __device__ inline int frag_class_items(int cls)
{
  return cls < 8 ? cls + 1 : (cls == 8 ? 10 : cls == 9 ? 12 : cls == 10 ? 16 : cls == 11 ? 24 : 32);
}
struct FragL1Args {
  const uint32_t *segStart; const int32_t *sCount; int32_t F;
  const uint32_t *hitLo, *hitCnt; const unsigned long long *hitOff;
  const uint32_t *posIdx; const int2 *recPos;    // recPos[r] = {wpos, seqId} of record r
  const int32_t *minHits; int fragLen, keyBits;
  int32_t *stSeq, *stStart, *stEnd;      // staging, addressed by global hit offset
  uint32_t *candCount;                   // per fragment
};
void frag_classify(Ctx *ctx, const uint32_t *segStart, const unsigned long long *hitOff, int32_t F,
                   uint32_t *candCount, uint32_t *fragClass, uint32_t *classCount, uint32_t *classList, unsigned long long maxFast);
void frag_l1_fast(Ctx *ctx, const FragL1Args &a, const uint32_t *classList, const uint32_t *classCount);
void cand_stage(Ctx *ctx, const int32_t *cFrag, const int32_t *cSeq, const int32_t *cStart, const int32_t *cEnd, uint32_t C,
                const uint32_t *segStart, const unsigned long long *hitOff, int32_t *stSeq, int32_t *stStart, int32_t *stEnd,
                uint32_t *candCount);
void cand_compact(Ctx *ctx, const uint32_t *segStart, const unsigned long long *hitOff, int32_t F,
                  const uint32_t *candCount, const uint32_t *candOff, const int32_t *stSeq, const int32_t *stStart,
                  const int32_t *stEnd, int32_t *cFrag, int32_t *cSeq, int32_t *cStart, int32_t *cEnd);

// synth.cu
void synth_genome(Ctx *ctx, uint64_t seed, uint32_t ancestor, uint32_t strain, uint32_t ppm,
                  int64_t len, uint8_t *hostOut);

inline unsigned nblk(uint64_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }    // blocks of t threads for n items

} // namespace bani
