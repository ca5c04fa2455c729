// capi.cu -- the extern "C" boundary declared in include/fastani_b200.h
#include "common.cuh"
#include <algorithm>
#include <cstring>
#include <cstdlib>

struct bani_ctx    { bani::Ctx c; };
struct bani_genome { bani::Genome g; };
struct bani_index  { bani::Index *ix; };
struct bani_qsketch { bani::QSketch *qs; };

namespace bani {
static thread_local std::string g_err;
void set_last_error(const std::string &m) { g_err = m; }
const char *const PATH_NAMES[NPATH] = {
  "l1.class0", "l1.class1", "l1.class2", "l1.class3", "l1.class4", "l1.class5", "l1.class6", "l1.class7", "l1.class8",
  "l1.class9", "l1.class10", "l1.class11", "l1.class12", "l1.device_wide",
  "lookup.walk_saturated", "lookup.walk_full_bucket",
  "l2.events_nt64", "l2.events_nt128", "l2.events_nt256", "l2.dir1024", "l2.dir4096", "l2.staged", "l2.direct",
  "l2.exact_at_bounds", "l2.exact_total",
  "piece.mapped", "piece.split_hits", "piece.split_events", "cgi.passes", "cgi.sparse"};
}

using namespace bani;

#define BANI_TRY try {
#define BANI_CATCH } catch (const bani::Error &e) { bani::set_last_error(e.what()); return e.code; } \
  catch (const std::bad_alloc &) { bani::set_last_error("host allocation failed"); return BANI_ERR_NOMEM; } \
  catch (const std::exception &e) { bani::set_last_error(e.what()); return BANI_ERR_INTERNAL; }

// a malloc'ed copy of v (nullptr when empty), for the caller to bani_free
template <typename T>
static T *host_copy(const std::vector<T> &v)
{
  if (v.empty()) return nullptr;
  T *p = (T *)malloc(sizeof(T) * v.size());
  if (!p) fail(BANI_ERR_NOMEM, "host allocation failed");
  memcpy(p, v.data(), sizeof(T) * v.size());
  return p;
}

static void map_cgi_sketch(bani_ctx *ctx, const bani_index *ix, const bani_qsketch *const *sketches, int32_t n_sketches, bool wantFrags,
                           MapOutput &mo)
{
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::vector<const QSketch *> qs(n_sketches);
  for (int i = 0; i < n_sketches; i++) { if (!sketches[i] || !sketches[i]->qs) fail(BANI_ERR_ARG, "null query sketch"); qs[i] = sketches[i]->qs; }
  qsketch_map(&ctx->c, ix->ix, qs.data(), n_sketches, false, true, mo, wantFrags);
}

extern "C" {

const char *bani_last_error(void) { return g_err.c_str(); }
const char *bani_version(void) { return "fastani_b200 0.1 (sm_90a)"; }

void bani_params_default(bani_params *p)
{
  // parseandSave defaults, src/map/include/parseCmdArgs.hpp:118-130
  memset(p, 0, sizeof *p);
  p->kmer_size = 16; p->window_size = 0; p->frag_len = 3000; p->perc_identity = 80.0f;
  p->p_value = 1e-3; p->reference_size = 5000000;
}

int bani_recommended_window_size(const bani_params *p)
{
  BANI_TRY
  if (!p || p->kmer_size < 1 || p->frag_len < 1) fail(BANI_ERR_ARG, "bad parameters");
  return stat_recommended_window_size(p->p_value, p->kmer_size, p->perc_identity, p->frag_len, p->reference_size);
  BANI_CATCH
}

int bani_stat_min_hits_relaxed(int s, int k, float pid)
{
  BANI_TRY
  if (s < 1 || k < 1) fail(BANI_ERR_ARG, "bad arguments");
  return stat_min_hits_relaxed(s, k, pid);
  BANI_CATCH
}

int bani_stat_identity(int shared, int s, int k, float *identity, float *upper)
{
  BANI_TRY
  if (s < 1 || k < 1 || shared < 0 || shared > s || !identity || !upper) fail(BANI_ERR_ARG, "bad arguments");
  stat_identity(shared, s, k, identity, upper);
  return BANI_OK;
  BANI_CATCH
}

int bani_device_count(int32_t *n)
{
  BANI_TRY
  if (!n) fail(BANI_ERR_ARG, "null argument");
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) { (void)cudaGetLastError(); c = 0; }
  *n = c;
  return BANI_OK;
  BANI_CATCH
}

int bani_ctx_create(int device, const bani_params *p, bani_ctx **out)
{
  BANI_TRY
  if (!p || !out) fail(BANI_ERR_ARG, "null argument");
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { (void)cudaGetLastError(); fail(BANI_ERR_CUDA, "no CUDA device available (this library has no CPU fallback)"); }
  if (device < 0 || device >= n) fail(BANI_ERR_ARG, "device %d out of range (%d devices)", device, n);
  BANI_CUDA(cudaSetDevice(device));
  std::unique_ptr<bani_ctx> c(new bani_ctx());
  c->c.device = device;
  c->c.prm = *p;
  if (c->c.prm.kmer_size < 1 || c->c.prm.kmer_size > 32) fail(BANI_ERR_LIMIT, "k-mer size %d outside [1, 32]", c->c.prm.kmer_size);
  if (c->c.prm.frag_len < 1) fail(BANI_ERR_ARG, "fragment length must be positive");
  if (c->c.prm.window_size <= 0)
    c->c.prm.window_size = stat_recommended_window_size(p->p_value, p->kmer_size, p->perc_identity, p->frag_len, p->reference_size);
  cudaDeviceProp prop;
  BANI_CUDA(cudaGetDeviceProperties(&prop, device));
  c->c.smCount = prop.multiProcessorCount;
  c->c.memTotal = prop.totalGlobalMem;
  {   // defaults of the run-time switches from the environment (see CtxFlags)
    CtxFlags &f = c->c.flags;
    if (getenv("BANI_NO_SKETCH_REUSE")) f.sketchReuse = 0;
    if (const char *e = getenv("BANI_MAX_HITS_PER_PIECE")) f.maxHitsPerPiece = std::max(1ll, atoll(e));
    if (const char *e = getenv("BANI_FRAG_L1_MAX")) f.fragL1Max = std::max(0ll, atoll(e));
    if (const char *e = getenv("BANI_L2_STAGE")) f.l2Stage = atoi(e) != 0;
    if (const char *e = getenv("BANI_TRACE")) f.trace = atoi(e) != 0;
    if (const char *e = getenv("BANI_L2E_BUCKETS")) { const int v = atoi(e); if (v == 1024 || v == 4096) f.l2eBuckets = v; }
    if (const char *e = getenv("BANI_CGI_SPARSE")) {
      const std::string v(e);
      if (v == "-1") f.cgiSparse = -1;
      else if (v == "0") f.cgiSparse = 0;
      else if (v == "1") f.cgiSparse = 1;
      else fail(BANI_ERR_ARG, "BANI_CGI_SPARSE=%s is not -1 (chosen per piece), 0 (dense) or 1 (sparse)", e);
    }
    uint64_t b = 0;
    if (const char *e = getenv("BANI_INDEX_BUDGET")) {
      if (!parse_byte_count(e, &b)) fail(BANI_ERR_ARG, "BANI_INDEX_BUDGET=%s is not a byte count (digits, optionally followed by K, M or G)", e);
      f.indexBytesBudget = b;
    }
    if (const char *e = getenv("BANI_QUERY_BUDGET")) {
      if (!parse_byte_count(e, &b)) fail(BANI_ERR_ARG, "BANI_QUERY_BUDGET=%s is not a byte count (digits, optionally followed by K, M or G)", e);
      f.querySketchBudget = b;
    }
  }
  dev_cache_flush(device);                   // blocks cached under streams of destroyed contexts
  BANI_CUDA(cudaStreamCreateWithFlags(&c->c.stream, cudaStreamNonBlocking));
  BANI_CUDA(cudaStreamCreateWithFlags(&c->c.copyStream, cudaStreamNonBlocking));
  *out = c.release();
  return BANI_OK;
  BANI_CATCH
}

void bani_ctx_destroy(bani_ctx *ctx)
{
  if (!ctx) return;
  cudaSetDevice(ctx->c.device);
  cudaStreamSynchronize(ctx->c.stream);
  ctx->c.d_minHits.release(); ctx->c.d_rowOff.release(); ctx->c.d_ident.release(); ctx->c.d_upper.release();
  ctx->c.slots.clear(); ctx->c.cubTemp.release();
  cudaStreamSynchronize(ctx->c.stream);
  cudaStreamSynchronize(ctx->c.copyStream);
  dev_cache_flush(ctx->c.device);            // blocks are keyed by stream: return them before it dies
  cudaStreamDestroy(ctx->c.stream);
  cudaStreamDestroy(ctx->c.copyStream);
  delete ctx;
}

int bani_ctx_params(const bani_ctx *ctx, bani_params *out)
{
  if (!ctx || !out) { set_last_error("null argument"); return BANI_ERR_ARG; }
  *out = ctx->c.prm; return BANI_OK;
}

int bani_ctx_sync(bani_ctx *ctx)
{
  BANI_TRY
  if (!ctx) fail(BANI_ERR_ARG, "null context");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  BANI_CUDA(cudaStreamSynchronize(ctx->c.copyStream));
  BANI_CUDA(cudaStreamSynchronize(ctx->c.stream));
  return BANI_OK;
  BANI_CATCH
}

int bani_ctx_set_flag(bani_ctx *ctx, const char *name, int64_t value)
{
  BANI_TRY
  if (!ctx || !name) fail(BANI_ERR_ARG, "null argument");
  CtxFlags &f = ctx->c.flags;
  const std::string n(name);
  if (n == "sketch_reuse") f.sketchReuse = value != 0;
  else if (n == "max_hits_per_piece") { if (value < 1) fail(BANI_ERR_ARG, "max_hits_per_piece must be positive"); f.maxHitsPerPiece = value; }
  else if (n == "frag_l1_max") { if (value < 0) fail(BANI_ERR_ARG, "frag_l1_max must not be negative"); f.fragL1Max = value; }
  else if (n == "l2e_buckets") { if (value != 0 && value != 1024 && value != 4096) fail(BANI_ERR_ARG, "l2e_buckets must be 0, 1024 or 4096"); f.l2eBuckets = (int)value; }
  else if (n == "l2_stage") f.l2Stage = value != 0;
  else if (n == "upload_group_words") { if (value < 1) fail(BANI_ERR_ARG, "upload_group_words must be positive"); f.uploadGroupWords = value; }
  else if (n == "frags_per_piece") { if (value < 1 || value > (1ll << 18)) fail(BANI_ERR_ARG, "frags_per_piece must be in [1, 2^18]"); f.fragsPerPiece = value; }
  else if (n == "event_bytes_per_piece") { if (value < 0) fail(BANI_ERR_ARG, "event_bytes_per_piece must not be negative"); f.eventBytesPerPiece = value; }
  else if (n == "cgi_table_queries") { if (value < 0) fail(BANI_ERR_ARG, "cgi_table_queries must not be negative"); f.cgiTableQueries = value; }
  else if (n == "l2_fast") f.l2Fast = value != 0;
  else if (n == "count_paths") f.countPaths = value != 0;
  else if (n == "cgi_sparse") { if (value < -1 || value > 1) fail(BANI_ERR_ARG, "cgi_sparse must be -1, 0 or 1"); f.cgiSparse = (int)value; }
  else if (n == "index_bytes_budget") { if (value < 0) fail(BANI_ERR_ARG, "index_bytes_budget must not be negative"); f.indexBytesBudget = (unsigned long long)value; }
  else if (n == "query_sketch_budget") { if (value < 0) fail(BANI_ERR_ARG, "query_sketch_budget must not be negative"); f.querySketchBudget = (unsigned long long)value; }
  else fail(BANI_ERR_ARG, "unknown flag '%s'", name);
  return BANI_OK;
  BANI_CATCH
}

int bani_ctx_path_counts(bani_ctx *ctx, char (*names)[32], uint64_t *counts, int32_t n_max, int32_t *n)
{
  BANI_TRY
  if (!ctx || !n || (n_max > 0 && (!names || !counts))) fail(BANI_ERR_ARG, "null argument");
  const int cnt = std::min<int>(n_max, NPATH);
  for (int i = 0; i < cnt; i++) { strncpy(names[i], PATH_NAMES[i], 31); names[i][31] = 0; counts[i] = ctx->c.paths[i]; }
  for (int i = 0; i < NPATH; i++) ctx->c.paths[i] = 0;
  *n = cnt;
  return BANI_OK;
  BANI_CATCH
}

int bani_ctx_profile_enable(bani_ctx *ctx, int on)
{
  if (!ctx) { set_last_error("null context"); return BANI_ERR_ARG; }
  ctx->c.profiling = on != 0;
  return BANI_OK;
}

int bani_ctx_profile_read(bani_ctx *ctx, char (*names)[32], double *ms, double *algo_bytes, int32_t *launches,
                          int32_t n_max, int32_t *n)
{
  BANI_TRY
  if (!ctx || !n) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  BANI_CUDA(cudaStreamSynchronize(ctx->c.stream));
  int cnt = 0;
  auto add = [&](const char *name, float t, double bytes) {
    int j = 0;
    for (; j < cnt; j++) if (strncmp(names[j], name, 31) == 0) break;
    if (j == cnt) {
      if (cnt >= n_max) return;
      strncpy(names[j], name, 31); names[j][31] = 0; ms[j] = 0; algo_bytes[j] = 0; launches[j] = 0; cnt++;
    }
    ms[j] += t; algo_bytes[j] += bytes; launches[j] += 1;
  };
  auto &evs = ctx->c.profEvents;
  for (size_t i = 0; i < evs.size(); i++) {
    float t = 0; cudaEventElapsedTime(&t, evs[i].a, evs[i].b);
    add(evs[i].name, t, evs[i].bytes);
    // device time between the end of the previous stage and the start of this one (kernels outside the stage timers,
    // memsets / copies, and idle time while the host decides what to launch next), filed under "gap>stage"
    if (i > 0) {
      float g = 0;
      if (cudaEventElapsedTime(&g, evs[i - 1].b, evs[i].a) == cudaSuccess && g > 0) {
        char nm[32]; snprintf(nm, sizeof nm, "gap>%s", evs[i].name);
        add(nm, g, 0.0);
      } else (void)cudaGetLastError();
    }
  }
  for (auto &e : evs) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
  evs.clear();
  *n = cnt;
  return BANI_OK;
  BANI_CATCH
}

uint64_t bani_ctx_launch_count(const bani_ctx *ctx) { return ctx ? ctx->c.launches : 0; }

int bani_ctx_mem_stats(bani_ctx *ctx, uint64_t *live, uint64_t *cached, uint64_t *peak_live)
{
  BANI_TRY
  if (!ctx) fail(BANI_ERR_ARG, "null context");
  size_t l = 0, c = 0, p = 0;
  dev_mem_stats(ctx->c.device, &l, &c, &p);
  dev_mem_peak_set(ctx->c.device, 0);
  if (live) *live = l;
  if (cached) *cached = c;
  if (peak_live) *peak_live = p;
  return BANI_OK;
  BANI_CATCH
}

int bani_ctx_trim(bani_ctx *ctx)
{
  BANI_TRY
  if (!ctx) fail(BANI_ERR_ARG, "null context");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  BANI_CUDA(cudaStreamSynchronize(ctx->c.stream));
  ctx->c.slots.clear(); ctx->c.cubTemp.release();
  dev_cache_flush(ctx->c.device);
  return BANI_OK;
  BANI_CATCH
}

static int plan_run_checked(const RunSize &r, const uint64_t *ref_len, const int32_t *ref_contigs, int32_t n_refs, const uint64_t *query_len,
                            const uint64_t *query_sketch_bytes, int32_t n_queries, int32_t *chunk_end, int32_t *n_chunks, int32_t *block_end,
                            int32_t *n_blocks, uint64_t *index_budget)
{
  if (n_refs < 0 || n_queries < 0 || (n_refs && (!ref_len || !ref_contigs || !chunk_end)) || (n_queries && (!query_len || !block_end)) ||
      !n_chunks || !n_blocks || r.k < 1 || r.w < 1 || r.fragLen < 1)
    fail(BANI_ERR_ARG, "bad argument");
  uint64_t ib = 0;
  const int32_t nc = plan_run(r, ref_len, ref_contigs, n_refs, query_len, query_sketch_bytes, n_queries, chunk_end, block_end, n_blocks, &ib);
  if (nc < 0)
    fail(BANI_ERR_LIMIT, "reference genome %d (%llu bases) alone does not fit the index budget of %llu bytes", -nc - 1,
         (unsigned long long)ref_len[-nc - 1], (unsigned long long)ib);
  *n_chunks = nc;
  if (index_budget) *index_budget = ib;
  return BANI_OK;
}

int bani_plan_run(uint64_t free_bytes, uint64_t device_bytes, int64_t max_hits_per_piece, int64_t event_bytes_per_piece,
                  uint64_t index_budget, uint64_t query_budget, int32_t k, int32_t w, int32_t frag_len,
                  const uint64_t *ref_len, const int32_t *ref_contigs, int32_t n_refs, const uint64_t *query_len,
                  const uint64_t *query_sketch_bytes, int32_t n_queries, int32_t *chunk_end, int32_t *n_chunks,
                  int32_t *block_end, int32_t *n_blocks, uint64_t *index_budget_used)
{
  BANI_TRY
  RunSize r;
  r.freeBytes = free_bytes; r.deviceBytes = device_bytes; r.maxHitsPerPiece = max_hits_per_piece; r.eventBytesPerPiece = event_bytes_per_piece;
  r.indexBudget = index_budget; r.queryBudget = query_budget; r.k = k; r.w = w; r.fragLen = frag_len;
  return plan_run_checked(r, ref_len, ref_contigs, n_refs, query_len, query_sketch_bytes, n_queries, chunk_end, n_chunks, block_end, n_blocks,
                          index_budget_used);
  BANI_CATCH
}

int bani_ctx_plan_run(bani_ctx *ctx, uint64_t index_budget, uint64_t query_budget, const uint64_t *ref_len, const int32_t *ref_contigs, int32_t n_refs, const uint64_t *query_len,
                      const uint64_t *query_sketch_bytes, int32_t n_queries, int32_t *chunk_end, int32_t *n_chunks,
                      int32_t *block_end, int32_t *n_blocks, uint64_t *index_budget_used)
{
  BANI_TRY
  if (!ctx) fail(BANI_ERR_ARG, "null context");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  size_t freeB = 0, totalB = 0, cached = 0;
  BANI_CUDA(cudaMemGetInfo(&freeB, &totalB));
  dev_mem_stats(ctx->c.device, nullptr, &cached, nullptr);
  const CtxFlags &f = ctx->c.flags;
  RunSize r;
  r.freeBytes = (uint64_t)freeB + (uint64_t)cached;                  // cached blocks go back to the driver on demand
  r.deviceBytes = ctx->c.memTotal; r.maxHitsPerPiece = f.maxHitsPerPiece; r.eventBytesPerPiece = f.eventBytesPerPiece;
  r.indexBudget = index_budget ? index_budget : f.indexBytesBudget; r.queryBudget = query_budget ? query_budget : f.querySketchBudget;
  r.k = ctx->c.prm.kmer_size; r.w = ctx->c.prm.window_size; r.fragLen = ctx->c.prm.frag_len;
  return plan_run_checked(r, ref_len, ref_contigs, n_refs, query_len, query_sketch_bytes, n_queries, chunk_end, n_chunks, block_end, n_blocks,
                          index_budget_used);
  BANI_CATCH
}

int bani_index_footprint(uint64_t n_minimizers, uint64_t n_unique_bound, uint64_t n_contigs, uint64_t bitmap_bits, uint64_t staging_cap,
                         uint64_t *build_peak, uint64_t *resident)
{
  BANI_TRY
  if (n_unique_bound > n_minimizers) fail(BANI_ERR_ARG, "more unique hashes than minimizers");
  const IndexFootprint f = index_footprint(n_minimizers, n_unique_bound, n_contigs, bitmap_bits, staging_cap);
  if (build_peak) *build_peak = f.peak;
  if (resident) *resident = f.resident;
  return BANI_OK;
  BANI_CATCH
}

int bani_map_working_set(uint64_t device_bytes, int64_t max_hits_per_piece, int64_t event_bytes_per_piece, uint64_t *bytes)
{
  BANI_TRY
  if (!bytes) fail(BANI_ERR_ARG, "null argument");
  *bytes = map_working_set(device_bytes, max_hits_per_piece, event_bytes_per_piece);
  return BANI_OK;
  BANI_CATCH
}

int bani_run_working_set(uint64_t device_bytes, int64_t max_hits_per_piece, int64_t event_bytes_per_piece, uint64_t query_hashes,
                         uint64_t query_fragments, int32_t n_queries, uint64_t ref_bases, int32_t n_refs, int32_t window_size,
                         int32_t frag_len, uint64_t *bytes)
{
  BANI_TRY
  if (!bytes || n_queries < 0 || n_refs < 0 || window_size < 1 || frag_len < 1) fail(BANI_ERR_ARG, "bad argument");
  *bytes = map_working_set_run(device_bytes, max_hits_per_piece, event_bytes_per_piece, query_hashes, query_fragments, (uint64_t)n_queries,
                               ref_bases, (uint64_t)n_refs, window_size, frag_len);
  return BANI_OK;
  BANI_CATCH
}

int bani_index_budget(uint64_t free_bytes, uint64_t query_sketch_bytes, uint64_t working_set, int32_t window_size, uint64_t *budget)
{
  BANI_TRY
  if (!budget || window_size < 1) fail(BANI_ERR_ARG, "bad argument");
  *budget = index_budget(free_bytes, query_sketch_bytes, working_set, window_size);
  return BANI_OK;
  BANI_CATCH
}

int bani_plan_chunks(const uint64_t *genome_len, const int32_t *genome_contigs, int32_t n, int32_t k, int32_t w, uint64_t budget,
                     int32_t *chunk_end, int32_t *n_chunks)
{
  BANI_TRY
  if (n < 0 || (n && (!genome_len || !genome_contigs || !chunk_end)) || !n_chunks || k < 1 || w < 1) fail(BANI_ERR_ARG, "bad argument");
  const int32_t r = plan_chunks(genome_len, genome_contigs, n, k, w, budget, chunk_end);
  if (r < 0) {
    const int32_t g = -r - 1;
    fail(BANI_ERR_LIMIT, "reference genome %d (%llu bases) alone does not fit the index budget of %llu bytes", g,
         (unsigned long long)genome_len[g], (unsigned long long)budget);
  }
  *n_chunks = r;
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_bytes_estimate(uint64_t len, int32_t w, int32_t frag_len, uint64_t *bytes)
{
  BANI_TRY
  if (!bytes || w < 1) fail(BANI_ERR_ARG, "bad argument");
  *bytes = qsketch_bytes_estimate(len, w, frag_len);
  return BANI_OK;
  BANI_CATCH
}

int bani_parse_byte_count(const char *s, uint64_t *out)
{
  BANI_TRY
  if (!out) fail(BANI_ERR_ARG, "null argument");
  if (!parse_byte_count(s, out)) fail(BANI_ERR_ARG, "'%s' is not a byte count (digits, optionally followed by K, M or G)", s ? s : "");
  return BANI_OK;
  BANI_CATCH
}

void *bani_ctx_stream(bani_ctx *ctx) { return ctx ? (void *)ctx->c.stream : nullptr; }

int bani_host_alloc(size_t bytes, void **out)
{
  BANI_TRY
  if (!out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return BANI_OK;
  BANI_CATCH
}
void bani_host_free(void *p) { if (p) cudaFreeHost(p); }

int bani_genome_create_batch(bani_ctx *ctx, int32_t n_genomes, const int32_t *gen_off, const int64_t *off,
                             const uint8_t *seq, bani_genome **out)
{
  BANI_TRY
  if (!ctx || !out || n_genomes < 0 || (n_genomes && (!gen_off || !off))) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  for (int g = 0; g < n_genomes; g++) {
    if (gen_off[g + 1] < gen_off[g]) fail(BANI_ERR_ARG, "genome offsets must ascend");
    for (int c = gen_off[g]; c < gen_off[g + 1]; c++) if (off[c + 1] < off[c]) fail(BANI_ERR_ARG, "contig offsets must ascend");
  }
  if (n_genomes && off[gen_off[n_genomes]] > off[gen_off[0]] && !seq) fail(BANI_ERR_ARG, "null sequence buffer");
  std::vector<Genome *> gs(n_genomes, nullptr);
  genome_create_batch(&ctx->c, n_genomes, gen_off, off, seq, gs.data());
  for (int g = 0; g < n_genomes; g++) {
    // bani_genome is a thin wrapper so that the handle type stays opaque in C
    bani_genome *h = new bani_genome();
    h->g = std::move(*gs[g]);
    delete gs[g];
    out[g] = h;
  }
  return BANI_OK;
  BANI_CATCH
}

int bani_pack_contig(const uint8_t *seq, int64_t len, uint32_t *words, uint32_t *exc_pos, uint8_t *exc_byte, uint64_t exc_cap, uint64_t *n_exc)
{
  BANI_TRY
  if (len < 0 || len > 0x7fffffff || (len && (!seq || !words)) || !n_exc || (exc_cap && (!exc_pos || !exc_byte))) fail(BANI_ERR_ARG, "bad argument");
  *n_exc = host_pack_contig(seq, len, words, exc_pos, exc_byte, exc_cap);
  return BANI_OK;
  BANI_CATCH
}

int bani_genome_create_packed_batch(bani_ctx *ctx, int32_t n_genomes, const int32_t *gen_off, const int32_t *contig_len, const int64_t *word_off,
                                    const uint32_t *words, const int64_t *exc_off, const uint32_t *exc_pos, const uint8_t *exc_byte,
                                    int32_t async, bani_genome **out)
{
  BANI_TRY
  if (!ctx || !out || n_genomes < 0 || (n_genomes && (!gen_off || !contig_len || !word_off || !exc_off))) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  for (int g = 0; g < n_genomes; g++) if (gen_off[g + 1] < gen_off[g]) fail(BANI_ERR_ARG, "genome offsets must ascend");
  if (n_genomes) {
    const int32_t c0 = gen_off[0], c1 = gen_off[n_genomes];
    bool anyBases = false;
    for (int32_t c = c0; c < c1; c++) anyBases |= contig_len[c] > 0;
    if (anyBases && !words) fail(BANI_ERR_ARG, "null packed buffer");
    if (exc_off[c1] > exc_off[c0] && (!exc_pos || !exc_byte)) fail(BANI_ERR_ARG, "null exception arrays");
  }
  std::vector<Genome *> gs(n_genomes, nullptr);
  genome_create_packed_batch(&ctx->c, n_genomes, gen_off, contig_len, word_off, words, exc_off, exc_pos, exc_byte, async != 0, gs.data());
  for (int g = 0; g < n_genomes; g++) { bani_genome *h = new bani_genome(); h->g = std::move(*gs[g]); delete gs[g]; out[g] = h; }
  return BANI_OK;
  BANI_CATCH
}

int bani_genome_create(bani_ctx *ctx, int32_t n_contigs, const int64_t *off, const uint8_t *seq, bani_genome **out)
{
  int32_t go[2] = {0, n_contigs};
  if (n_contigs < 0) { set_last_error("negative contig count"); return BANI_ERR_ARG; }
  int64_t zero[1] = {0};
  return bani_genome_create_batch(ctx, 1, go, n_contigs ? off : zero, seq, out);
}

void bani_genome_destroy(bani_genome *g)
{
  if (!g) return;
  cudaSetDevice(g->g.device);
  delete g;
}

int bani_genome_info(const bani_genome *g, int32_t *n_contigs, uint64_t *total_len, uint64_t *n_exceptions, uint64_t *n_fragments)
{
  if (!g) { set_last_error("null genome"); return BANI_ERR_ARG; }
  if (n_contigs) *n_contigs = g->g.nContigs;
  if (total_len) *total_len = g->g.totalLen;
  if (n_exceptions) *n_exceptions = g->g.nExc;
  if (n_fragments) *n_fragments = 0;
  return BANI_OK;
}

int bani_genome_decode(bani_ctx *ctx, const bani_genome *g, int32_t contig, uint8_t *out, int64_t cap)
{
  BANI_TRY
  if (!ctx || !g || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  genome_decode(&ctx->c, &g->g, contig, out, cap);
  return BANI_OK;
  BANI_CATCH
}

int bani_index_build(bani_ctx *ctx, bani_genome *const *refs, int32_t n_refs, bani_index **out)
{
  BANI_TRY
  if (!ctx || !out || n_refs < 0 || (n_refs && !refs)) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  ctx->c.mark("index_build: called");
  std::vector<Genome *> gs(n_refs);
  for (int i = 0; i < n_refs; i++) { if (!refs[i]) fail(BANI_ERR_ARG, "null genome handle"); gs[i] = &refs[i]->g; }
  Index *ix = index_build(&ctx->c, gs.data(), n_refs);
  bani_index *h = new bani_index(); h->ix = ix; *out = h;
  return BANI_OK;
  BANI_CATCH
}

int bani_index_build_budget(bani_ctx *ctx, bani_genome *const *refs, int32_t n_refs, uint64_t max_bytes, bani_index **out,
                            int32_t *n_taken, uint64_t *peak_bytes)
{
  BANI_TRY
  if (!ctx || !out || !n_taken || n_refs < 1 || !refs) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::vector<Genome *> gs(n_refs);
  for (int i = 0; i < n_refs; i++) { if (!refs[i]) fail(BANI_ERR_ARG, "null genome handle"); gs[i] = &refs[i]->g; }
  int32_t taken = 0; uint64_t peak = 0;
  Index *ix = index_build_budget(&ctx->c, gs.data(), n_refs, max_bytes, &taken, &peak);
  bani_index *h = new bani_index(); h->ix = ix; *out = h;
  *n_taken = taken;
  if (peak_bytes) *peak_bytes = peak;
  return BANI_OK;
  BANI_CATCH
}

void bani_index_destroy(bani_index *ix)
{
  if (!ix) return;
  if (ix->ix) { cudaSetDevice(ix->ix->device); delete ix->ix; }
  delete ix;
}

int bani_index_stats(const bani_index *ix, uint64_t *n_minimizers, uint64_t *n_unique, uint64_t *total_len,
                     uint64_t *n_contigs, uint64_t *n_genomes)
{
  if (!ix || !ix->ix) { set_last_error("null index"); return BANI_ERR_ARG; }
  if (n_minimizers) *n_minimizers = ix->ix->M;
  if (n_unique) *n_unique = ix->ix->U;
  if (total_len) *total_len = ix->ix->totalLen;
  if (n_contigs) *n_contigs = (uint64_t)ix->ix->nContigs;
  if (n_genomes) *n_genomes = (uint64_t)ix->ix->nGenomes;
  return BANI_OK;
}

int bani_index_save(bani_ctx *ctx, const bani_index *ix, const char *path)
{
  BANI_TRY
  if (!ctx || !ix || !ix->ix || !path) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  index_save(&ctx->c, ix->ix, path);
  return BANI_OK;
  BANI_CATCH
}

int bani_index_load(bani_ctx *ctx, const char *path, bani_index **out)
{
  BANI_TRY
  if (!ctx || !path || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  Index *ix = index_load(&ctx->c, path);
  bani_index *h = new bani_index(); h->ix = ix; *out = h;
  return BANI_OK;
  BANI_CATCH
}

int bani_index_file_info(const char *path, int32_t *version, int32_t *k, int32_t *w, int32_t *frag_len, int32_t *n_genomes,
                         uint64_t *n_contigs, uint64_t *n_minimizers, int32_t *genome_contigs, uint64_t *genome_len, uint64_t *genome_records,
                         uint64_t *genome_bits, uint64_t cap_genomes, int32_t *contig_len, uint64_t cap_contigs)
{
  BANI_TRY
  if (!path) fail(BANI_ERR_ARG, "null path");
  const IndexFileInfo x = index_file_info(path);
  const uint64_t nG = x.nGenomes, nC = x.nContigs;
  if ((genome_contigs || genome_len || genome_records || genome_bits) && cap_genomes < nG) fail(BANI_ERR_ARG, "genome buffer too small");
  if (contig_len && cap_contigs < nC) fail(BANI_ERR_ARG, "contig buffer too small");
  for (uint64_t g = 0; g < nG; g++) {
    const uint64_t c0 = x.contig_begin((int32_t)g), c1 = (uint64_t)x.seqsByFile[g];
    uint64_t len = 0;
    for (uint64_t c = c0; c < c1; c++) len += (uint64_t)x.contigLen[c];
    if (genome_contigs) genome_contigs[g] = (int32_t)(c1 - c0);
    if (genome_len) genome_len[g] = len;
    if (genome_records) genome_records[g] = x.recOff[c1] - x.recOff[c0];
    if (genome_bits) genome_bits[g] = x.bitOff[c1] - x.bitOff[c0];
  }
  if (contig_len && nC) memcpy(contig_len, x.contigLen.data(), 4 * nC);
  if (version) *version = x.version;
  if (k) *k = x.k;
  if (w) *w = x.w;
  if (frag_len) *frag_len = x.fragLen;
  if (n_genomes) *n_genomes = (int32_t)nG;
  if (n_contigs) *n_contigs = nC;
  if (n_minimizers) *n_minimizers = x.M;
  return BANI_OK;
  BANI_CATCH
}

int bani_index_load_budget(bani_ctx *ctx, const char *path, int32_t first_genome, uint64_t max_bytes, bani_index **out, int32_t *n_taken,
                           uint64_t *peak_bytes)
{
  BANI_TRY
  if (!ctx || !path || !out || !n_taken) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  int32_t taken = 0; uint64_t peak = 0;
  Index *ix = index_load_budget(&ctx->c, path, first_genome, max_bytes, &taken, &peak);
  bani_index *h = new bani_index(); h->ix = ix; *out = h;
  *n_taken = taken;
  if (peak_bytes) *peak_bytes = peak;
  return BANI_OK;
  BANI_CATCH
}

int bani_index_file_extend(bani_ctx *ctx, const char *in_path, const bani_index *added, const char *out_path)
{
  BANI_TRY
  if (!ctx || !in_path || !added || !added->ix || !out_path) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  index_file_extend(&ctx->c, in_path, added->ix, out_path);
  return BANI_OK;
  BANI_CATCH
}

int bani_index_contigs(const bani_index *ix, int32_t *contig_len, uint64_t cap_contigs, int32_t *seqs_by_file, uint64_t cap_genomes)
{
  BANI_TRY
  if (!ix || !ix->ix) fail(BANI_ERR_ARG, "null index");
  const Index *x = ix->ix;
  if (contig_len) { if (cap_contigs < x->contigLen.size()) fail(BANI_ERR_ARG, "contig buffer too small"); memcpy(contig_len, x->contigLen.data(), 4 * x->contigLen.size()); }
  if (seqs_by_file) { if (cap_genomes < x->seqsByFile.size()) fail(BANI_ERR_ARG, "genome buffer too small"); memcpy(seqs_by_file, x->seqsByFile.data(), 4 * x->seqsByFile.size()); }
  return BANI_OK;
  BANI_CATCH
}

int bani_index_minimizers(bani_ctx *ctx, const bani_index *ixh, bani_minimizer *out, uint64_t cap)
{
  BANI_TRY
  if (!ctx || !ixh || !ixh->ix || (!out && cap)) fail(BANI_ERR_ARG, "null argument");
  const Index *ix = ixh->ix;
  if (cap < ix->M) fail(BANI_ERR_ARG, "output buffer too small (%llu < %llu)", (unsigned long long)cap, (unsigned long long)ix->M);
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  const size_t M = ix->M;
  if (!M) return BANI_OK;
  std::vector<uint32_t> h(M); std::vector<int32_t> s(M), w(M);
  BANI_CUDA(cudaStreamSynchronize(ctx->c.stream));
  BANI_CUDA(cudaMemcpy(h.data(), ix->hash.p, 4 * M, cudaMemcpyDeviceToHost));
  BANI_CUDA(cudaMemcpy(s.data(), ix->seqId.p, 4 * M, cudaMemcpyDeviceToHost));
  BANI_CUDA(cudaMemcpy(w.data(), ix->wpos.p, 4 * M, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < M; i++) { out[i].hash = h[i]; out[i].seqId = s[i]; out[i].wpos = w[i]; }
  return BANI_OK;
  BANI_CATCH
}

int bani_index_lookup(bani_ctx *ctx, const bani_index *ixh, uint32_t hash, int32_t *seqId, int32_t *wpos, uint64_t cap, uint64_t *n)
{
  BANI_TRY
  if (!ctx || !ixh || !ixh->ix || !n) fail(BANI_ERR_ARG, "null argument");
  const Index *ix = ixh->ix;
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  BANI_CUDA(cudaStreamSynchronize(ctx->c.stream));
  *n = 0;
  if (!ix->U) return BANI_OK;
  // host-driven probe of the device structures (test hook; the mapping kernels do this on the device)
  const uint32_t b = hash >> (32 - ix->dirBits);
  uint32_t d[2];
  BANI_CUDA(cudaMemcpy(d, ix->dir.p + b, 8, cudaMemcpyDeviceToHost));
  if (d[1] <= d[0]) return BANI_OK;
  std::vector<uint32_t> keys(d[1] - d[0]);
  BANI_CUDA(cudaMemcpy(keys.data(), ix->ukeys.p + d[0], 4 * keys.size(), cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < keys.size(); i++) if (keys[i] == hash) {
    uint32_t o[2];
    BANI_CUDA(cudaMemcpy(o, ix->uoff.p + d[0] + i, 8, cudaMemcpyDeviceToHost));
    const uint64_t cnt = o[1] - o[0];
    *n = cnt;
    const uint64_t m = cnt < cap ? cnt : cap;
    std::vector<uint32_t> pi(m);
    if (m) BANI_CUDA(cudaMemcpy(pi.data(), ix->posIdx.p + o[0], 4 * m, cudaMemcpyDeviceToHost));
    for (uint64_t j = 0; j < m; j++) {
      BANI_CUDA(cudaMemcpy(&seqId[j], ix->seqId.p + pi[j], 4, cudaMemcpyDeviceToHost));
      BANI_CUDA(cudaMemcpy(&wpos[j], ix->wpos.p + pi[j], 4, cudaMemcpyDeviceToHost));
    }
    break;
  }
  return BANI_OK;
  BANI_CATCH
}

int bani_map_genome(bani_ctx *ctx, const bani_index *ix, const bani_genome *query, bani_mapping **rows, uint64_t *n_rows,
                    uint64_t *total_query_fragments, bani_map_counters *counters)
{
  BANI_TRY
  if (!ctx || !ix || !ix->ix || !query || !rows || !n_rows) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  MapOutput mo;
  const Genome *q = &query->g;
  map_queries(&ctx->c, ix->ix, &q, 1, true, false, mo);
  *n_rows = mo.rows.size();
  *rows = nullptr;
  if (!mo.rows.empty()) {
    *rows = (bani_mapping *)malloc(sizeof(bani_mapping) * mo.rows.size());
    if (!*rows) fail(BANI_ERR_NOMEM, "host allocation failed");
    memcpy(*rows, mo.rows.data(), sizeof(bani_mapping) * mo.rows.size());
  }
  if (total_query_fragments) *total_query_fragments = mo.totalQueryFragments[0];
  if (counters) *counters = mo.ctr;
  return BANI_OK;
  BANI_CATCH
}

int bani_map_cgi(bani_ctx *ctx, const bani_index *ix, bani_genome *const *queries, int32_t n_queries,
                 bani_cgi_result **results, uint64_t *n_results, uint64_t *total_query_fragments, bani_map_counters *counters)
{
  BANI_TRY
  if (!ctx || !ix || !ix->ix || n_queries < 0 || (n_queries && !queries) || !results || !n_results) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::vector<const Genome *> qs(n_queries);
  for (int i = 0; i < n_queries; i++) { if (!queries[i]) fail(BANI_ERR_ARG, "null genome handle"); qs[i] = &queries[i]->g; }
  MapOutput mo;
  ctx->c.mark("map_cgi: enter");
  map_queries(&ctx->c, ix->ix, qs.data(), n_queries, false, true, mo);
  ctx->c.mark("map_cgi: map_queries returned");
  *n_results = mo.cgi.size();
  *results = nullptr;
  if (!mo.cgi.empty()) {
    *results = (bani_cgi_result *)malloc(sizeof(bani_cgi_result) * mo.cgi.size());
    if (!*results) fail(BANI_ERR_NOMEM, "host allocation failed");
    memcpy(*results, mo.cgi.data(), sizeof(bani_cgi_result) * mo.cgi.size());
  }
  if (total_query_fragments) for (int i = 0; i < n_queries; i++) total_query_fragments[i] = mo.totalQueryFragments[i];
  if (counters) *counters = mo.ctr;
  ctx->c.mark("map_cgi: results copied");
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_create(bani_ctx *ctx, bani_genome *const *queries, int32_t n_queries, const int32_t *query_ids,
                        const bani_index *hint, bani_qsketch **out)
{
  BANI_TRY
  if (!ctx || n_queries < 0 || (n_queries && !queries) || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::vector<const Genome *> qs(n_queries);
  for (int i = 0; i < n_queries; i++) { if (!queries[i]) fail(BANI_ERR_ARG, "null genome handle"); qs[i] = &queries[i]->g; }
  std::unique_ptr<bani_qsketch> h(new bani_qsketch());
  h->qs = qsketch_create(&ctx->c, qs.data(), n_queries, query_ids, hint ? hint->ix : nullptr);
  *out = h.release();
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_from_index(bani_ctx *ctx, const bani_index *ix, const int32_t *genome_ordinals, int32_t n_queries,
                            const int32_t *query_ids, bani_qsketch **out)
{
  BANI_TRY
  if (!ctx || !ix || !ix->ix || n_queries < 0 || (n_queries && !genome_ordinals) || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::unique_ptr<bani_qsketch> h(new bani_qsketch());
  h->qs = qsketch_from_index(&ctx->c, ix->ix, genome_ordinals, n_queries, query_ids);
  *out = h.release();
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_from_index_file(bani_ctx *ctx, const char *path, const int32_t *genome_ordinals, int32_t n_queries,
                                 const int32_t *query_ids, bani_qsketch **out)
{
  BANI_TRY
  if (!ctx || !path || n_queries < 0 || (n_queries && !genome_ordinals) || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::unique_ptr<bani_qsketch> h(new bani_qsketch());
  h->qs = qsketch_from_index_file(&ctx->c, path, genome_ordinals, n_queries, query_ids);
  *out = h.release();
  return BANI_OK;
  BANI_CATCH
}

void bani_qsketch_destroy(bani_qsketch *qs)
{
  if (!qs) return;
  if (qs->qs) { cudaSetDevice(qs->qs->device); delete qs->qs; }
  delete qs;
}

int bani_qsketch_info(const bani_qsketch *qs, int32_t *n_queries, uint64_t *n_fragments, uint64_t *n_hashes, uint64_t *export_bytes)
{
  BANI_TRY
  if (!qs || !qs->qs) fail(BANI_ERR_ARG, "null argument");
  if (n_queries) *n_queries = (int32_t)qs->qs->queryId.size();
  if (n_fragments) *n_fragments = qs->qs->F;
  if (n_hashes) *n_hashes = qs->qs->T;
  if (export_bytes) *export_bytes = qsketch_export_bytes(qs->qs);
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_export(bani_ctx *ctx, const bani_qsketch *qs, void *device_buf, uint64_t cap)
{
  BANI_TRY
  if (!ctx || !qs || !qs->qs || !device_buf) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  qsketch_export(&ctx->c, qs->qs, device_buf, cap);
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_import(bani_ctx *ctx, const void *device_buf, uint64_t bytes, bani_qsketch **out)
{
  BANI_TRY
  if (!ctx || !device_buf || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::unique_ptr<bani_qsketch> h(new bani_qsketch());
  h->qs = qsketch_import(&ctx->c, device_buf, bytes);
  *out = h.release();
  return BANI_OK;
  BANI_CATCH
}

int bani_qsketch_merge(bani_ctx *ctx, const bani_qsketch *const *sketches, int32_t n_sketches, bani_qsketch **out)
{
  BANI_TRY
  if (!ctx || n_sketches < 0 || (n_sketches && !sketches) || !out) fail(BANI_ERR_ARG, "null argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  std::vector<const QSketch *> qs(n_sketches);
  for (int i = 0; i < n_sketches; i++) { if (!sketches[i] || !sketches[i]->qs) fail(BANI_ERR_ARG, "null query sketch"); qs[i] = sketches[i]->qs; }
  std::unique_ptr<bani_qsketch> h(new bani_qsketch());
  h->qs = qsketch_merge(&ctx->c, qs.data(), n_sketches);
  *out = h.release();
  return BANI_OK;
  BANI_CATCH
}

int bani_map_cgi_sketch(bani_ctx *ctx, const bani_index *ix, const bani_qsketch *const *sketches, int32_t n_sketches,
                        bani_cgi_result **results, uint64_t *n_results, bani_map_counters *counters)
{
  BANI_TRY
  if (!ctx || !ix || !ix->ix || n_sketches < 0 || (n_sketches && !sketches) || !results || !n_results) fail(BANI_ERR_ARG, "null argument");
  MapOutput mo;
  map_cgi_sketch(ctx, ix, sketches, n_sketches, false, mo);
  *results = host_copy(mo.cgi);
  *n_results = mo.cgi.size();
  if (counters) *counters = mo.ctr;
  return BANI_OK;
  BANI_CATCH
}

int bani_map_cgi_sketch_frags(bani_ctx *ctx, const bani_index *ix, const bani_qsketch *const *sketches, int32_t n_sketches,
                              bani_cgi_result **results, uint64_t *n_results, bani_frag_mapping **frags, uint64_t *n_frags,
                              bani_map_counters *counters)
{
  BANI_TRY
  if (!ctx || !ix || !ix->ix || n_sketches < 0 || (n_sketches && !sketches) || !results || !n_results || !frags || !n_frags)
    fail(BANI_ERR_ARG, "null argument");
  MapOutput mo;
  map_cgi_sketch(ctx, ix, sketches, n_sketches, true, mo);
  std::unique_ptr<bani_cgi_result, void (*)(void *)> res(host_copy(mo.cgi), free);
  *frags = host_copy(mo.frags);
  *n_frags = mo.frags.size();
  *results = res.release();
  *n_results = mo.cgi.size();
  if (counters) *counters = mo.ctr;
  return BANI_OK;
  BANI_CATCH
}

void bani_free(void *p) { free(p); }

int bani_synth_genome(bani_ctx *ctx, uint64_t seed, uint32_t ancestor_id, uint32_t strain_id, uint32_t sub_rate_ppm,
                      int64_t len, uint8_t *host_out)
{
  BANI_TRY
  if (!ctx || (len > 0 && !host_out) || len < 0) fail(BANI_ERR_ARG, "bad argument");
  BANI_CUDA(cudaSetDevice(ctx->c.device));
  synth_genome(&ctx->c, seed, ancestor_id, strain_id, sub_rate_ppm, len, host_out);
  return BANI_OK;
  BANI_CATCH
}

} // extern "C"
