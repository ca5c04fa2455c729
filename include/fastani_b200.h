/* fastani_b200.h -- C ABI of the H100-native ANI hot path.
 *
 * This is the drop-in boundary for the two data-parallel hot paths of FastANI
 * (reference citations are relative to the upstream tree, ParBLiSS/FastANI):
 *
 *   HP1  reference index build   skch::Sketch::Sketch(const Parameters&)
 *                                 src/map/include/winSketch.hpp:109-115
 *   HP2  query mapping           skch::Map::Map(const Parameters&, const Sketch&,
 *                                 uint64_t& totalQueryFragments, int queryno, callback)
 *                                 src/map/include/computeMap.hpp:93-102
 *   (+)  per-pair reduction      cgi::computeCGI
 *                                 src/cgi/include/computeCoreIdentity.hpp:166-298
 *
 * The reference has no FFI layer; its seam is those two constructors and one
 * callback.  The entry points below are what a binding for that seam needs:
 * plain pointers and sizes, no C++ or torch types.  All device work runs on the
 * CUDA device the context was created on (sm_90a kernels); there is NO CPU
 * fallback -- every call fails with BANI_ERR_CUDA if no device is usable.
 *
 * Conventions: every function returns 0 (BANI_OK) or a negative bani_status;
 * bani_last_error() gives a thread-local message for the last failure.  The
 * library allocates outputs; the caller frees them through the library.
 * Handles are not thread-safe individually; distinct contexts may be used from
 * distinct threads concurrently.
 */
#ifndef FASTANI_B200_H
#define FASTANI_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BANI_API __attribute__((visibility("default")))

typedef enum {
  BANI_OK = 0,
  BANI_ERR_ARG = -1,       /* invalid argument */
  BANI_ERR_CUDA = -2,      /* CUDA runtime failure / no usable device */
  BANI_ERR_NOMEM = -3,     /* host or device allocation failed */
  BANI_ERR_LIMIT = -4,     /* an implementation limit was exceeded (message says which) */
  BANI_ERR_INTERNAL = -5
} bani_status;

/* skch::Parameters, src/map/include/map_parameters.hpp:22-41 -- the fields the
 * hot path reads.  Zero-initialise, then call bani_params_default(). */
typedef struct {
  int32_t  kmer_size;          /* kmerSize            (default 16) */
  int32_t  window_size;        /* windowSize; <=0 => Stat::recommendedWindowSize */
  int32_t  frag_len;           /* minReadLength       (default 3000) */
  float    perc_identity;      /* percentageIdentity  (default 80) */
  double   p_value;            /* p_value             (default 1e-3) */
  uint64_t reference_size;     /* referenceSize       (default 5000000) */
  int32_t  reserved[8];
} bani_params;

/* skch::MappingResult, src/map/include/base_types.hpp:89-102 (44 bytes, same field order) */
typedef struct {
  int32_t queryLen, refStartPos, refEndPos, queryStartPos, queryEndPos;
  int32_t refSeqId, querySeqId;
  float   nucIdentity, nucIdentityUpperBound;
  int32_t sketchSize, conservedSketches;
} bani_mapping;

/* skch::MinimizerInfo, src/map/include/base_types.hpp:21-53 (12 bytes) */
typedef struct { uint32_t hash; int32_t seqId; int32_t wpos; } bani_minimizer;

/* cgi::CGI_Results, src/cgi/include/cgid_types.hpp:68-80.  refGenomeId is the
 * ordinal of the genome inside the index it was mapped against. */
typedef struct {
  int32_t refGenomeId, qryGenomeId, countSeq, totalQueryFragments;
  float   identity;
} bani_cgi_result;

/* One 2-way mapping behind a bani_cgi_result (cgi::MappingResult_CGI, cgid_types.hpp:18-28; 20 bytes): the fragment
 * querySeqId (the reference's seqCounter: fragments of a query genome in order, a contig shorter than a fragment
 * counting as one id) of query qryGenomeId won the position bin refStartPos / (fragLen - 20) of contig refSeqId (the
 * contig ordinal inside the index) with this identity.  What outputVisualizationFile writes one .visual line for. */
typedef struct {
  int32_t qryGenomeId, querySeqId, refSeqId, refStartPos;
  float   identity;
} bani_frag_mapping;

/* Integer work counters of one mapping call; SURVEY.md section 8(d) defines the
 * algorithmic bytes of HP2 from these (same meaning as the oracle's counters). */
typedef struct {
  uint64_t fragments;     /* F   query fragments considered                      */
  uint64_t sum_s;         /* sum of unique query minimizers probed               */
  uint64_t hits;          /* H   index positions gathered                        */
  uint64_t candidates;    /* L1 candidate regions                                */
  uint64_t n2;            /* position-ordered records scanned over all candidates*/
  uint64_t mappings;      /* P   mapping records kept                            */
  uint64_t reserved[4];
} bani_map_counters;

typedef struct bani_ctx    bani_ctx;      /* one per CUDA device: stream, scratch, statistic LUTs */
typedef struct bani_genome bani_genome;   /* a genome resident in HBM: 2-bit packed contigs + exceptions */
typedef struct bani_index  bani_index;    /* a reference index resident in HBM (HP1 output)             */

BANI_API const char *bani_last_error(void);
BANI_API const char *bani_version(void);
BANI_API void bani_params_default(bani_params *p);

/* Stat::recommendedWindowSize, src/map/include/map_stats.hpp:226-256 (host, double math). */
BANI_API int bani_recommended_window_size(const bani_params *p);
/* Stat::estimateMinimumHitsRelaxed (map_stats.hpp:142-167) and the identity /
 * upper-bound expressions of Map::doL2Mapping (computeMap.hpp:375-381): exposed
 * so the statistic LUT the kernels consume can be checked on its own. */
BANI_API int bani_stat_min_hits_relaxed(int s, int k, float perc_identity);
BANI_API int bani_stat_identity(int shared, int s, int k, float *identity, float *upper_bound);

/* Number of usable CUDA devices (0 without a driver / GPU); lets a host program shard the reference list
 * (cgi::splitReferenceGenomes, computeCoreIdentity.hpp:457-474) without linking the CUDA runtime itself. */
BANI_API int bani_device_count(int32_t *n);

/* ---- context -------------------------------------------------------------- */
BANI_API int  bani_ctx_create(int device, const bani_params *p, bani_ctx **out);
BANI_API void bani_ctx_destroy(bani_ctx *ctx);
BANI_API int  bani_ctx_params(const bani_ctx *ctx, bani_params *out);   /* window_size resolved */
BANI_API int  bani_ctx_sync(bani_ctx *ctx);
/* Raw CUDA stream (cudaStream_t) every launch of this context goes to; for event timing. */
BANI_API void *bani_ctx_stream(bani_ctx *ctx);

/* Run-time switches of a context.  name: "sketch_reuse" (1 = read the fragment sketches of index members from the
 * index, 0 = always hash the query fragments: what a run with --ql != --rl does), "max_hits_per_piece",
 * "frag_l1_max", "l2e_buckets", "l2_stage", "upload_group_words" (tuning / test switches; results never depend on them).
 * A "frag_l1_max" below 8192 sends fragments with more hits to the device-wide sort instead of one CTA each.
 * Environment, read when a context is created: BANI_NO_SKETCH_REUSE, BANI_MAX_HITS_PER_PIECE, BANI_FRAG_L1_MAX,
 * BANI_L2E_BUCKETS, BANI_L2_STAGE set the defaults of those switches; BANI_TRACE=1 prints the host wall clock between
 * marks of the orchestration (index build, query sketches, every piece of the mapping) on stderr.
 * Switches that bring branches which otherwise need very large inputs down to test size (results never depend on them):
 * "frags_per_piece" (1 .. 2^18, default 2^18: fragments per query piece; exported sketches do not depend on it),
 * "event_bytes_per_piece" (0 = a quarter of device memory: a piece whose L2 event streams take more is mapped in halves),
 * "cgi_table_queries" (0 = as many as 3 GiB of bin table hold: queries per pass of the identity reduction),
 * "l2_fast" (1; 0 sends every L2 candidate to the exact kernel),
 * "cgi_sparse" (-1 = chosen per piece: the identity reduction reduces a piece's rows by sorting them when its dense
 * query x genome output would exceed both the rows and 2^22 entries, as with many small genomes; 0 = always the dense
 * tables; 1 = always the sorted rows; environment default BANI_CGI_SPARSE, any other value makes bani_ctx_create fail
 * with BANI_ERR_ARG).  "count_paths" (default 0) turns on the branch counters
 * of bani_ctx_path_counts; with it off the mapping launches exactly the same kernels with the same work.
 * Budgets of a run that builds its reference list in chunks (bani_ctx_plan_run; results never depend on them):
 * "index_bytes_budget" (0 = derived from device memory: the build peak one chunk's index may take) and
 * "query_sketch_budget" (0 = derived: a quarter of the free device memory; query sketches above it are mapped in blocks).
 * Environment defaults: BANI_INDEX_BUDGET, BANI_QUERY_BUDGET (bytes, optionally with a K, M or G suffix, binary units); a
 * value that is not a byte count makes bani_ctx_create fail with BANI_ERR_ARG. */
BANI_API int  bani_ctx_set_flag(bani_ctx *ctx, const char *name, int64_t value);

/* Which branches of the mapping path ran since the last call (counted only while the switch "count_paths" is on):
 * fills up to n_max (name, count) pairs -- names in buffers of 32 chars, always the same list in the same order --
 * sets *n, and clears the counters.  Counters: l1.class0 .. l1.class12 and l1.device_wide (fragments per L1 size class),
 * lookup.walk_saturated / lookup.walk_full_bucket (probes that walked the sorted keys), l2.events_nt64|128|256,
 * l2.dir1024|4096, l2.staged, l2.direct (L2 candidates with window events, per event-kernel variant), l2.exact_at_bounds /
 * l2.exact_total (candidates left to the exact kernel after the bounds pass / in all), piece.mapped, piece.split_hits,
 * piece.split_events, cgi.passes (passes of the dense identity reduction), cgi.sparse (pieces whose identity reduction
 * took the sparse path).  All but piece.split_* describe the pieces that were mapped, not those split. */
BANI_API int  bani_ctx_path_counts(bani_ctx *ctx, char (*names)[32], uint64_t *counts, int32_t n_max, int32_t *n);

/* Per-stage device timing.  When enabled, every stage of HP1/HP2 is bracketed by CUDA events on
 * the context's stream; bani_ctx_profile_read() synchronises, sums the elapsed time, launch count and
 * algorithmic bytes per stage name since the last read, and clears the record.  names: n_max
 * buffers of 32 chars. */
BANI_API int  bani_ctx_profile_enable(bani_ctx *ctx, int on);
BANI_API int  bani_ctx_profile_read(bani_ctx *ctx, char (*names)[32], double *ms, double *algo_bytes,
                                    int32_t *launches, int32_t n_max, int32_t *n);

/* Device memory of the context's DEVICE as the caching allocator sees it (every context and index on that device counts):
 * bytes handed out and not freed, bytes freed and kept for reuse, and the most bytes handed out at once since the previous
 * call (read and reset).  bani_ctx_trim drops the context's scratch slots and returns every cached block of the device to
 * the driver: blocks are cached by exact size, so a run that builds indexes of different sizes one after another calls
 * it between them. */
BANI_API int  bani_ctx_mem_stats(bani_ctx *ctx, uint64_t *live, uint64_t *cached, uint64_t *peak_live);
BANI_API int  bani_ctx_trim(bani_ctx *ctx);

/* Number of this library's own kernels launched on the context so far (CUB launches excluded). */
BANI_API uint64_t bani_ctx_launch_count(const bani_ctx *ctx);

/* Pinned host memory for staging genomes (optional; pageable buffers also work). */
BANI_API int  bani_host_alloc(size_t bytes, void **out);
BANI_API void bani_host_free(void *p);

/* ---- genome ingest --------------------------------------------------------
 * A genome is what one FASTA file holds: n_contigs sequences given as the raw
 * bytes kseq_read() yields (seq->seq.s / seq->seq.l, winSketch.hpp:147-150):
 * any case, any IUPAC or other byte.  Bytes are upper-cased (a-z only,
 * commonFunc.hpp:57-66) and packed on the GPU to 2 bits/base; every non-ACGT
 * byte is carried out of band so hashing sees exactly the reference's bytes.
 * `seq` is one host buffer; contig c occupies [off[c], off[c+1]).
 * Contigs keep their ordinal even when shorter than k or w (winSketch.hpp:150-164). */
BANI_API int  bani_genome_create(bani_ctx *ctx, int32_t n_contigs, const int64_t *off,
                                 const uint8_t *seq, bani_genome **out);
/* Several genomes in one call (one device synchronisation for the whole batch).
 * genome g owns contigs [gen_off[g], gen_off[g+1]) of the off[] table. */
BANI_API int  bani_genome_create_batch(bani_ctx *ctx, int32_t n_genomes, const int32_t *gen_off,
                                       const int64_t *off, const uint8_t *seq, bani_genome **out);
/* Host-packed ingest: the 2-bit layout of the device (16 bases per uint32, A0 C1 G2 T3, base i in bits [2*(i%16), +2);
 * every other byte after upper-casing a-z is code 0 plus an out-of-band (contig-relative position, byte) entry) produced
 * on the HOST -- by the reader threads, as the bytes come off kseq_read -- so that 0.25 bytes per base cross PCIe instead
 * of 1.  bani_pack_contig needs no GPU; it writes (len + 15) / 16 words and returns the exception count through *n_exc
 * (only the first exc_cap are stored: retry with larger arrays if it is bigger).
 * bani_genome_create_packed_batch: contig c of the batch has contig_len[c] bases at words + word_off[c] (multiple of 4,
 * ascending, no overlap) and its exceptions at [exc_off[c], exc_off[c+1]); genome g owns contigs
 * [gen_off[g], gen_off[g+1]).  The copies run on a second stream in groups of <= 64 MB so that an index build that
 * follows hashes the first groups while the last are in flight.  async = 0: the call returns when the copies are done;
 * async != 0: it returns at once and the host arrays (pinned) must stay untouched until the genomes have been consumed
 * by a call that returns results (bani_index_build, bani_map_*, bani_qsketch_create) or bani_ctx_sync. */
BANI_API int  bani_pack_contig(const uint8_t *seq, int64_t len, uint32_t *words, uint32_t *exc_pos, uint8_t *exc_byte,
                               uint64_t exc_cap, uint64_t *n_exc);
BANI_API int  bani_genome_create_packed_batch(bani_ctx *ctx, int32_t n_genomes, const int32_t *gen_off, const int32_t *contig_len,
                                              const int64_t *word_off, const uint32_t *words, const int64_t *exc_off,
                                              const uint32_t *exc_pos, const uint8_t *exc_byte, int32_t async, bani_genome **out);
BANI_API void bani_genome_destroy(bani_genome *g);
BANI_API int  bani_genome_info(const bani_genome *g, int32_t *n_contigs, uint64_t *total_len,
                               uint64_t *n_exceptions, uint64_t *n_fragments);
/* Device -> host decode of one contig back to (upper-cased) ASCII; test hook for the packer. */
BANI_API int  bani_genome_decode(bani_ctx *ctx, const bani_genome *g, int32_t contig, uint8_t *out, int64_t cap);

/* ---- HP1: reference index build -------------------------------------------
 * Sketch::build + Sketch::index (winSketch.hpp:124-193) over the given genomes
 * in order; seqId runs over all contigs of all genomes (sequencesByFileInfo,
 * winSketch.hpp:75,167).  An empty list builds an empty index. */
BANI_API int  bani_index_build(bani_ctx *ctx, bani_genome *const *refs, int32_t n_refs, bani_index **out);
BANI_API void bani_index_destroy(bani_index *ix);
/* The index of the longest prefix of refs whose build fits in max_bytes of device memory (bani_index_footprint with the
 * exact record count of every genome, known after the sketch launch, and U bounded by it), at least one genome:
 * *n_taken genomes, the index equal byte for byte to bani_index_build's of exactly those.  A first genome that does not
 * fit alone gives BANI_ERR_LIMIT (never a failed allocation).  *peak_bytes (optional): the most device memory the call
 * held above what was held on entry. */
BANI_API int  bani_index_build_budget(bani_ctx *ctx, bani_genome *const *refs, int32_t n_refs, uint64_t max_bytes,
                                      bani_index **out, int32_t *n_taken, uint64_t *peak_bytes);

/* ---- chunked runs: footprint, budget and plan (host arithmetic, no device needed) ----------------------------------
 * bani_index_footprint: peak device bytes of an index build of n_minimizers records (U <= n_unique_bound, n_contigs
 * contigs, bitmap_bits validity bits, th/tw/ts staging for staging_cap records) and the bytes of the index it leaves.
 * bani_map_working_set: the mapping working set bounded by the piece caps (max_hits_per_piece x 12 B of L1 staging, the L2
 * event cap -- event_bytes_per_piece, 0 = a quarter of device_bytes -- and the 3 GiB bin table of the identity reduction).
 * bani_run_working_set: the working set a run can reach, each term clamped by its cap: about query_hashes x n_refs hits
 * (a query hash meets a reference genome about once), one L2 candidate per query fragment and reference genome, the bin
 * table of ref_bases and n_queries -- megabytes for a run of a few genomes, the caps for a run of config 3's size.
 * bani_index_budget: the build peak of the largest index (at the expected 2 / (w + 1) minimizers per base) for which
 * max(build peak, resident index + working set) <= free_bytes - query_sketch_bytes: the build and the mapping are never
 * alive at once.  bani_plan_chunks: cuts genomes (total length, contig count) into consecutive chunks, each the longest
 * run whose expected build peak fits the budget and whose staging stays below 2^32 records; chunk c ends before genome
 * chunk_end[c] (cap >= n).  A genome that alone exceeds the budget gives BANI_ERR_LIMIT naming it.
 * bani_qsketch_bytes_estimate: export bytes of a genome's query sketch before it is built.
 * bani_plan_run: the plan of one GPU's run -- reference chunks (chunk_end, cap >= n_refs) and query blocks (block_end,
 * cap >= n_queries) -- from the free bytes, the device size, the piece caps and the budgets (0 = derived; the forced
 * values of "index_bytes_budget" / "query_sketch_budget").  query_sketch_bytes (optional) are the sketches' export bytes,
 * else they are estimated from query_len.  Query sketches above the query budget are mapped in blocks, unless that
 * budget is derived and the run fits one index with every sketch resident.  The index budget leaves room for the largest
 * block's sketches and the working set that block can reach (bani_run_working_set).  A derived budget that cannot hold a
 * genome does not refuse the run: it is planned as one chunk and one block, on one index, as a run that fits; a forced one
 * gives BANI_ERR_LIMIT naming the genome.  *index_budget_used (optional): the budget the chunks were cut with.
 * bani_ctx_plan_run: the same with this context's free device memory (cudaMemGetInfo plus the cached blocks), size,
 * switches and parameters; index_budget / query_budget override the switches when not 0. */
BANI_API int  bani_index_footprint(uint64_t n_minimizers, uint64_t n_unique_bound, uint64_t n_contigs, uint64_t bitmap_bits,
                                   uint64_t staging_cap, uint64_t *build_peak, uint64_t *resident);
BANI_API int  bani_map_working_set(uint64_t device_bytes, int64_t max_hits_per_piece, int64_t event_bytes_per_piece, uint64_t *bytes);
BANI_API int  bani_run_working_set(uint64_t device_bytes, int64_t max_hits_per_piece, int64_t event_bytes_per_piece,
                                   uint64_t query_hashes, uint64_t query_fragments, int32_t n_queries, uint64_t ref_bases,
                                   int32_t n_refs, int32_t window_size, int32_t frag_len, uint64_t *bytes);
BANI_API int  bani_index_budget(uint64_t free_bytes, uint64_t query_sketch_bytes, uint64_t working_set, int32_t window_size,
                                uint64_t *budget);
BANI_API int  bani_plan_chunks(const uint64_t *genome_len, const int32_t *genome_contigs, int32_t n, int32_t k, int32_t w,
                               uint64_t budget, int32_t *chunk_end, int32_t *n_chunks);
BANI_API int  bani_qsketch_bytes_estimate(uint64_t len, int32_t w, int32_t frag_len, uint64_t *bytes);
BANI_API int  bani_plan_run(uint64_t free_bytes, uint64_t device_bytes, int64_t max_hits_per_piece, int64_t event_bytes_per_piece,
                            uint64_t index_budget, uint64_t query_budget, int32_t k, int32_t w, int32_t frag_len,
                            const uint64_t *ref_len, const int32_t *ref_contigs, int32_t n_refs, const uint64_t *query_len,
                            const uint64_t *query_sketch_bytes, int32_t n_queries, int32_t *chunk_end, int32_t *n_chunks,
                            int32_t *block_end, int32_t *n_blocks, uint64_t *index_budget_used);
BANI_API int  bani_ctx_plan_run(bani_ctx *ctx, uint64_t index_budget, uint64_t query_budget, const uint64_t *ref_len, const int32_t *ref_contigs, int32_t n_refs,
                                const uint64_t *query_len, const uint64_t *query_sketch_bytes, int32_t n_queries,
                                int32_t *chunk_end, int32_t *n_chunks, int32_t *block_end, int32_t *n_blocks,
                                uint64_t *index_budget_used);
/* "123", "64M", "2G" (binary units) -> bytes: how BANI_INDEX_BUDGET / BANI_QUERY_BUDGET are read. */
BANI_API int  bani_parse_byte_count(const char *s, uint64_t *out);
/* Totals needed by Sketch::sanityCheck (winSketch.hpp:298-318) and the log lines. */
BANI_API int  bani_index_stats(const bani_index *ix, uint64_t *n_minimizers, uint64_t *n_unique,
                               uint64_t *total_len, uint64_t *n_contigs, uint64_t *n_genomes);
/* The position-ordered minimizer table (== Sketch::minimizerIndex, winSketch.hpp:94), copied to host. */
BANI_API int  bani_index_minimizers(bani_ctx *ctx, const bani_index *ix, bani_minimizer *out, uint64_t cap);
/* The lookup side (== Sketch::minimizerPosLookupIndex, winSketch.hpp:84): all positions of one hash.
 * Returns the count through *n; writes at most cap (seqId, wpos) pairs. */
BANI_API int  bani_index_lookup(bani_ctx *ctx, const bani_index *ix, uint32_t hash,
                                int32_t *seqId, int32_t *wpos, uint64_t cap, uint64_t *n);

/* ---- on-disk sketch cache (the reference has none: scripts/splitDatabase.sh + README.md:104-106 re-sketch every
 * reference in every run).  bani_index_save writes what only the sketch launch can produce -- position-ordered
 * (hash, wpos) records, contig table, validity bitmap, parameters, checksums -- as one flat file; bani_index_load reads
 * it back on a context with the SAME k / window / fragLen (anything else is refused, like an in-memory mismatch) and
 * rebuilds the lookup side on the GPU.  Host metadata (genome paths, contig names) is the caller's to store. */
BANI_API int  bani_index_save(bani_ctx *ctx, const bani_index *ix, const char *path);
BANI_API int  bani_index_load(bani_ctx *ctx, const char *path, bani_index **out);
/* Contig lengths of the index in seqId order (cap >= n_contigs of bani_index_stats) and the cumulative contig count per
 * genome (== Sketch::sequencesByFileInfo, winSketch.hpp:75; cap >= n_genomes): what a host needs to rebuild
 * Sketch::metadata lengths and computeGenomeLengths (computeCoreIdentity.hpp:48-92) for a loaded index. */
BANI_API int  bani_index_contigs(const bani_index *ix, int32_t *contig_len, uint64_t cap_contigs, int32_t *seqs_by_file, uint64_t cap_genomes);

/* ---- saved index files read in ranges: a file need not fit the device, nor was it necessarily saved on as many GPUs.
 * Files are written in version 3 (bani_index_save): besides the whole-file checksum they hold a checksum of the header and
 * contig tables and one per genome (its records and validity bitmap words), so that a run of genomes can be read and
 * verified alone.  Version 2 files (whole-file checksum only) still load whole with bani_index_load; the two calls that
 * read ranges refuse them with BANI_ERR_ARG (save the index again).
 *
 * bani_index_file_info: the header and tables of a saved index file, checked as bani_index_load checks them (version 3:
 * against their checksum).  Host only: no context, no device.  Every output is optional (NULL skips it).  Per genome
 * (cap_genomes >= *n_genomes): genome_contigs its contig count, genome_len its total length in bases, genome_records its
 * minimizer count, genome_bits its validity bitmap bits (its contig lengths, each rounded up to 32).  contig_len: every
 * contig's length in seqId order (cap_contigs >= *n_contigs).  Call once without arrays for the counts.  What a host
 * needs to plan chunks (bani_plan_run, bani_index_footprint) and the --minFraction genome lengths without loading. */
BANI_API int  bani_index_file_info(const char *path, int32_t *version, int32_t *k, int32_t *w, int32_t *frag_len, int32_t *n_genomes,
                                   uint64_t *n_contigs, uint64_t *n_minimizers, int32_t *genome_contigs, uint64_t *genome_len,
                                   uint64_t *genome_records, uint64_t *genome_bits, uint64_t cap_genomes, int32_t *contig_len,
                                   uint64_t cap_contigs);
/* The loading twin of bani_index_build_budget: the index of the longest run of genomes [first_genome, first_genome +
 * *n_taken) of a saved file whose load fits max_bytes of device memory (bani_index_footprint of the run's exact minimizer,
 * contig and bitmap counts, with no sketch staging), at least one genome; a first genome that does not fit alone gives
 * BANI_ERR_LIMIT (never a failed allocation).  Only that run's contig tables, records and bitmap words are read, each
 * checked against its checksum.  The index equals byte for byte bani_index_build's of exactly those genomes (minimizers,
 * stats, contigs, validity bitmap, mappings, derived query sketches).  *peak_bytes (optional): the most device memory the
 * call held above what was held on entry.  Same k / window / fragLen as the context, as for bani_index_load. */
BANI_API int  bani_index_load_budget(bani_ctx *ctx, const char *path, int32_t first_genome, uint64_t max_bytes, bani_index **out,
                                     int32_t *n_taken, uint64_t *peak_bytes);
/* The saved index file in_path (version 3) followed by the genomes of `added` (an index on ctx's device), written to
 * out_path: equal byte for byte to bani_index_save of bani_index_build(in_path's genomes, then added's genomes).  The
 * saved genomes are not sketched again: in_path is streamed through a fixed host buffer, never loaded onto the device,
 * and each of its genomes is checked against its checksum on the way (a mismatch names the genome).  added may hold no
 * records (genomes whose contigs are all shorter than k + w - 1).  BANI_ERR_ARG: out_path is in_path, in_path has other
 * k / window / fragLen than the context, is version 2 (save it again), holds no records (build it again with the new
 * genomes) or is corrupt.  BANI_ERR_LIMIT: the joined index exceeds 2^32 minimizers.  On any failure no file is left at
 * out_path. */
BANI_API int  bani_index_file_extend(bani_ctx *ctx, const char *in_path, const bani_index *added, const char *out_path);

/* ---- HP2: query mapping ---------------------------------------------------
 * Map::mapQuery (computeMap.hpp:112-196) for one query genome: every mapping the
 * reference would pass to its callback, in the same (fragment, candidate) order.
 * *rows is allocated by the library (free with bani_free). */
BANI_API int  bani_map_genome(bani_ctx *ctx, const bani_index *ix, const bani_genome *query,
                              bani_mapping **rows, uint64_t *n_rows,
                              uint64_t *total_query_fragments, bani_map_counters *counters);

/* Map + cgi::computeCGI fused on the device for a batch of query genomes: one
 * bani_cgi_result per (query, reference genome) pair with at least one 2-way
 * mapping, ordered by (query, refGenomeId); qryGenomeId = position in `queries`.
 * total_query_fragments (optional, n_queries entries) is filled per query. */
BANI_API int  bani_map_cgi(bani_ctx *ctx, const bani_index *ix, bani_genome *const *queries, int32_t n_queries,
                           bani_cgi_result **results, uint64_t *n_results,
                           uint64_t *total_query_fragments, bani_map_counters *counters);

/* ---- query sketch: the first half of HP2 as an object -------------------------
 * Map::doL1Mapping, computeMap.hpp:252-276: the sorted unique minimizer hashes of every 3 kb fragment of a
 * set of query genomes.  bani_map_cgi() builds it internally; building it separately lets a multi-GPU run
 * sketch each query ONCE (rank r sketches queries r, r+N, ...), move the sketches between GPUs
 * (export -> NCCL all-gather -> import; a sketch is ~0.33 bytes per query base) and map every sketch against
 * each rank's reference shard.  query_ids[i] is reported as qryGenomeId (NULL: 0..n-1).
 * hint (optional): an index on the same device.  Queries that are genomes the hint index was built from get their
 * fragment sketches from its minimizer records instead of being hashed again (the windows of a fragment are the
 * contig windows inside it) -- all-vs-all runs, and every rank of the multi-GPU split, hash each genome once.
 * bani_map_genome / bani_map_cgi pass their index as the hint themselves. */
typedef struct bani_qsketch bani_qsketch;
BANI_API int  bani_qsketch_create(bani_ctx *ctx, bani_genome *const *queries, int32_t n_queries, const int32_t *query_ids,
                                  const bani_index *hint, bani_qsketch **out);
/* The same for genomes OF the index, by genome ordinal, from the index alone (no genome handle, no bases): an index
 * loaded from disk is also the query side of an all-vs-all run. */
BANI_API int  bani_qsketch_from_index(bani_ctx *ctx, const bani_index *ix, const int32_t *genome_ordinals, int32_t n_queries,
                                      const int32_t *query_ids, bani_qsketch **out);
/* bani_qsketch_from_index for genomes of a saved file (version 3), by genome ordinal, without loading the index: only those genomes'
 * records, bitmap words and contig tables are read, each checked against its genome's checksum.  bani_qsketch_info and
 * every mapping result equal those of bani_qsketch_from_index on the whole loaded file. */
BANI_API int  bani_qsketch_from_index_file(bani_ctx *ctx, const char *path, const int32_t *genome_ordinals, int32_t n_queries,
                                           const int32_t *query_ids, bani_qsketch **out);
BANI_API void bani_qsketch_destroy(bani_qsketch *qs);
BANI_API int  bani_qsketch_info(const bani_qsketch *qs, int32_t *n_queries, uint64_t *n_fragments, uint64_t *n_hashes,
                                uint64_t *export_bytes);
/* Pack into / rebuild from one flat DEVICE buffer (cap >= export_bytes; 16-byte aligned). */
BANI_API int  bani_qsketch_export(bani_ctx *ctx, const bani_qsketch *qs, void *device_buf, uint64_t cap);
BANI_API int  bani_qsketch_import(bani_ctx *ctx, const void *device_buf, uint64_t bytes, bani_qsketch **out);
/* Several sketches of this device as ONE (queries in the order given; the sources stay valid and may be destroyed): the
 * sketches a rank received from its peers are then mapped in a few large passes instead of one small pass per peer. */
BANI_API int  bani_qsketch_merge(bani_ctx *ctx, const bani_qsketch *const *sketches, int32_t n_sketches, bani_qsketch **out);
/* bani_map_cgi for prebuilt sketches (all on this context's device); results ordered by (sketch, query, refGenomeId). */
BANI_API int  bani_map_cgi_sketch(bani_ctx *ctx, const bani_index *ix, const bani_qsketch *const *sketches, int32_t n_sketches,
                                  bani_cgi_result **results, uint64_t *n_results, bani_map_counters *counters);
/* bani_map_cgi_sketch that also returns the 2-way mappings behind every result (what --visualize writes).
 * - results are byte for byte those of bani_map_cgi_sketch.
 * - frags are ordered by (sketch, query, refSeqId, refStartPos / (fragLen - 20)).
 * - The frags of one (query, reference genome) pair number countSeq; their float32 sum in that order, divided by
 *   countSeq, is identity.
 * - Among fragments of equal identity in one bin, the largest querySeqId wins (computeCGI's stable sort).
 * Both arrays are allocated by the library (free with bani_free).  The reduction's bin table holds 8 bytes per bin
 * instead of 4, so a pass covers half as many queries. */
BANI_API int  bani_map_cgi_sketch_frags(bani_ctx *ctx, const bani_index *ix, const bani_qsketch *const *sketches, int32_t n_sketches,
                                        bani_cgi_result **results, uint64_t *n_results, bani_frag_mapping **frags, uint64_t *n_frags,
                                        bani_map_counters *counters);

BANI_API void bani_free(void *p);

/* ---- bench utilities -------------------------------------------------------
 * Deterministic synthetic genome, generated on the device and written to a host
 * buffer as upper-case ACGT ASCII (counter-based generator; fastani_b200/synth.py
 * is the same function in numpy).  ancestor_id picks the ancestor sequence,
 * strain_id the substitution stream, sub_rate_ppm the per-base substitution rate. */
BANI_API int  bani_synth_genome(bani_ctx *ctx, uint64_t seed, uint32_t ancestor_id, uint32_t strain_id,
                                uint32_t sub_rate_ppm, int64_t len, uint8_t *host_out);

#ifdef __cplusplus
}
#endif
#endif /* FASTANI_B200_H */
