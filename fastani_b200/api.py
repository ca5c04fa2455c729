"""ctypes host side of libfastani_b200.so, mirroring the reference's seam for the hot path:

    skch::Parameters  -> Parameters        (src/map/include/map_parameters.hpp:22-41)
    skch::Sketch      -> Sketch            (src/map/include/winSketch.hpp:44-115)
    skch::Map         -> Map               (src/map/include/computeMap.hpp:35-102)
    cgi::computeCGI   -> compute_cgi       (src/cgi/include/computeCoreIdentity.hpp:166-298)

Same names and argument meaning; errors surface as BaniError (the reference exit(1)s earlier,
in validateInputFiles).  No CPU fallback: a missing library or GPU raises.
"""
import ctypes as C
import os
import weakref
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "libfastani_b200.so")
_LIB = None

MAPPING_DTYPE = np.dtype([
    ("queryLen", "<i4"), ("refStartPos", "<i4"), ("refEndPos", "<i4"),
    ("queryStartPos", "<i4"), ("queryEndPos", "<i4"), ("refSeqId", "<i4"),
    ("querySeqId", "<i4"), ("nucIdentity", "<f4"), ("nucIdentityUpperBound", "<f4"),
    ("sketchSize", "<i4"), ("conservedSketches", "<i4")])
MINIMIZER_DTYPE = np.dtype([("hash", "<u4"), ("seqId", "<i4"), ("wpos", "<i4")])
CGI_DTYPE = np.dtype([("refGenomeId", "<i4"), ("qryGenomeId", "<i4"), ("countSeq", "<i4"),
                      ("totalQueryFragments", "<i4"), ("identity", "<f4")])
# bani_frag_mapping: one 2-way mapping behind a CGI_DTYPE row (what a .visual line shows)
FRAG_DTYPE = np.dtype([("qryGenomeId", "<i4"), ("querySeqId", "<i4"), ("refSeqId", "<i4"), ("refStartPos", "<i4"),
                       ("identity", "<f4")])


class BaniError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("fastani_b200 error %d: %s" % (code, msg))
        self.code = code


class _Params(C.Structure):
    _fields_ = [("kmer_size", C.c_int32), ("window_size", C.c_int32), ("frag_len", C.c_int32),
                ("perc_identity", C.c_float), ("p_value", C.c_double), ("reference_size", C.c_uint64),
                ("reserved", C.c_int32 * 8)]


class MapCounters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("fragments", "sum_s", "hits", "candidates", "n2", "mappings")] + \
               [("reserved", C.c_uint64 * 4)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n in ("fragments", "sum_s", "hits", "candidates", "n2", "mappings")}


def library_path():
    return _LIB_PATH


def load_library():
    """Loads the CUDA library.  Raises (never falls back) when it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(_LIB_PATH):
        raise BaniError(-2, "%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(there is no CPU fallback)" % _LIB_PATH)
    L = C.CDLL(_LIB_PATH)
    vp, i32, i64, u64, u32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_uint32
    P = C.POINTER
    sig = {
        "bani_last_error": (C.c_char_p, []),
        "bani_version": (C.c_char_p, []),
        "bani_params_default": (None, [P(_Params)]),
        "bani_recommended_window_size": (C.c_int, [P(_Params)]),
        "bani_stat_min_hits_relaxed": (C.c_int, [C.c_int, C.c_int, C.c_float]),
        "bani_stat_identity": (C.c_int, [C.c_int, C.c_int, C.c_int, P(C.c_float), P(C.c_float)]),
        "bani_ctx_create": (C.c_int, [C.c_int, P(_Params), P(vp)]),
        "bani_ctx_destroy": (None, [vp]),
        "bani_ctx_params": (C.c_int, [vp, P(_Params)]),
        "bani_ctx_sync": (C.c_int, [vp]),
        "bani_ctx_stream": (vp, [vp]),
        "bani_ctx_launch_count": (u64, [vp]),
        "bani_ctx_set_flag": (C.c_int, [vp, C.c_char_p, i64]),
        "bani_ctx_profile_enable": (C.c_int, [vp, C.c_int]),
        "bani_ctx_profile_read": (C.c_int, [vp, vp, vp, vp, vp, i32, P(i32)]),
        "bani_ctx_path_counts": (C.c_int, [vp, vp, vp, i32, P(i32)]),
        "bani_host_alloc": (C.c_int, [C.c_size_t, P(vp)]),
        "bani_host_free": (None, [vp]),
        "bani_genome_create": (C.c_int, [vp, i32, vp, vp, P(vp)]),
        "bani_genome_create_batch": (C.c_int, [vp, i32, vp, vp, vp, P(vp)]),
        "bani_pack_contig": (C.c_int, [vp, i64, vp, vp, vp, u64, P(u64)]),
        "bani_genome_create_packed_batch": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, P(vp)]),
        "bani_genome_destroy": (None, [vp]),
        "bani_genome_info": (C.c_int, [vp, P(i32), P(u64), P(u64), P(u64)]),
        "bani_genome_decode": (C.c_int, [vp, vp, i32, vp, i64]),
        "bani_index_build": (C.c_int, [vp, P(vp), i32, P(vp)]),
        "bani_index_destroy": (None, [vp]),
        "bani_index_stats": (C.c_int, [vp, P(u64), P(u64), P(u64), P(u64), P(u64)]),
        "bani_index_minimizers": (C.c_int, [vp, vp, vp, u64]),
        "bani_index_save": (C.c_int, [vp, vp, C.c_char_p]),
        "bani_index_load": (C.c_int, [vp, C.c_char_p, P(vp)]),
        "bani_index_contigs": (C.c_int, [vp, vp, u64, vp, u64]),
        "bani_qsketch_from_index": (C.c_int, [vp, vp, vp, i32, vp, P(vp)]),
        "bani_index_lookup": (C.c_int, [vp, vp, u32, vp, vp, u64, P(u64)]),
        "bani_map_genome": (C.c_int, [vp, vp, vp, P(vp), P(u64), P(u64), P(MapCounters)]),
        "bani_map_cgi": (C.c_int, [vp, vp, P(vp), i32, P(vp), P(u64), vp, P(MapCounters)]),
        "bani_device_count": (C.c_int, [P(i32)]),
        "bani_qsketch_create": (C.c_int, [vp, P(vp), i32, vp, vp, P(vp)]),
        "bani_qsketch_destroy": (None, [vp]),
        "bani_qsketch_info": (C.c_int, [vp, P(i32), P(u64), P(u64), P(u64)]),
        "bani_qsketch_export": (C.c_int, [vp, vp, vp, u64]),
        "bani_qsketch_import": (C.c_int, [vp, vp, u64, P(vp)]),
        "bani_qsketch_merge": (C.c_int, [vp, P(vp), i32, P(vp)]),
        "bani_map_cgi_sketch": (C.c_int, [vp, vp, P(vp), i32, P(vp), P(u64), P(MapCounters)]),
        "bani_map_cgi_sketch_frags": (C.c_int, [vp, vp, P(vp), i32, P(vp), P(u64), P(vp), P(u64), P(MapCounters)]),
        "bani_free": (None, [vp]),
        "bani_synth_genome": (C.c_int, [vp, u64, u32, u32, u32, i64, vp]),
        "bani_index_build_budget": (C.c_int, [vp, P(vp), i32, u64, P(vp), P(i32), P(u64)]),
        "bani_ctx_mem_stats": (C.c_int, [vp, P(u64), P(u64), P(u64)]),
        "bani_ctx_trim": (C.c_int, [vp]),
        "bani_ctx_plan_run": (C.c_int, [vp, u64, u64, vp, vp, i32, vp, vp, i32, vp, P(i32), vp, P(i32), P(u64)]),
        "bani_plan_run": (C.c_int, [u64, u64, i64, i64, u64, u64, i32, i32, i32, vp, vp, i32, vp, vp, i32, vp, P(i32), vp, P(i32), P(u64)]),
        "bani_run_working_set": (C.c_int, [u64, i64, i64, u64, u64, i32, u64, i32, i32, i32, P(u64)]),
        "bani_index_footprint": (C.c_int, [u64, u64, u64, u64, u64, P(u64), P(u64)]),
        "bani_map_working_set": (C.c_int, [u64, i64, i64, P(u64)]),
        "bani_index_budget": (C.c_int, [u64, u64, u64, i32, P(u64)]),
        "bani_plan_chunks": (C.c_int, [vp, vp, i32, i32, i32, u64, vp, P(i32)]),
        "bani_qsketch_bytes_estimate": (C.c_int, [u64, i32, i32, P(u64)]),
        "bani_parse_byte_count": (C.c_int, [C.c_char_p, P(u64)]),
        "bani_index_file_info": (C.c_int, [C.c_char_p, P(i32), P(i32), P(i32), P(i32), P(i32), P(u64), P(u64), vp, vp, vp, vp, u64, vp, u64]),
        "bani_index_load_budget": (C.c_int, [vp, C.c_char_p, i32, u64, P(vp), P(i32), P(u64)]),
        "bani_qsketch_from_index_file": (C.c_int, [vp, C.c_char_p, vp, i32, vp, P(vp)]),
        "bani_index_file_extend": (C.c_int, [vp, C.c_char_p, vp, C.c_char_p]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)          # AttributeError if the ABI lost a symbol
        fn.restype = res
        fn.argtypes = args
    _LIB = L
    return L


EXPORTED_SYMBOLS = [
    "bani_last_error", "bani_version", "bani_params_default", "bani_recommended_window_size", "bani_device_count",
    "bani_stat_min_hits_relaxed", "bani_stat_identity", "bani_ctx_create", "bani_ctx_destroy", "bani_ctx_params",
    "bani_ctx_sync", "bani_ctx_stream", "bani_ctx_launch_count", "bani_ctx_set_flag", "bani_ctx_profile_enable", "bani_ctx_profile_read", "bani_ctx_path_counts", "bani_host_alloc", "bani_host_free", "bani_genome_create",
    "bani_genome_create_batch", "bani_pack_contig", "bani_genome_create_packed_batch", "bani_genome_destroy", "bani_genome_info", "bani_genome_decode", "bani_index_build",
    "bani_index_destroy", "bani_index_stats", "bani_index_minimizers", "bani_index_save", "bani_index_load", "bani_index_contigs",
    "bani_qsketch_from_index", "bani_index_lookup", "bani_map_genome",
    "bani_map_cgi", "bani_free", "bani_synth_genome", "bani_qsketch_create", "bani_qsketch_destroy", "bani_qsketch_info",
    "bani_qsketch_export", "bani_qsketch_import", "bani_qsketch_merge", "bani_map_cgi_sketch", "bani_map_cgi_sketch_frags",
    "bani_index_build_budget", "bani_ctx_mem_stats", "bani_ctx_trim", "bani_ctx_plan_run", "bani_plan_run", "bani_run_working_set", "bani_index_footprint",
    "bani_map_working_set", "bani_index_budget", "bani_plan_chunks", "bani_qsketch_bytes_estimate", "bani_parse_byte_count",
    "bani_index_file_info", "bani_index_load_budget", "bani_qsketch_from_index_file", "bani_index_file_extend"]


def _check(rc):
    if rc != 0:
        raise BaniError(rc, load_library().bani_last_error().decode())


def _records_from(ptr, n, dtype):
    """n records of a structured dtype copied out of a C buffer with ONE memmove.  (np.frombuffer(...).copy() walks a
    structured array field by field: ~100 ns per record, milliseconds for the rows of a 1000 x 1000 step.)"""
    out = np.empty(int(n), dtype)
    if n:
        C.memmove(out.ctypes.data, ptr, int(n) * out.dtype.itemsize)
    return out


class Parameters:
    """skch::Parameters with the defaults of parseandSave (parseCmdArgs.hpp:118-130)."""

    def __init__(self, kmerSize=16, minReadLength=3000, windowSize=0, percentageIdentity=80.0,
                 p_value=1e-3, referenceSize=5000000, minFraction=0.2):
        self.kmerSize = kmerSize
        self.minReadLength = minReadLength
        self.windowSize = windowSize
        self.percentageIdentity = percentageIdentity
        self.p_value = p_value
        self.referenceSize = referenceSize
        self.minFraction = minFraction

    def _c(self):
        p = _Params()
        load_library().bani_params_default(C.byref(p))
        p.kmer_size = self.kmerSize
        p.window_size = self.windowSize
        p.frag_len = self.minReadLength
        p.perc_identity = self.percentageIdentity
        p.p_value = self.p_value
        p.reference_size = self.referenceSize
        return p

    def recommendedWindowSize(self):
        """Stat::recommendedWindowSize (map_stats.hpp:226-256)."""
        p = self._c()
        r = load_library().bani_recommended_window_size(C.byref(p))
        if r < 0:
            _check(r)
        return r


class Context:
    """One per GPU: CUDA stream, scratch pool and statistic tables."""

    def __init__(self, params=None, device=0):
        self.lib = load_library()
        self.params = params or Parameters()
        p = self.params._c()
        h = C.c_void_p()
        _check(self.lib.bani_ctx_create(device, C.byref(p), C.byref(h)))
        self.h = h
        self.device = device
        q = _Params()
        _check(self.lib.bani_ctx_params(self.h, C.byref(q)))
        self.windowSize = q.window_size

    def sync(self):
        _check(self.lib.bani_ctx_sync(self.h))

    @property
    def stream(self):
        return self.lib.bani_ctx_stream(self.h)

    def launch_count(self):
        return int(self.lib.bani_ctx_launch_count(self.h))

    def set_flag(self, name, value):
        """bani_ctx_set_flag: "sketch_reuse", "max_hits_per_piece", "frag_l1_max", "l2e_buckets", "l2_stage",
        "upload_group_words", "frags_per_piece", "event_bytes_per_piece", "cgi_table_queries", "l2_fast", "count_paths",
        "cgi_sparse" (-1 chosen per piece, 0 dense, 1 sparse identity reduction), "index_bytes_budget", "query_sketch_budget"."""
        _check(self.lib.bani_ctx_set_flag(self.h, name.encode(), int(value)))

    def path_counts(self):
        """{branch: count} of the mapping path since the last read (bani_ctx_path_counts; needs count_paths = 1)."""
        nmax = 64
        names = (C.c_char * 32 * nmax)()
        cnt = (C.c_uint64 * nmax)(); n = C.c_int32()
        _check(self.lib.bani_ctx_path_counts(self.h, names, cnt, nmax, C.byref(n)))
        return {names[i].value.decode(): int(cnt[i]) for i in range(n.value)}

    def mem_stats(self):
        """{"live", "cached", "peak_live"} device bytes of this context's device (bani_ctx_mem_stats; the peak is reset)."""
        a = [C.c_uint64() for _ in range(3)]
        _check(self.lib.bani_ctx_mem_stats(self.h, *[C.byref(x) for x in a]))
        return dict(zip(("live", "cached", "peak_live"), [x.value for x in a]))

    def trim(self):
        """Drops the scratch slots and returns every cached block of the device to the driver (bani_ctx_trim)."""
        _check(self.lib.bani_ctx_trim(self.h))

    def plan_run(self, ref_lengths, ref_contigs, query_lengths, query_sketch_bytes=None, index_budget=0, query_budget=0):
        """bani_ctx_plan_run with this context's free device memory: ([(first, end)] reference chunks, [(first, end)]
        query blocks, index budget).  index_budget / query_budget (bytes) override the context's switches when not 0."""
        return _plan_run(lambda *a: self.lib.bani_ctx_plan_run(self.h, int(index_budget), int(query_budget), *a),
                         ref_lengths, ref_contigs, query_lengths, query_sketch_bytes)

    def profile(self, on=True):
        _check(self.lib.bani_ctx_profile_enable(self.h, 1 if on else 0))

    def profile_read(self):
        """{stage: (ms, algorithmic_bytes, launches)} accumulated since the last read."""
        nmax = 128
        names = (C.c_char * 32 * nmax)()
        ms = (C.c_double * nmax)(); by = (C.c_double * nmax)(); la = (C.c_int32 * nmax)(); n = C.c_int32()
        _check(self.lib.bani_ctx_profile_read(self.h, names, ms, by, la, nmax, C.byref(n)))
        return {names[i].value.decode(): (ms[i], by[i], la[i]) for i in range(n.value)}

    def close(self):
        if getattr(self, "h", None):
            self.lib.bani_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- genomes
    def genome(self, contigs):
        return self.genomes([contigs])[0]

    def genomes(self, list_of_contig_lists, names=None):
        """list_of_contig_lists[g] = [(name, bytes-like)] or [bytes-like].  One device sync for the batch."""
        metas, flat = [], []
        for cl in list_of_contig_lists:
            m = []
            for c in cl:
                nm, sq = c if isinstance(c, tuple) else ("", c)
                a = np.frombuffer(sq, dtype=np.uint8) if not isinstance(sq, np.ndarray) else sq
                m.append((nm, len(a)))
                flat.append(a)
            metas.append(m)
        gen_off = np.zeros(len(metas) + 1, np.int32)
        gen_off[1:] = np.cumsum([len(m) for m in metas])
        off = np.zeros(len(flat) + 1, np.int64)
        if flat:
            off[1:] = np.cumsum([len(a) for a in flat])
        seq = np.concatenate(flat) if flat else np.zeros(1, np.uint8)
        return self.genomes_from_buffer(seq, off, gen_off, metas)

    def genomes_from_buffer(self, seq, off, gen_off, metas=None):
        """seq: one uint8 host buffer (numpy, may be pinned); contig c = seq[off[c]:off[c+1]];
        genome g owns contigs gen_off[g]:gen_off[g+1]."""
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.int64)
        gen_off = np.ascontiguousarray(gen_off, dtype=np.int32)
        n = len(gen_off) - 1
        hs = (C.c_void_p * max(n, 1))()
        _check(self.lib.bani_genome_create_batch(self.h, n, gen_off.ctypes.data, off.ctypes.data, seq.ctypes.data, hs))
        out = []
        for g in range(n):
            c0, c1 = int(gen_off[g]), int(gen_off[g + 1])
            meta = metas[g] if metas is not None else [("", int(off[c + 1] - off[c])) for c in range(c0, c1)]
            out.append(Genome(self, C.c_void_p(hs[g]), meta))
        return out

    def genomes_from_packed(self, batch, async_=False):
        """Host-packed ingest (bani_genome_create_packed_batch): `batch` is a PackedBatch.  async_=True returns at once;
        the batch's (pinned) arrays must then stay untouched until the genomes have been consumed."""
        n = len(batch.gen_off) - 1
        hs = (C.c_void_p * max(n, 1))()
        _check(self.lib.bani_genome_create_packed_batch(
            self.h, n, batch.gen_off.ctypes.data, batch.contig_len.ctypes.data, batch.word_off.ctypes.data, batch.words.ctypes.data,
            batch.exc_off.ctypes.data, batch.exc_pos.ctypes.data, batch.exc_byte.ctypes.data, 1 if async_ else 0, hs))
        return [Genome(self, C.c_void_p(hs[g]), batch.metas[g]) for g in range(n)]

    def pinned(self, nbytes):
        """A pinned uint8 host buffer (numpy view); freed when the returned array's base is collected."""
        p = C.c_void_p()
        _check(self.lib.bani_host_alloc(nbytes, C.byref(p)))
        buf = (C.c_uint8 * max(nbytes, 1)).from_address(p.value)
        weakref.finalize(buf, self.lib.bani_host_free, p.value)      # the array's base: page-locked memory goes back with it
        return np.frombuffer(buf, dtype=np.uint8, count=nbytes)

    def synth_genome(self, seed, ancestor, strain, ppm, length, out=None):
        if out is None:
            out = np.empty(length, np.uint8)
        _check(self.lib.bani_synth_genome(self.h, seed, ancestor, strain, ppm, length, out.ctypes.data))
        return out


class PackedBatch:
    """Genomes 2-bit packed on the HOST (bani_pack_contig; no GPU needed): what a reader thread hands to the upload.
    list_of_contig_lists[g] = [(name, bytes-like)] or [bytes-like]; alloc(nbytes) -> uint8 array (e.g. Context.pinned)."""

    def __init__(self, list_of_contig_lists, alloc=None, threads=0):
        lib = load_library()
        alloc = alloc or (lambda n: np.empty(max(n, 1), np.uint8))
        contigs, self.metas, gen_off = [], [], [0]
        for cl in list_of_contig_lists:
            m = []
            for c in cl:
                nm, sq = c if isinstance(c, tuple) else ("", c)
                a = np.frombuffer(sq, dtype=np.uint8) if not isinstance(sq, np.ndarray) else np.ascontiguousarray(sq, dtype=np.uint8)
                m.append((nm, len(a)))
                contigs.append(a)
            self.metas.append(m)
            gen_off.append(len(contigs))
        nc = len(contigs)
        self.gen_off = np.asarray(gen_off, np.int32)
        self.contig_len = np.asarray([len(a) for a in contigs] + [0], np.int32)
        wlen = [((len(a) + 15) // 16 + 3) // 4 * 4 for a in contigs]
        self.word_off = np.zeros(nc + 1, np.int64)
        self.word_off[1:] = np.cumsum(wlen)
        total_words = int(self.word_off[nc])
        self.words = alloc(4 * (total_words + 8)).view(np.uint32)
        self.words[:] = 0
        exc = [None] * nc

        def one(c):
            a = contigs[c]
            cap = max(len(a) // 256, 64)
            while True:
                ep = np.empty(cap, np.uint32); eb = np.empty(cap, np.uint8); n = C.c_uint64()
                _check(lib.bani_pack_contig(a.ctypes.data, len(a), self.words[int(self.word_off[c]):].ctypes.data, ep.ctypes.data, eb.ctypes.data, cap, C.byref(n)))
                if n.value <= cap:
                    exc[c] = (ep[:n.value], eb[:n.value])
                    return
                cap = n.value

        if threads > 1 and nc > 1:
            from concurrent.futures import ThreadPoolExecutor
            with ThreadPoolExecutor(threads) as ex:
                list(ex.map(one, range(nc)))
        else:
            for c in range(nc):
                one(c)
        self.exc_off = np.zeros(nc + 1, np.int64)
        if nc:
            self.exc_off[1:] = np.cumsum([len(e[0]) for e in exc])
        ne = int(self.exc_off[nc])
        self.exc_pos = alloc(4 * max(ne, 1)).view(np.uint32)
        self.exc_byte = alloc(max(ne, 1))
        for c in range(nc):
            a, b = int(self.exc_off[c]), int(self.exc_off[c + 1])
            self.exc_pos[a:b] = exc[c][0]; self.exc_byte[a:b] = exc[c][1]
        self.h2d_bytes = 4 * total_words + 5 * ne


class Genome:
    """A genome resident in HBM (2-bit packed contigs + exception list)."""

    def __init__(self, ctx, handle, meta):
        self.ctx, self.h, self.metadata = ctx, handle, meta     # metadata: [(name, len)] == ContigInfo

    def info(self):
        nc, tl, ne, nf = C.c_int32(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        _check(self.ctx.lib.bani_genome_info(self.h, C.byref(nc), C.byref(tl), C.byref(ne), C.byref(nf)))
        return {"n_contigs": nc.value, "total_len": tl.value, "n_exceptions": ne.value}

    def decode(self, contig):
        n = self.metadata[contig][1]
        out = np.empty(max(n, 1), np.uint8)
        _check(self.ctx.lib.bani_genome_decode(self.ctx.h, self.h, contig, out.ctypes.data, n))
        return out[:n]

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.lib.bani_genome_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Sketch:
    """skch::Sketch: builds the reference index on construction (winSketch.hpp:109-115)."""

    def __init__(self, ctx, ref_genomes, _handle=None):
        self.ctx = ctx
        if _handle is not None:
            self.h, self.refs = _handle, []
            return
        self.refs = list(ref_genomes)
        arr = (C.c_void_p * max(len(self.refs), 1))(*[g.h for g in self.refs])
        h = C.c_void_p()
        _check(ctx.lib.bani_index_build(ctx.h, arr, len(self.refs), C.byref(h)))
        self.h = h
        # public members of the reference class
        self.metadata = [m for g in self.refs for m in g.metadata]                  # winSketch.hpp:66
        self.sequencesByFileInfo = list(np.cumsum([len(g.metadata) for g in self.refs]).astype(int))   # :75

    @classmethod
    def build_budget(cls, ctx, ref_genomes, max_bytes):
        """bani_index_build_budget: the index of the longest prefix of ref_genomes whose build fits max_bytes (at least one
        genome).  Returns (Sketch, n_taken, peak_bytes)."""
        refs = list(ref_genomes)
        arr = (C.c_void_p * max(len(refs), 1))(*[g.h for g in refs])
        h = C.c_void_p(); n = C.c_int32(); peak = C.c_uint64()
        _check(ctx.lib.bani_index_build_budget(ctx.h, arr, len(refs), int(max_bytes), C.byref(h), C.byref(n), C.byref(peak)))
        sk = cls(ctx, None, _handle=h)
        sk.refs = refs[:n.value]
        sk.metadata = [m for g in sk.refs for m in g.metadata]
        sk.sequencesByFileInfo = list(np.cumsum([len(g.metadata) for g in sk.refs]).astype(int))
        return sk, n.value, peak.value

    def save(self, path):
        """On-disk sketch cache (bani_index_save): records + contig table + parameters; names are the caller's."""
        _check(self.ctx.lib.bani_index_save(self.ctx.h, self.h, os.fsencode(path)))

    @classmethod
    def load(cls, ctx, path, names=None):
        """bani_index_load on a context with the same k / window / fragLen; metadata lengths come from the file,
        contig names from `names` (optional list, one per contig)."""
        h = C.c_void_p()
        _check(ctx.lib.bani_index_load(ctx.h, os.fsencode(path), C.byref(h)))
        return cls._loaded(ctx, h, names)

    @classmethod
    def load_budget(cls, ctx, path, first, max_bytes, names=None):
        """bani_index_load_budget: the index of the longest run of genomes of a saved file, from genome `first`, whose load
        fits max_bytes (at least one genome); only that run is read.  names: optional, one per contig of the run.
        Returns (Sketch, n_taken, peak_bytes)."""
        h = C.c_void_p(); n = C.c_int32(); peak = C.c_uint64()
        _check(ctx.lib.bani_index_load_budget(ctx.h, os.fsencode(path), int(first), int(max_bytes), C.byref(h), C.byref(n),
                                              C.byref(peak)))
        return cls._loaded(ctx, h, names), n.value, peak.value

    @classmethod
    def _loaded(cls, ctx, h, names):
        sk = cls(ctx, None, _handle=h)
        st = sk.stats()
        cl = np.zeros(max(st["n_contigs"], 1), np.int32); sbf = np.zeros(max(st["n_genomes"], 1), np.int32)
        _check(ctx.lib.bani_index_contigs(h, cl.ctypes.data, len(cl), sbf.ctypes.data, len(sbf)))
        nc = st["n_contigs"]
        sk.metadata = [((names[c] if names else ""), int(cl[c])) for c in range(nc)]
        sk.sequencesByFileInfo = [int(x) for x in sbf[:st["n_genomes"]]]
        return sk

    def stats(self):
        a = [C.c_uint64() for _ in range(5)]
        _check(self.ctx.lib.bani_index_stats(self.h, *[C.byref(x) for x in a]))
        return dict(zip(("n_minimizers", "n_unique", "total_len", "n_contigs", "n_genomes"), [x.value for x in a]))

    def minimizerIndex(self):
        """Sketch::minimizerIndex (position order), as a MINIMIZER_DTYPE array."""
        n = self.stats()["n_minimizers"]
        out = np.empty(max(n, 1), MINIMIZER_DTYPE)
        _check(self.ctx.lib.bani_index_minimizers(self.ctx.h, self.h, out.ctypes.data, n))
        return out[:n]

    def lookup(self, hash_value, cap=1 << 16):
        """minimizerPosLookupIndex.find(hash) -> [(seqId, wpos)]"""
        s = np.empty(cap, np.int32); w = np.empty(cap, np.int32); n = C.c_uint64()
        _check(self.ctx.lib.bani_index_lookup(self.ctx.h, self.h, int(hash_value), s.ctypes.data, w.ctypes.data, cap, C.byref(n)))
        m = min(n.value, cap)
        return list(zip(s[:m].tolist(), w[:m].tolist())), n.value

    def sanityCheck(self, maxRatioDiff):
        """Sketch::sanityCheck (winSketch.hpp:298-318), float32 arithmetic as in the reference."""
        st = self.stats()
        if st["n_minimizers"] == 0 or st["n_unique"] == 0:
            return True, np.float32(0)
        hashRatio = np.float32(st["total_len"]) / np.float32(st["n_minimizers"])
        uniqHashRatio = np.float32(st["total_len"]) / np.float32(st["n_unique"])
        diff = np.float32(abs(hashRatio - uniqHashRatio))
        return (not diff > np.float32(maxRatioDiff)), diff

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.ctx.lib.bani_index_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Map:
    """skch::Map: maps one query genome on construction and hands every mapping to `f`
    (computeMap.hpp:93-102); results also kept in .rows (MAPPING_DTYPE)."""

    def __init__(self, ctx, refSketch, query_genome, f=None):
        rows = C.c_void_p(); n = C.c_uint64(); tot = C.c_uint64(); ctr = MapCounters()
        _check(ctx.lib.bani_map_genome(ctx.h, refSketch.h, query_genome.h, C.byref(rows), C.byref(n), C.byref(tot), C.byref(ctr)))
        if n.value:
            self.rows = _records_from(rows.value, n.value, MAPPING_DTYPE)
            ctx.lib.bani_free(rows)
        else:
            self.rows = np.empty(0, MAPPING_DTYPE)
        self.totalQueryFragments = tot.value
        self.counters = ctr
        if f is not None:
            for r in self.rows:
                f(r)


def compute_cgi(ctx, refSketch, query_genomes):
    """Fused map + cgi::computeCGI on the device for a list of query genomes.
    Returns (results[CGI_DTYPE], totalQueryFragments[len(queries)], MapCounters)."""
    qs = list(query_genomes)
    arr = (C.c_void_p * max(len(qs), 1))(*[g.h for g in qs])
    res = C.c_void_p(); n = C.c_uint64(); ctr = MapCounters()
    tot = np.zeros(max(len(qs), 1), np.uint64)
    _check(ctx.lib.bani_map_cgi(ctx.h, refSketch.h, arr, len(qs), C.byref(res), C.byref(n), tot.ctypes.data, C.byref(ctr)))
    if n.value:
        out = _records_from(res.value, n.value, CGI_DTYPE)
        ctx.lib.bani_free(res)
    else:
        out = np.empty(0, CGI_DTYPE)
    return out, tot[:len(qs)], ctr


class QuerySketch:
    """The first half of skch::Map as an object (Map::doL1Mapping, computeMap.hpp:252-276): sorted unique
    minimizer hashes of every fragment of a list of query genomes, resident on the GPU.  It can be packed into
    a flat device buffer (export_to) and rebuilt on another GPU (from_device_buffer), which is what a multi-GPU
    run exchanges instead of sketching every query on every rank."""

    def __init__(self, ctx, query_genomes=None, query_ids=None, hint=None, _handle=None):
        self.ctx = ctx
        if _handle is not None:
            self.h = _handle
            return
        if query_genomes is None:
            raise ValueError("query genomes, or QuerySketch.from_index / from_device_buffer")
        qs = list(query_genomes)
        arr = (C.c_void_p * max(len(qs), 1))(*[g.h for g in qs])
        ids = None
        if query_ids is not None:
            ids = np.ascontiguousarray(query_ids, dtype=np.int32)
            assert len(ids) == len(qs)
        h = C.c_void_p()
        _check(ctx.lib.bani_qsketch_create(ctx.h, arr, len(qs), ids.ctypes.data if ids is not None else None,
                                           hint.h if hint is not None else None, C.byref(h)))
        self.h = h

    @classmethod
    def from_index(cls, ctx, sketch, genome_ordinals, query_ids=None):
        """Fragment sketches of genomes OF the index by ordinal, from the index alone (bani_qsketch_from_index)."""
        ords = np.ascontiguousarray(genome_ordinals, dtype=np.int32)
        ids = np.ascontiguousarray(query_ids if query_ids is not None else genome_ordinals, dtype=np.int32)
        assert len(ids) == len(ords)
        h = C.c_void_p()
        _check(ctx.lib.bani_qsketch_from_index(ctx.h, sketch.h, ords.ctypes.data, len(ords), ids.ctypes.data, C.byref(h)))
        return cls(ctx, _handle=h)

    @classmethod
    def from_index_file(cls, ctx, path, genome_ordinals, query_ids=None):
        """from_index for genomes of a saved index file, reading only their records (bani_qsketch_from_index_file)."""
        ords = np.ascontiguousarray(genome_ordinals, dtype=np.int32)
        ids = np.ascontiguousarray(query_ids if query_ids is not None else genome_ordinals, dtype=np.int32)
        assert len(ids) == len(ords)
        h = C.c_void_p()
        _check(ctx.lib.bani_qsketch_from_index_file(ctx.h, os.fsencode(path), ords.ctypes.data, len(ords), ids.ctypes.data, C.byref(h)))
        return cls(ctx, _handle=h)

    @classmethod
    def from_device_buffer(cls, ctx, device_ptr, nbytes):
        h = C.c_void_p()
        _check(ctx.lib.bani_qsketch_import(ctx.h, C.c_void_p(int(device_ptr)), int(nbytes), C.byref(h)))
        return cls(ctx, _handle=h)

    @classmethod
    def merge(cls, ctx, sketches):
        """One sketch holding the queries of `sketches` in order (bani_qsketch_merge); the sources stay valid."""
        qs = list(sketches)
        arr = (C.c_void_p * max(len(qs), 1))(*[q.h for q in qs])
        h = C.c_void_p()
        _check(ctx.lib.bani_qsketch_merge(ctx.h, arr, len(qs), C.byref(h)))
        return cls(ctx, _handle=h)

    def info(self):
        n = C.c_int32(); f = C.c_uint64(); t = C.c_uint64(); b = C.c_uint64()
        _check(self.ctx.lib.bani_qsketch_info(self.h, C.byref(n), C.byref(f), C.byref(t), C.byref(b)))
        return {"n_queries": n.value, "n_fragments": f.value, "n_hashes": t.value, "export_bytes": b.value}

    def export_to(self, device_ptr, cap):
        _check(self.ctx.lib.bani_qsketch_export(self.ctx.h, self.h, C.c_void_p(int(device_ptr)), int(cap)))

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.bani_qsketch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _take_records(lib, ptr, n, dtype):
    if not n.value:
        return np.empty(0, dtype)
    out = _records_from(ptr.value, n.value, dtype)
    lib.bani_free(ptr)
    return out


def compute_cgi_sketched(ctx, refSketch, query_sketches, fragments=False):
    """compute_cgi for prebuilt QuerySketch objects; qryGenomeId = the query_ids the sketches were built with.
    Returns (results[CGI_DTYPE], MapCounters).  fragments=True (bani_map_cgi_sketch_frags) returns
    (results, MapCounters, frags[FRAG_DTYPE]): the same results and the 2-way mappings behind them, ordered by
    (sketch, query, refSeqId, position bin); report.visual_lines writes them as .visual lines."""
    qs = list(query_sketches)
    arr = (C.c_void_p * max(len(qs), 1))(*[q.h for q in qs])
    res = C.c_void_p(); n = C.c_uint64(); ctr = MapCounters()
    if not fragments:
        _check(ctx.lib.bani_map_cgi_sketch(ctx.h, refSketch.h, arr, len(qs), C.byref(res), C.byref(n), C.byref(ctr)))
        return _take_records(ctx.lib, res, n, CGI_DTYPE), ctr
    fr = C.c_void_p(); nf = C.c_uint64()
    _check(ctx.lib.bani_map_cgi_sketch_frags(ctx.h, refSketch.h, arr, len(qs), C.byref(res), C.byref(n), C.byref(fr), C.byref(nf),
                                             C.byref(ctr)))
    out = _take_records(ctx.lib, res, n, CGI_DTYPE)
    return out, ctr, _take_records(ctx.lib, fr, nf, FRAG_DTYPE)


# ---------------------------------------------------------------------------------------- chunked runs
def index_footprint(n_minimizers, n_unique_bound, n_contigs, bitmap_bits, staging_cap):
    """(build peak, resident index) in device bytes of an index build (bani_index_footprint; no GPU needed)."""
    pk, rs = C.c_uint64(), C.c_uint64()
    _check(load_library().bani_index_footprint(int(n_minimizers), int(n_unique_bound), int(n_contigs), int(bitmap_bits),
                                               int(staging_cap), C.byref(pk), C.byref(rs)))
    return pk.value, rs.value


def map_working_set(device_bytes, max_hits_per_piece=3 << 29, event_bytes_per_piece=0):
    """Device bytes of the mapping working set from its caps (bani_map_working_set; no GPU needed)."""
    b = C.c_uint64()
    _check(load_library().bani_map_working_set(int(device_bytes), int(max_hits_per_piece), int(event_bytes_per_piece), C.byref(b)))
    return b.value


def index_budget(free_bytes, query_sketch_bytes, working_set, window_size):
    """The index budget (bani_index_budget; no GPU needed)."""
    b = C.c_uint64()
    _check(load_library().bani_index_budget(int(free_bytes), int(query_sketch_bytes), int(working_set), int(window_size), C.byref(b)))
    return b.value


def plan_chunks(genome_lengths, genome_contigs, k, w, budget):
    """Consecutive chunks [(first, end)] of a reference list whose indexes fit `budget` (bani_plan_chunks; no GPU needed).
    Raises BaniError (BANI_ERR_LIMIT) naming a genome that alone does not fit."""
    ln = np.ascontiguousarray(genome_lengths, dtype=np.uint64)
    nc = np.ascontiguousarray(genome_contigs, dtype=np.int32)
    assert len(ln) == len(nc)
    ends = np.zeros(max(len(ln), 1), np.int32); n = C.c_int32()
    _check(load_library().bani_plan_chunks(ln.ctypes.data, nc.ctypes.data, len(ln), int(k), int(w), int(budget),
                                           ends.ctypes.data, C.byref(n)))
    return _ranges(ends[:n.value].tolist())


def parse_byte_count(text):
    """How BANI_INDEX_BUDGET / BANI_QUERY_BUDGET are read ("123", "64M", "2G"); raises BaniError otherwise."""
    b = C.c_uint64()
    _check(load_library().bani_parse_byte_count(text.encode(), C.byref(b)))
    return b.value


def _ranges(ends):
    out, a = [], 0
    for e in ends:
        out.append((a, e)); a = e
    return out


def _plan_run(call, ref_lengths, ref_contigs, query_lengths, query_sketch_bytes):
    rl = np.ascontiguousarray(ref_lengths, dtype=np.uint64)
    rc = np.ascontiguousarray(ref_contigs, dtype=np.int32)
    ql = np.ascontiguousarray(query_lengths, dtype=np.uint64)
    qb = None if query_sketch_bytes is None else np.ascontiguousarray(query_sketch_bytes, dtype=np.uint64)
    assert len(rl) == len(rc) and (qb is None or len(qb) == len(ql))
    ce = np.zeros(max(len(rl), 1), np.int32); be = np.zeros(max(len(ql), 1), np.int32)
    nc, nb, ib = C.c_int32(), C.c_int32(), C.c_uint64()
    _check(call(rl.ctypes.data, rc.ctypes.data, len(rl), ql.ctypes.data, qb.ctypes.data if qb is not None else None, len(ql),
                ce.ctypes.data, C.byref(nc), be.ctypes.data, C.byref(nb), C.byref(ib)))
    return _ranges(ce[:nc.value].tolist()), _ranges(be[:nb.value].tolist()), ib.value


def plan_run(free_bytes, device_bytes, ref_lengths, ref_contigs, query_lengths, query_sketch_bytes=None, k=16, w=24, frag_len=3000,
             index_budget=0, query_budget=0, max_hits_per_piece=3 << 29, event_bytes_per_piece=0):
    """bani_plan_run (no GPU needed): ([(first, end)] reference chunks, [(first, end)] query blocks, index budget) of one GPU's
    run with free_bytes of device memory free.  Budgets of 0 are derived; a derived budget that cannot hold a genome plans
    the run on one index, a forced one raises BaniError naming the genome."""
    return _plan_run(lambda *a: load_library().bani_plan_run(int(free_bytes), int(device_bytes), int(max_hits_per_piece),
                                                             int(event_bytes_per_piece), int(index_budget), int(query_budget),
                                                             int(k), int(w), int(frag_len), *a),
                     ref_lengths, ref_contigs, query_lengths, query_sketch_bytes)


def run_working_set(device_bytes, query_hashes, query_fragments, n_queries, ref_bases, n_refs, w=24, frag_len=3000,
                    max_hits_per_piece=3 << 29, event_bytes_per_piece=0):
    """The mapping working set a run of this size can reach (bani_run_working_set; no GPU needed)."""
    b = C.c_uint64()
    _check(load_library().bani_run_working_set(int(device_bytes), int(max_hits_per_piece), int(event_bytes_per_piece), int(query_hashes),
                                               int(query_fragments), int(n_queries), int(ref_bases), int(n_refs), int(w), int(frag_len),
                                               C.byref(b)))
    return b.value


def compute_cgi_chunked(ctx, ref_contig_lists, query_sketches, index_budget=None, query_budget=None):
    """compute_cgi_sketched against a reference list that need not fit the device at once: Context.plan_run cuts the
    references into chunks and the query sketches into blocks (each sketch counts as one query of its hashes' expected
    length); every chunk is uploaded, indexed (bani_index_build_budget: genomes it does not take stay uploaded for the
    next chunk) and mapped against every block.  refGenomeId is the position in ref_contig_lists.  Budgets (bytes)
    default to the context's switches, else to what its free device memory allows.  A run of one chunk and one block is
    compute_cgi_sketched on one index.
    Returns (results[CGI_DTYPE] ordered by (query, ref), plan) with plan = {"chunks": [(first, end)] per index built,
    "blocks": [(first, end)] ranges of query_sketches, "index_budget", "device_bytes": live + cached device bytes after
    every chunk}."""
    refs = list(ref_contig_lists)
    qs = list(query_sketches)
    infos = [q.info() for q in qs]
    qlen = [x["n_hashes"] * (ctx.windowSize + 1) // 2 for x in infos]
    lens = [sum(len(c[1] if isinstance(c, tuple) else c) for c in cl) for cl in refs]
    planned, blocks, ib = ctx.plan_run(lens, [len(cl) for cl in refs], qlen, [x["export_bytes"] for x in infos],
                                       index_budget or 0, query_budget or 0)
    plan = {"chunks": [], "blocks": blocks, "index_budget": ib, "device_bytes": []}
    if len(planned) <= 1 and len(blocks) <= 1:                    # fits: one index, one mapping call
        sk = Sketch(ctx, ctx.genomes(refs))
        res, _ = compute_cgi_sketched(ctx, sk, qs)
        plan["chunks"] = [(0, len(refs))]
        return res, plan
    parts = []
    for bi, (q0, q1) in enumerate(blocks):
        nxt, pending, first = 0, [], 0
        while nxt < len(planned) or pending:
            if not pending:
                a, e = planned[nxt]; nxt += 1
                pending, first = ctx.genomes(refs[a:e]), a
            sk, taken, _ = Sketch.build_budget(ctx, pending, ib)
            for g in pending[:taken]:
                g.close()
            pending = pending[taken:]
            res, _ = compute_cgi_sketched(ctx, sk, qs[q0:q1])
            res["refGenomeId"] += first
            parts.append(res)
            sk.close()
            ctx.trim()
            if bi == 0:
                plan["chunks"].append((first, first + taken))
                m = ctx.mem_stats()
                plan["device_bytes"].append(m["live"] + m["cached"])
            first += taken
    out = np.concatenate(parts) if parts else np.empty(0, CGI_DTYPE)
    out = out[np.lexsort((out["refGenomeId"], out["qryGenomeId"]))]
    return out, plan


def index_file_info(path):
    """Header and tables of a saved index file (bani_index_file_info; no GPU needed): {"version", "k", "w", "frag_len",
    "n_genomes", "n_contigs", "n_minimizers"} and per genome numpy arrays "genome_contigs", "genome_length" (bases),
    "genome_records" (minimizers), "genome_bits" (validity bitmap bits), and "contig_length" in seqId order."""
    lib = load_library()
    p = os.fsencode(path)
    ver, k, w, fl, ng = (C.c_int32() for _ in range(5))
    nc, nm = C.c_uint64(), C.c_uint64()
    scalars = [C.byref(x) for x in (ver, k, w, fl, ng, nc, nm)]
    _check(lib.bani_index_file_info(p, *scalars, None, None, None, None, 0, None, 0))
    gc = np.zeros(max(ng.value, 1), np.int32); gl = np.zeros(max(ng.value, 1), np.uint64)
    gr = np.zeros(max(ng.value, 1), np.uint64); gb = np.zeros(max(ng.value, 1), np.uint64)
    cl = np.zeros(max(nc.value, 1), np.int32)
    _check(lib.bani_index_file_info(p, *scalars, gc.ctypes.data, gl.ctypes.data, gr.ctypes.data, gb.ctypes.data, len(gc),
                                    cl.ctypes.data, len(cl)))
    n, m = ng.value, nc.value
    return {"version": ver.value, "k": k.value, "w": w.value, "frag_len": fl.value, "n_genomes": n, "n_contigs": m,
            "n_minimizers": nm.value, "genome_contigs": gc[:n], "genome_length": gl[:n], "genome_records": gr[:n],
            "genome_bits": gb[:n], "contig_length": cl[:m]}


def index_file_extend(ctx, in_path, added_sketch, out_path):
    """bani_index_file_extend: the saved index file in_path (version 3) followed by the genomes of added_sketch (a Sketch on
    ctx's device), written to out_path byte for byte as Sketch(in_path's genomes + added_sketch's genomes).save(out_path)
    would write it.  in_path's genomes are not sketched again; its records are streamed through host memory and checked
    against their checksums.  Raises BaniError (nothing is left at out_path) when out_path is in_path, the parameters
    differ, in_path is version 2, holds no records or is corrupt, or the joined index exceeds 2^32 minimizers."""
    _check(ctx.lib.bani_index_file_extend(ctx.h, os.fsencode(in_path), added_sketch.h, os.fsencode(out_path)))


def compute_cgi_from_index_file(ctx, path, query_sketches, index_budget=None, query_budget=None):
    """compute_cgi_chunked against the genomes of a saved index file (Sketch.save), which need not fit the device at once:
    Context.plan_run plans chunks and query blocks from the file's genome lengths (index_file_info); if the run needs more
    than one chunk or block, every block is mapped against the file's genomes loaded in runs that fit the index budget
    (Sketch.load_budget from genome 0 until every genome is taken).  refGenomeId is the genome's ordinal in the file.  A
    run of one chunk and one block is Sketch.load + compute_cgi_sketched.
    Returns (results[CGI_DTYPE] ordered by (query, ref), plan) with the keys of compute_cgi_chunked; "chunks" are the runs
    that were loaded."""
    info = index_file_info(path)
    n = info["n_genomes"]
    qs = list(query_sketches)
    infos = [q.info() for q in qs]
    qlen = [x["n_hashes"] * (ctx.windowSize + 1) // 2 for x in infos]
    planned, blocks, ib = ctx.plan_run(info["genome_length"], info["genome_contigs"], qlen, [x["export_bytes"] for x in infos],
                                       index_budget or 0, query_budget or 0)
    plan = {"chunks": [], "blocks": blocks, "index_budget": ib, "device_bytes": []}
    if len(planned) <= 1 and len(blocks) <= 1:                    # fits: one index, one mapping call
        sk = Sketch.load(ctx, path)
        res, _ = compute_cgi_sketched(ctx, sk, qs)
        plan["chunks"] = [(0, n)]
        return res, plan
    parts = []
    for bi, (q0, q1) in enumerate(blocks):
        first = 0
        while first < n:
            sk, taken, _ = Sketch.load_budget(ctx, path, first, ib)
            res, _ = compute_cgi_sketched(ctx, sk, qs[q0:q1])
            res["refGenomeId"] += first
            parts.append(res)
            sk.close()
            ctx.trim()
            if bi == 0:
                plan["chunks"].append((first, first + taken))
                m = ctx.mem_stats()
                plan["device_bytes"].append(m["live"] + m["cached"])
            first += taken
    out = np.concatenate(parts) if parts else np.empty(0, CGI_DTYPE)
    out = out[np.lexsort((out["refGenomeId"], out["qryGenomeId"]))]
    return out, plan
