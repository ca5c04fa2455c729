"""GPU (-m gpu): every dispatch branch of the mapping path against the oracle, with the branch named.

The mapping path picks among many kernel variants by the shape of the data (L1 size classes, lookup fallbacks, the L2
fast path and its exact fallback, event-kernel variants, piece splits, passes of the identity reduction).  Each test
below builds a small workload that reaches one family of branches, compares every mapping row byte for byte with
pyoracle.map_genome (and identity results bit for bit with pyoracle.cgi), and asserts from Context.path_counts() that
the branch it targets ran -- with the exact count where the host can predict it.

`python tests/test_gpu_paths.py` (no GPU needed) prints the oracle side of every workload and the predicted L1 class
histograms."""
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN                  # first: it puts the repository and the oracle on sys.path (also for the rehearsal)
import fastani_b200 as fb
import pyoracle as po
from fastani_b200.synth import synth_genome

pytestmark = pytest.mark.gpu

K, L = 16, 3000
CLASS_HITS = [256 * i for i in (1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 16, 24, 32)]       # upper bound of every L1 size class


def _ctx(**kw):
    ctx = fb.Context(fb.Parameters(**kw))
    ctx.set_flag("count_paths", 1)
    return ctx


def _paths(ctx, tag):
    p = ctx.path_counts()
    print(tag, {k: v for k, v in p.items() if v})
    return p


def _oracle_index(genomes, k, w):
    rec, sbf, _ = po.sketch_genomes(genomes, k, w)
    return rec, sbf, po.Index(rec)


def _map_and_compare(ctx, sk, oix, genome, handle, k, w, frag_len):
    """Rows byte for byte and the work counters the oracle keeps; returns the oracle rows."""
    rows, tq, octr = po.map_genome(oix, genome, k, w, frag_len)
    m = fb.Map(ctx, sk, handle)
    assert m.totalQueryFragments == tq
    assert m.rows.tobytes() == rows.tobytes()
    c = m.counters.as_dict()
    assert (c["sum_s"], c["hits"], c["candidates"], c["mappings"]) == (octr.sum_s, octr.hits, octr.candidates, octr.mappings)
    return rows


def _fragment_sketches(genome, k, w, frag_len):
    """Sorted unique minimizer hashes of every fragment (computeMap.hpp:131-189, :260-276), as the oracle cuts them."""
    out = []
    for _, sq in genome:
        u = po.upper(sq)
        if len(u) < max(w, k, frag_len):
            continue
        for f in range(len(u) // frag_len):
            h = np.unique(po.minimizers(u[f * frag_len:(f + 1) * frag_len], k, w)["hash"])
            if len(h):
                out.append(h)
    return out


def _hits_per_fragment(frag_hashes, rec):
    keys, cnt = np.unique(rec["hash"], return_counts=True)
    res = []
    for h in frag_hashes:
        i = np.searchsorted(keys, h)
        i = np.minimum(i, len(keys) - 1)
        res.append(int(np.where(keys[i] == h, cnt[i], 0).sum()))
    return res


def predicted_classes(hits, frag_l1_max=8192):
    """L1 size class of every fragment (hits.cu: frag_classify_kernel): 0..12 by hit count, 13 = device-wide sort."""
    hist = [0] * 14
    for n in hits:
        if n == 0:
            continue
        if n > frag_l1_max:
            hist[13] += 1
        else:
            hist[next(c for c, top in enumerate(CLASS_HITS) if n <= top)] += 1
    return hist


def _class_counts(p):
    return [p["l1.class%d" % c] for c in range(13)] + [p["l1.device_wide"]]


# ---------------------------------------------------------------- workloads (CPU side; shared with the rehearsal below)
LADDER_N = list(range(1, 41)) + [48]


def ladder_workload():
    """One query strain and 48 sister strains of its ancestor (0.2 % substitutions each): an index of the first n
    strains gives every fragment about 230 * n hits, so n = 1 ... 40, 48 walks through every L1 size class."""
    q = [("q", synth_genome(41, 1, 0, 0, 30000).tobytes())]
    strains = [[("s%d" % i, synth_genome(41, 1, i, 2000, 30000).tobytes())] for i in range(1, max(LADDER_N) + 1)]
    return q, strains


UNIT_COPIES = (254, 255, 256, 310)


def repeat_workload():
    """A reference whose 1 kbp units occur in 254, 255, 256 and 310 single-unit contigs (the probe table stores counts
    up to 255), a query strain of its backbone carrying the four units, and an unrelated query (probes that find a
    full bucket without their key)."""
    backbone = synth_genome(43, 1, 0, 0, 400000).tobytes()
    units = [synth_genome(43, 2 + i, 0, 0, 1000).tobytes() for i in range(len(UNIT_COPIES))]
    ref = [("backbone", backbone)]
    for u, n in zip(units, UNIT_COPIES):
        ref += [("u%d" % len(ref), u)] * n
    qs = bytearray(synth_genome(43, 1, 1, 5000, 60000).tobytes())
    for i, u in enumerate(units):
        qs[4000 + 12000 * i:5000 + 12000 * i] = u
    return ref, [("q", bytes(qs))], [("far", synth_genome(43, 9, 0, 0, 300000).tobytes())]


def sparse_query_workload():
    """A strain whose fragments are N except 40 ... 200 bases: sketches of a few hashes, so every gap between two
    neighbouring query hashes holds dozens of foreign window hashes of the unmasked reference."""
    ref = synth_genome(47, 1, 0, 0, 60000).tobytes()
    q = bytearray(b"N" * 60000)
    strain = synth_genome(47, 1, 1, 2000, 60000).tobytes()
    for f in range(20):
        keep = (40, 60, 80, 120, 200)[f % 5]
        o = f * 3000 + 1000
        q[o:o + keep] = strain[o:o + keep]
    return [("ref", ref)], [("sparse", bytes(q))]


def tandem_workload():
    """A 5-base unit repeated over 3 Mbp: one L1 candidate spans the whole contig, more than 2^20 window events."""
    unit = b"AACGT"
    ref = [("rep", unit * 600000), ("flank", synth_genome(53, 1, 0, 0, 20000).tobytes())]
    q = [("q", unit * 600 + synth_genome(53, 2, 0, 0, 3000).tobytes())]
    return ref, q


def piece_workload():
    """17 multi-contig genomes of two clusters (30 ... 200 kbp, so some exceed a piece of 7 or 64 fragments); the
    index holds the even ones, so the query list alternates index members with non-members, and every two neighbouring
    queries include one of the first cluster, which the index holds most of."""
    gs = []
    for i in range(17):
        n = (30000, 60000, 200000, 45000, 120000)[i % 5]
        seq = synth_genome(59, 1 + (i % 3 == 2), i, 4000 + 500 * i, n).tobytes()
        if i % 3 == 1:
            gs.append([("g%d_a" % i, seq[:n // 2]), ("g%d_tiny" % i, seq[n // 2:n // 2 + 700]), ("g%d_b" % i, seq[n // 2 + 700:])])
        else:
            gs.append([("g%d" % i, seq)])
    return gs


def cgi_edge_workload():
    """Reference genome 0: a 9 kbp region present on two contigs and twice within one contig (ties between rows of one
    fragment and genome); genome 1: contigs with no rows at all; genome 2: a sister strain."""
    dup = synth_genome(61, 1, 0, 0, 9000).tobytes()
    a = synth_genome(61, 2, 0, 0, 20000).tobytes()
    # the middle fragment of the duplicate maps 2995 bases into it: from 5945, that is 8940, the start of bin 3 (fragLen - 20)
    ref0 = [("dup_a", a[:5945] + dup + a[5945:10945] + dup + a[10945:]), ("dup_b", dup + a[:3000])]
    ref1 = [("none1", synth_genome(61, 3, 0, 0, 30000).tobytes()), ("none2", synth_genome(61, 4, 0, 0, 5000).tobytes())]
    ref2 = [("sis", synth_genome(61, 2, 1, 8000, 40000).tobytes())]
    q = [("q", synth_genome(61, 2, 2, 6000, 30000).tobytes()[:12000] + dup + synth_genome(61, 2, 2, 6000, 30000).tobytes()[12000:])]
    return [ref0, ref1, ref2], q


# ---------------------------------------------------------------- tests
def test_l1_class_ladder():
    """Hits per fragment sweep past every L1 size class boundary (warp kernels up to 512 hits, the CTA kernel's 11
    classes with 8- and 10-bit digits, the device-wide sort above 8192): the class histogram equals the one predicted
    from the oracle's fragment sketches and index counts, and the rows equal the oracle's with the per-fragment kernels
    and with every fragment on the device-wide path (frag_l1_max = 0)."""
    q, strains = ladder_workload()
    ctx = _ctx()
    w = ctx.windowSize
    hq = ctx.genome(q)
    hs = ctx.genomes(strains)
    frag = _fragment_sketches(q, K, w, L)
    seen = [0] * 14
    for n in LADDER_N:
        rec = po.sketch_genomes(strains[:n], K, w)[0]
        oix = po.Index(rec)
        sk = fb.Sketch(ctx, hs[:n])
        want = predicted_classes(_hits_per_fragment(frag, rec))
        for cap in (8192, 0):
            ctx.set_flag("frag_l1_max", cap)
            _map_and_compare(ctx, sk, oix, q, hq, K, w, L)
            got = _class_counts(_paths(ctx, "n=%d frag_l1_max=%d" % (n, cap)))
            assert got == (want if cap else [0] * 13 + [sum(want)]), (n, cap)
        seen = [a + b for a, b in zip(seen, want)]
    assert all(seen), seen                                  # every class and the device-wide path were reached


def test_lookup_fallbacks():
    """Hashes with 254, 255, 256 and 310 positions: the probe table saturates at 255 and sends those probes to the sorted
    keys; a non-member query meets full buckets without its key.  Lookups, rows and work counters equal the oracle's."""
    ref, q, far = repeat_workload()
    ctx = _ctx()
    w = ctx.windowSize
    hr, hq, hf = ctx.genomes([ref, q, far])
    sk = fb.Sketch(ctx, [hr])
    rec, _, oix = _oracle_index([ref], K, w)
    assert (sk.minimizerIndex() == rec).all()
    keys, cnt = np.unique(rec["hash"], return_counts=True)
    for c in (254, 255, 256, 310):
        hs = keys[cnt == c]
        assert len(hs), c
        for h in hs[:3]:
            pos, n = sk.lookup(int(h))
            sel = rec[rec["hash"] == h]
            assert n == c and pos == list(zip(sel["seqId"].tolist(), sel["wpos"].tolist()))
    fq = _fragment_sketches(q, K, w, L)
    saturated = sum(int(np.isin(h, keys[cnt >= 255]).sum()) for h in fq)
    assert saturated > 0
    _map_and_compare(ctx, sk, oix, q, hq, K, w, L)
    p = _paths(ctx, "repeat query")
    assert p["lookup.walk_saturated"] > 0
    assert p["lookup.walk_saturated"] + p["lookup.walk_full_bucket"] >= saturated
    _map_and_compare(ctx, sk, oix, far, hf, K, w, L)
    p = _paths(ctx, "unrelated query")
    assert p["lookup.walk_full_bucket"] > 0


def test_l2_gap_counter_overflow_goes_to_the_exact_kernel():
    """Sketches of a few hashes against an unmasked reference: a 7-bit gap counter of l2_seq_kernel reaches 64 and the
    candidate is handed to l2_kernel after the fast path ran (s <= sLimit)."""
    ref, q = sparse_query_workload()
    ctx = _ctx()
    w = ctx.windowSize
    hr, hq = ctx.genomes([ref, q])
    sk = fb.Sketch(ctx, [hr])
    _, _, oix = _oracle_index([ref], K, w)
    rows = _map_and_compare(ctx, sk, oix, q, hq, K, w, L)
    p = _paths(ctx, "sparse query")
    assert len(rows) > 0
    assert p["l2.exact_total"] > p["l2.exact_at_bounds"]
    assert p["l2.events_nt64"] + p["l2.events_nt128"] + p["l2.events_nt256"] > 0


def test_l2_million_event_candidate_goes_to_the_exact_kernel():
    """One candidate over a 3 Mbp tandem repeat has more than 2^20 window events: l2_bounds_kernel hands it to
    l2_kernel.  (The oracle sweeps the same 600 k records; a few seconds.)"""
    ref, q = tandem_workload()
    ctx = _ctx()
    w = ctx.windowSize
    hr, hq = ctx.genomes([ref, q])
    sk = fb.Sketch(ctx, [hr])
    rec, _, oix = _oracle_index([ref], K, w)
    assert (rec["seqId"] == 0).sum() > (1 << 19)
    rows = _map_and_compare(ctx, sk, oix, q, hq, K, w, L)
    p = _paths(ctx, "tandem repeat")
    assert len(rows) > 0 and p["l2.exact_at_bounds"] >= 1 and p["l1.device_wide"] >= 1


@pytest.mark.parametrize("w,frag_len", [(30, 45), (25, 40)])
def test_l2_without_window_links_uses_the_exact_kernel(w, frag_len):
    """fragLen < w + k - 1 (cmw < 2, computeMap.hpp:427): the index has no window links for the fast path, so every
    candidate goes to l2_kernel."""
    ref = [("r", synth_genome(67, 1, 0, 0, 20000).tobytes())]
    q = [("q", synth_genome(67, 1, 1, 10000, 20000).tobytes())]
    ctx = _ctx(windowSize=w, minReadLength=frag_len)
    assert ctx.windowSize == w
    hr, hq = ctx.genomes([ref, q])
    sk = fb.Sketch(ctx, [hr])
    _, _, oix = _oracle_index([ref], K, w)
    rows = _map_and_compare(ctx, sk, oix, q, hq, K, w, frag_len)
    p = _paths(ctx, "cmw=%d" % (frag_len - w - K + 2))
    assert len(rows) > 0
    assert p["l2.exact_total"] == p["l2.exact_at_bounds"] > 0
    assert p["l2.events_nt64"] + p["l2.events_nt128"] + p["l2.events_nt256"] == 0


def test_exact_kernel_alone_reproduces_the_real_pair():
    """l2_fast = 0: the exact kernel as a second, independent L2 on the E. coli / Shigella pair (all 4138 rows of the
    reference's own output)."""
    ec, sh = fb.read_fasta(os.path.join(GOLDEN, "Escherichia_coli_str_K12_MG1655.fna.gz")), fb.read_fasta(os.path.join(GOLDEN, "Shigella_flexneri_2a_01.fna.gz"))
    ctx = _ctx()
    ge, gs = ctx.genomes([ec, sh])
    ctx.set_flag("l2_fast", 0)
    m = fb.Map(ctx, fb.Sketch(ctx, [ge]), gs)
    want = np.fromfile(os.path.join(GOLDEN, "s2e.k16.map"), dtype=fb.MAPPING_DTYPE)
    assert m.rows.tobytes() == want.tobytes()
    p = _paths(ctx, "l2_fast=0")
    assert p["l2.exact_at_bounds"] == p["l2.exact_total"] == m.counters.as_dict()["candidates"]
    assert p["l2.events_nt64"] + p["l2.events_nt128"] + p["l2.events_nt256"] == 0


@pytest.mark.parametrize("n,nt", [(1, 64), (4, 128), (8, 256)])
def test_l2_event_kernel_variants(n, nt):
    """About 1, 4 and 8 candidates per fragment select l2_events_kernel<64 / 128 / 256>; each runs with both rank
    directories and both ways of writing the event codes, and every cell equals the oracle."""
    strains = [[("s%d" % i, synth_genome(71, 1, i, 3000, 60000).tobytes())] for i in range(n + 1)]
    ctx = _ctx()
    w = ctx.windowSize
    hs = ctx.genomes(strains)
    sk = fb.Sketch(ctx, hs[1:])
    _, _, oix = _oracle_index(strains[1:], K, w)
    for nb in (1024, 4096):
        for stage in (1, 0):
            ctx.set_flag("l2e_buckets", nb)
            ctx.set_flag("l2_stage", stage)
            _map_and_compare(ctx, sk, oix, strains[0], hs[0], K, w, L)
            p = _paths(ctx, "n=%d buckets=%d stage=%d" % (n, nb, stage))
            ev = p["l2.events_nt%d" % nt]
            assert ev > 0 and ev == p["l2.dir%d" % nb] == p["l2.staged"] + p["l2.direct"]
            assert p["l2.events_nt64"] + p["l2.events_nt128"] + p["l2.events_nt256"] == ev
            assert p["l2.dir1024"] + p["l2.dir4096"] == ev
            assert (p["l2.staged"] > 0) if stage else (p["l2.direct"] == ev)
            assert p["l2.exact_total"] == 0                  # ordinary strains: the fast path solves every candidate


def _pieces(nfrags, member, cap):
    """Pieces of a query list (map.cu: qsketch_build): whole queries, at most `cap` fragments unless one query alone
    has more, and either all derived from the index or all hashed."""
    n, F, m = 0, None, None
    for nf, mem in zip(nfrags, member):
        if F is None or F + nf > cap or mem != m:
            n, F, m = n + 1, 0, mem
        F += nf
    return n


def test_pieces_splits_and_cgi_passes():
    """Small pieces (1, 7, 64 fragments), pieces halved down to single queries because of their event streams, and the
    identity reduction in passes of 1, 2, 3 queries: identity rows and work counters equal the default run's, which
    equals the oracle; the piece and pass counters show the splits."""
    gs = piece_workload()
    nq = len(gs)
    ctx = _ctx()
    w = ctx.windowSize
    hs = ctx.genomes(gs)
    members = list(range(0, nq, 2))
    sk = fb.Sketch(ctx, [hs[i] for i in members])
    base, tot0, ctr0 = fb.compute_cgi(ctx, sk, hs)
    p0 = _paths(ctx, "default")
    _, sbf, oix = _oracle_index([gs[i] for i in members], K, w)
    exp, nfrags = [], []
    for qi, g in enumerate(gs):
        rows, tq, _ = po.map_genome(oix, g, K, w, L)
        nfrags.append(tq)
        exp += [(qi, gi, c, np.float32(i).view(np.uint32), tq) for gi, c, i in po.cgi(rows, sbf, L)]
    got = [(int(r["qryGenomeId"]), int(r["refGenomeId"]), int(r["countSeq"]), np.float32(r["identity"]).view(np.uint32),
            int(r["totalQueryFragments"])) for r in base]
    assert got == exp and len(got) >= nq
    is_member = [i % 2 == 0 for i in range(nq)]
    assert p0["piece.mapped"] == _pieces(nfrags, is_member, 1 << 18) == nq
    assert max(nfrags) > 64

    def run(tag, **flags):
        for k, v in flags.items():
            ctx.set_flag(k, v)
        res, tot, ctr = fb.compute_cgi(ctx, sk, hs)
        p = _paths(ctx, tag)
        assert res.tobytes() == base.tobytes(), tag
        assert (tot == tot0).all() and ctr.as_dict() == ctr0.as_dict(), tag
        ctx.set_flag("frags_per_piece", 1 << 18); ctx.set_flag("event_bytes_per_piece", 0)
        ctx.set_flag("cgi_table_queries", 0); ctx.set_flag("sketch_reuse", 1)
        return p

    for cap in (1, 7, 64):
        for reuse in (1, 0):
            p = run("frags_per_piece=%d reuse=%d" % (cap, reuse), frags_per_piece=cap, sketch_reuse=reuse)
            assert p["piece.mapped"] == _pieces(nfrags, is_member if reuse else [False] * nq, cap)
    p = run("one piece", sketch_reuse=0)
    assert p["piece.mapped"] == 1 and p["cgi.passes"] == 1
    p = run("event split", sketch_reuse=0, event_bytes_per_piece=1)
    assert p["piece.split_events"] == nq - 1 and p["piece.mapped"] == nq
    for c in (1, 2, 3):
        p = run("cgi_table_queries=%d" % c, sketch_reuse=0, cgi_table_queries=c)
        assert p["piece.mapped"] == 1 and p["cgi.passes"] == math.ceil(nq / c)
    # pieces of merged sketches are packed to the same limit
    ctx.set_flag("frags_per_piece", 64)
    halves = [fb.QuerySketch(ctx, hs[:9], list(range(9))), fb.QuerySketch(ctx, hs[9:], list(range(9, nq)))]
    merged = fb.QuerySketch.merge(ctx, halves)
    res, ctr = fb.compute_cgi_sketched(ctx, sk, [merged])
    p = _paths(ctx, "merged, frags_per_piece=64")
    ctx.set_flag("frags_per_piece", 1 << 18)
    assert res.tobytes() == base.tobytes() and ctr.as_dict() == ctr0.as_dict()
    assert p["piece.mapped"] > 2


def test_cgi_reduction_edges():
    """Identity ties between rows of one fragment and genome (a duplicated region on two contigs and twice in one
    contig; the later row wins), a genome with contigs but no rows, and a sister strain: counts and identity bit
    patterns equal pyoracle.cgi."""
    refs, q = cgi_edge_workload()
    ctx = _ctx()
    w = ctx.windowSize
    hr = ctx.genomes(refs)
    hq = ctx.genome(q)
    sk = fb.Sketch(ctx, hr)
    _, sbf, oix = _oracle_index(refs, K, w)
    rows = _map_and_compare(ctx, sk, oix, q, hq, K, w, L)
    # ties: fragments with two or more rows of equal identity in genome 0
    g0 = rows[rows["refSeqId"] < 2]
    _, cnt = np.unique(np.stack([g0["querySeqId"], g0["nucIdentity"].view(np.int32)]), axis=1, return_counts=True)
    assert (cnt > 1).any()
    assert (g0["refStartPos"] == 3 * (L - 20)).any()          # a row on a bin boundary
    exp =[(g, c, np.float32(i).view(np.uint32)) for g, c, i in po.cgi(rows, sbf, L)]
    res, tot, _ = fb.compute_cgi(ctx, sk, [hq])
    got = [(int(r["refGenomeId"]), int(r["countSeq"]), np.float32(r["identity"]).view(np.uint32)) for r in res]
    assert got == exp and {g for g, _, _ in got} == {0, 2}


# ---------------------------------------------------------------- CPU rehearsal: the oracle side of every workload
if __name__ == "__main__":
    import time
    w = 24                                   # Stat::recommendedWindowSize at k 16, fragLen 3000 (the GPU tests read it from the context)
    t = time.time()
    q, strains = ladder_workload()
    frag = _fragment_sketches(q, K, w, L)
    for n in LADDER_N:
        rec = po.sketch_genomes(strains[:n], K, w)[0]
        hits = _hits_per_fragment(frag, rec)
        rows, _, c = po.map_genome(po.Index(rec), q, K, w, L)
        print("ladder n=%2d hits %s classes %s rows %d cand %d" % (n, hits, predicted_classes(hits), len(rows), c.candidates))
    print("ladder %.1f s" % (time.time() - t))
    for name, wl in (("repeat", repeat_workload), ("sparse", sparse_query_workload), ("tandem", tandem_workload)):
        t = time.time()
        parts = wl()
        ref, queries = parts[0], parts[1:]
        rec, _, oix = _oracle_index([ref], K, w)
        keys, cnt = np.unique(rec["hash"], return_counts=True)
        for qq in queries:
            rows, tq, c = po.map_genome(oix, qq, K, w, L)
            print(name, "records %d max count %d rows %d frags %d hits %d cand %d" % (len(rec), cnt.max(), len(rows), tq, c.hits, c.candidates))
        print(name, "%.1f s" % (time.time() - t))
    for ww, fl in ((30, 45), (31, 45)):
        ref = [("r", synth_genome(67, 1, 0, 0, 20000).tobytes())]
        qq = [("q", synth_genome(67, 1, 1, 10000, 20000).tobytes())]
        rec, _, oix = _oracle_index([ref], K, ww)
        rows, tq, c = po.map_genome(oix, qq, K, ww, fl)
        print("cmw w=%d L=%d rows %d cand %d" % (ww, fl, len(rows), c.candidates))
    t = time.time()
    gs = piece_workload()
    _, sbf, oix = _oracle_index(gs[::2], K, w)
    for qi, g in enumerate(gs):
        rows, tq, _ = po.map_genome(oix, g, K, w, L)
        print("pieces q%d frags %d cgi %s" % (qi, tq, po.cgi(rows, sbf, L)))
    print("pieces %.1f s" % (time.time() - t))
    refs, q = cgi_edge_workload()
    _, sbf, oix = _oracle_index(refs, K, w)
    rows, _, _ = po.map_genome(oix, q, K, w, L)
    print("cgi edges rows %d cgi %s" % (len(rows), po.cgi(rows, sbf, L)))
