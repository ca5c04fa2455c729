"""GPU (-m gpu): the sparse path of the identity reduction (stage H), which reduces a piece's mapping rows by sorting
them instead of filling dense query x genome tables.  Forced sparse against forced dense byte for byte (results and
fragment rows), forced sparse against the oracle and the reference's goldens, and the automatic choice: sparse on a
collection of many small genomes, dense on the few-large-genome workloads.  Every case prints the path counters."""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

import fastani_b200 as fb
import pyoracle as po
from conftest import GOLDEN, ROOT
from fastani_b200 import report, workloads as W
from fastani_b200.synth import synth_genome

pytestmark = pytest.mark.gpu

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")
EC = os.path.join(GOLDEN, "Escherichia_coli_str_K12_MG1655.fna.gz")
SH = os.path.join(GOLDEN, "Shigella_flexneri_2a_01.fna.gz")
L = 3000


def _golden(name):
    op = gzip.open if name.endswith(".gz") else open
    with op(os.path.join(GOLDEN, name), "rt") as f:
        return f.read()


def _ctx(sparse, **params):
    ctx = fb.Context(fb.Parameters(**params))
    ctx.set_flag("count_paths", 1)
    ctx.set_flag("cgi_sparse", sparse)
    return ctx


def _paths(ctx, tag):
    p = ctx.path_counts()
    print(tag, {k: v for k, v in p.items() if v})
    return p


def _check_path(p, sparse):
    """The branch that ran: sparse pieces only, or dense passes only."""
    if sparse == 1:
        assert p["cgi.sparse"] > 0 and p["cgi.passes"] == 0, p
    elif sparse == 0:
        assert p["cgi.sparse"] == 0 and p["cgi.passes"] > 0, p


def _both(run, tag):
    """run(sparse) -> (results, frags, ctx) with the switch forced each way: the same bytes."""
    out = {}
    for sparse in (0, 1):
        res, frags, ctx = run(sparse)
        p = _paths(ctx, "%s cgi_sparse=%d" % (tag, sparse))
        _check_path(p, sparse)
        out[sparse] = (res, frags, p)
    assert out[1][0].tobytes() == out[0][0].tobytes(), tag
    assert out[1][1].tobytes() == out[0][1].tobytes(), tag
    assert len(out[1][0]) > 0
    return out[1]


def _lines(res, names, glen, min_fraction=0.2):
    rows = [(int(x["qryGenomeId"]), int(x["refGenomeId"]), int(x["countSeq"]), int(x["totalQueryFragments"]), x["identity"])
            for x in res]
    return report.output_lines(rows, names, names, glen, glen, L, min_fraction)


def _two_gpus():
    cnt = C.c_int32()
    fb.load_library().bani_device_count(C.byref(cnt))
    return cnt.value >= 2


def _cli(d, args, sparse=None, budget=None):
    env = dict(os.environ)
    for v in ("BANI_CLI_HOST_CGI", "BANI_INDEX_BUDGET", "BANI_QUERY_BUDGET", "BANI_CGI_SPARSE"):
        env.pop(v, None)
    if sparse is not None:
        env["BANI_CGI_SPARSE"] = str(sparse)
    if budget:
        env["BANI_INDEX_BUDGET"] = str(budget)
    return subprocess.run([EXE] + args + ["-t", "8"], cwd=d, capture_output=True, text=True, timeout=900, env=env)


def _ok(r):
    assert r.returncode == 0, r.stderr[-3000:]
    return r


# ---------------------------------------------------------------------------------------- forced sparse == forced dense
@pytest.fixture(scope="module")
def real():
    return fb.read_fasta(EC), fb.read_fasta(SH)


def test_real_pair_sparse_equals_dense_the_oracle_and_the_goldens(real):
    ec, sh = real
    names = {"e": "data/Escherichia_coli_str_K12_MG1655.fna", "s": "data/Shigella_flexneri_2a_01.fna"}
    for tag, (q, qn), (r, rn) in (("e2s", (ec, "e"), (sh, "s")), ("s2e", (sh, "s"), (ec, "e"))):
        def run(sparse):
            ctx = _ctx(sparse)
            gq, gr = ctx.genomes([q, r])
            sk = fb.Sketch(ctx, [gr])
            res, _, frags = fb.compute_cgi_sketched(ctx, sk, [fb.QuerySketch(ctx, [gq], [0], hint=sk)], fragments=True)
            run.sk, run.ctx, run.rows = sk, ctx, fb.Map(ctx, sk, gq).rows
            return res, frags, ctx
        res, frags, _ = _both(run, tag)
        # bit for bit with the host rule over the same mapping rows
        want = po.cgi(run.rows, run.sk.sequencesByFileInfo, L)
        have = [(int(x["refGenomeId"]), int(x["countSeq"]), np.float32(x["identity"])) for x in res]
        assert [(g, c, np.float32(i).view(np.uint32)) for g, c, i in have] == [(g, c, np.float32(i).view(np.uint32)) for g, c, i in want]
        if tag == "e2s":
            lines = report.visual_lines(frags, [names[qn]], [names[rn]],
                                        [report.fragment_lengths([len(s) for _, s in q], L, 16, run.ctx.windowSize)],
                                        [l for _, l in run.sk.metadata], run.sk.sequencesByFileInfo, L)
            assert "\n".join(lines) + "\n" == _golden("e2s.txt.visual")


def test_edge_contigs_sparse_equals_dense(real):
    """edge_mixed.fa (short contigs, N runs, lower case) at fragLen 1000, hashed and index-derived sketches."""
    ec, _ = real
    edge = fb.read_fasta(os.path.join(GOLDEN, "edge_mixed.fa"))
    other = [("ec_a", ec[0][1][:40000]), ("ec_b", edge[3][1] + ec[0][1][50000:52000].lower())]

    def run(sparse):
        ctx = _ctx(sparse, minReadLength=1000)
        ga, gb = ctx.genomes([edge, other])
        sk = fb.Sketch(ctx, [ga, gb])
        hashed = fb.QuerySketch(ctx, [ga, gb], [0, 1])
        derived = fb.QuerySketch.from_index(ctx, sk, [1, 0], [2, 3])
        res, _, frags = fb.compute_cgi_sketched(ctx, sk, [hashed, derived], fragments=True)
        return res, frags, ctx
    _, frags, _ = _both(run, "edge_mixed")
    assert len(frags) > 10


@pytest.fixture(scope="module")
def cfg4():
    specs = W.config4(clusters=2)
    ctx = fb.Context(fb.Parameters())
    contigs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs]
    ctx.close()
    return specs, contigs


@pytest.mark.parametrize("flags", [{}, {"frags_per_piece": 2500, "max_hits_per_piece": 1}, {"frags_per_piece": 700}])
def test_cfg4_sketches_pieces_and_splits_sparse_equals_dense_and_the_golden(cfg4, flags):
    """40 x 40 multi-contig drafts, ten query sketches; pieces of 700 or 2500 fragments, and pieces split down to one
    query each because of their hit counts."""
    specs, contigs = cfg4

    def run(sparse):
        ctx = _ctx(sparse)
        for k, v in flags.items():
            ctx.set_flag(k, v)
        hs = ctx.genomes(contigs)
        sk = fb.Sketch(ctx, hs)
        qs = [fb.QuerySketch(ctx, hs[i:i + 4], list(range(i, i + 4)), hint=sk) for i in range(0, 40, 4)]
        res, _, frags = fb.compute_cgi_sketched(ctx, sk, qs, fragments=True)
        run.res2, _ = fb.compute_cgi_sketched(ctx, sk, qs)
        assert run.res2.tobytes() == res.tobytes()
        return res, frags, ctx
    res, _, p = _both(run, "cfg4 %s" % flags)
    if "frags_per_piece" in flags:
        assert p["piece.mapped"] > 10
    if flags.get("max_hits_per_piece") == 1:
        assert p["piece.split_hits"] > 0
    names = [s.name + ".fna" for s in specs]
    glen = [report.genome_length(s.contig_lengths(), L) for s in specs]
    assert sorted(_lines(res, names, glen)) == sorted(_golden("cfg4_40x40.txt").splitlines())


def test_cfg4_and_bench_queries_stay_dense_on_auto(cfg4):
    """A few large genomes per piece: the dense output is smaller than the rows, so auto keeps the dense path."""
    specs, contigs = cfg4
    ctx = _ctx(-1)
    hs = ctx.genomes(contigs)
    sk = fb.Sketch(ctx, hs)
    res, _, _ = fb.compute_cgi(ctx, sk, hs)
    p = _paths(ctx, "cfg4 auto")
    assert p["cgi.sparse"] == 0 and p["cgi.passes"] > 0
    ctx.set_flag("cgi_sparse", 1)
    res1, _, _ = fb.compute_cgi(ctx, sk, hs)
    assert res1.tobytes() == res.tobytes()
    # bench.py's config 3 shape: 8 queries against references of 5 Mbp strains
    specs3 = W.config3(clusters=2, strains=20)
    ctx = _ctx(-1)
    g3 = [ctx.genome(s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length))) for s in specs3]
    sk3 = fb.Sketch(ctx, g3)
    qi = W.sample_queries(2, 20, 8)
    res3, _, _ = fb.compute_cgi(ctx, sk3, [g3[i] for i in qi])
    p = _paths(ctx, "config 3 shape auto")
    assert p["cgi.sparse"] == 0 and p["cgi.passes"] > 0 and len(res3) > 0


def test_cfg5_k21_sparse_equals_dense_and_the_goldens(tmp_path):
    specs = W.config3(clusters=2, strains=10)
    names = [s.name + ".fna" for s in specs]
    k = 21

    def run(sparse):
        ctx = _ctx(sparse, kmerSize=k)
        hs = [ctx.genome(s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length))) for s in specs]
        sk = fb.Sketch(ctx, hs)
        res, _, frags = fb.compute_cgi_sketched(ctx, sk, [fb.QuerySketch(ctx, hs, list(range(20)), hint=sk)], fragments=True)
        return res, frags, ctx
    res, _, _ = _both(run, "cfg5 k21")
    glen = [report.genome_length([s.length], L) for s in specs]
    want = _golden("cfg5_20x20.k21.L3000.txt")
    assert sorted(_lines(res, names, glen)) == sorted(want.splitlines())
    ctx = fb.Context(fb.Parameters())
    for s in specs:
        W.write_fasta(str(tmp_path / (s.name + ".fna")), s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)))
    ctx.close()
    open(tmp_path / "all.txt", "w").write("\n".join(names) + "\n")
    _ok(_cli(tmp_path, ["--ql", "all.txt", "--rl", "all.txt", "-o", "m.txt", "-k", "21", "--fragLen", "3000", "--minFraction", "0.2",
                        "--matrix", "--gpus", "1"], sparse=1))
    assert sorted(open(tmp_path / "m.txt").read().splitlines()) == sorted(want.splitlines())
    assert open(tmp_path / "m.txt.matrix").read() == _golden("cfg5_20x20.k21.L3000.txt.matrix")


def test_identity_tie_in_one_bin_goes_to_the_later_fragment():
    """Query fragments 3 and 7 are the same 3 kb: both win the same bin of the reference with the same identity.  The
    sorted path keeps the one the dense 64-bit maximum keeps: the larger querySeqId."""
    base = synth_genome(31, 1, 0, 0, 60000).tobytes()
    x = base[9000:12000]
    qseq = base[:21000] + x + base[24000:30000]
    rseq = synth_genome(31, 1, 1, 20000, 60000).tobytes()

    def run(sparse):
        ctx = _ctx(sparse)
        gq, gr = ctx.genomes([[("q", qseq)], [("r", rseq)]])
        sk = fb.Sketch(ctx, [gr])
        run.rows = fb.Map(ctx, sk, gq).rows
        res, _, frags = fb.compute_cgi_sketched(ctx, sk, [fb.QuerySketch(ctx, [gq], [0], hint=sk)], fragments=True)
        return res, frags, ctx
    _, frags, _ = _both(run, "tie")
    rows = run.rows
    r3, r7 = rows[rows["querySeqId"] == 3], rows[rows["querySeqId"] == 7]
    best3, best7 = r3[np.argmax(r3["nucIdentity"])], r7[np.argmax(r7["nucIdentity"])]
    assert best3["nucIdentity"] == best7["nucIdentity"] and best3["refStartPos"] == best7["refStartPos"]
    at = frags[(frags["refSeqId"] == best3["refSeqId"]) & (frags["refStartPos"] // 2980 == best3["refStartPos"] // 2980)]
    assert len(at) == 1 and at[0]["querySeqId"] == 7 and at[0]["identity"] == best3["nucIdentity"]


# ---------------------------------------------------------------------------------------- many small genomes, auto
@pytest.fixture(scope="module")
def small(tmp_path_factory):
    specs = W.small_genomes()
    d = tmp_path_factory.mktemp("small")
    ctx = fb.Context(fb.Parameters())
    contigs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs]
    ctx.close()
    for s, c in zip(specs, contigs):
        W.write_fasta(str(d / (s.name + ".fna")), c)
    open(d / "all.txt", "w").write("\n".join(s.name + ".fna" for s in specs) + "\n")
    return specs, contigs, d


def test_small_genomes_auto_takes_the_sparse_path_and_matches_the_golden(small):
    specs, contigs, d = small
    names = [s.name + ".fna" for s in specs]
    glen = [report.genome_length(s.contig_lengths(), L) for s in specs]
    want = sorted(_golden("small_3000.txt.gz").splitlines())
    ctx = _ctx(-1)
    hs = ctx.genomes(contigs)
    sk = fb.Sketch(ctx, hs)
    res, _, _ = fb.compute_cgi(ctx, sk, hs)
    p = _paths(ctx, "small auto")
    assert p["cgi.sparse"] > 0 and p["cgi.passes"] == 0
    assert sorted(_lines(res, names, glen)) == want
    ctx.set_flag("cgi_sparse", 0)
    res0, _, _ = fb.compute_cgi(ctx, sk, hs)
    _check_path(_paths(ctx, "small dense"), 0)
    assert res0.tobytes() == res.tobytes()
    # the command line, chosen per piece and forced dense
    for sparse, out in ((None, "a.txt"), (0, "d.txt")):
        _ok(_cli(d, ["--ql", "all.txt", "--rl", "all.txt", "-o", out, "--matrix", "--gpus", "1"], sparse=sparse))
        assert sorted(open(d / out).read().splitlines()) == want, out
        assert open(d / (out + ".matrix")).read() == _golden("small_3000.txt.matrix.gz"), out


# ---------------------------------------------------------------------------------------- command line, forced sparse
def test_cli_sparse_visualize_reproduces_the_reference_goldens(tmp_path):
    os.mkdir(tmp_path / "data")
    for n in ("Escherichia_coli_str_K12_MG1655.fna", "Shigella_flexneri_2a_01.fna"):
        os.symlink(os.path.join(GOLDEN, n + ".gz"), tmp_path / "data" / n)
    E, S = "data/Escherichia_coli_str_K12_MG1655.fna", "data/Shigella_flexneri_2a_01.fna"
    _ok(_cli(tmp_path, ["-q", E, "-r", S, "-o", "e2s.txt", "--matrix", "--visualize", "--gpus", "1"], sparse=1))
    for ext in ("", ".matrix", ".visual"):
        assert open(tmp_path / ("e2s.txt" + ext)).read() == _golden("e2s.txt" + ext), ext


@pytest.fixture(scope="module")
def cfg4_dir(tmp_path_factory, cfg4):
    specs, contigs = cfg4
    d = tmp_path_factory.mktemp("cfg4s")
    for s, c in zip(specs, contigs):
        W.write_fasta(str(d / (s.name + ".fna")), c)
    open(d / "all.txt", "w").write("\n".join(s.name + ".fna" for s in specs) + "\n")
    return d


def _chunks(stderr):
    return [int(l.split("reference chunks : ")[1].split(",")[0]) for l in stderr.splitlines() if "reference chunks : " in l]


def test_cli_sparse_chunked_build_and_load_reproduce_the_golden(cfg4_dir):
    d = cfg4_dir
    want = sorted(_golden("cfg4_40x40.txt").splitlines())
    r = _ok(_cli(d, ["--ql", "all.txt", "--rl", "all.txt", "-o", "c.txt", "--gpus", "1"], sparse=1, budget="300M"))
    assert _chunks(r.stderr)[0] > 1
    assert sorted(open(d / "c.txt").read().splitlines()) == want
    _ok(_cli(d, ["--ql", "all.txt", "--rl", "all.txt", "-o", "s.txt", "--gpus", "1", "--saveIndex", "db"]))
    r = _ok(_cli(d, ["--ql", "all.txt", "--loadIndex", "db", "-o", "l.txt"], sparse=1, budget="300M"))
    assert _chunks(r.stderr)[0] > 1
    assert sorted(open(d / "l.txt").read().splitlines()) == want


def test_bad_switch_values_are_refused(cfg4_dir):
    r = _cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "x.txt", "--gpus", "1"], sparse="x")
    assert r.returncode == 1 and "BANI_CGI_SPARSE" in r.stderr, r.stderr[-2000:]
    old = os.environ.get("BANI_CGI_SPARSE")
    os.environ["BANI_CGI_SPARSE"] = "2"
    try:
        with pytest.raises(fb.BaniError):
            fb.Context(fb.Parameters())
    finally:
        if old is None:
            del os.environ["BANI_CGI_SPARSE"]
        else:
            os.environ["BANI_CGI_SPARSE"] = old
    ctx = fb.Context(fb.Parameters())
    for bad in (-2, 2):
        with pytest.raises(fb.BaniError):
            ctx.set_flag("cgi_sparse", bad)


# ---------------------------------------------------------------------------------------- two GPUs
def test_two_gpus_sparse_equals_dense(cfg4, cfg4_dir):
    if not _two_gpus():
        pytest.skip("needs two GPUs")
    specs, contigs = cfg4
    # the sharded Python path: each GPU maps every query against its shard of the references
    from fastani_b200 import parallel
    for rank in range(2):
        mine = parallel.shard_refs(len(contigs), 2, rank)
        got = {}
        for sparse in (0, 1):
            ctx = fb.Context(fb.Parameters(), device=rank)
            ctx.set_flag("count_paths", 1); ctx.set_flag("cgi_sparse", sparse)
            hs = ctx.genomes(contigs)
            sk = fb.Sketch(ctx, [hs[i] for i in mine])
            got[sparse], _, frags = fb.compute_cgi_sketched(ctx, sk, [fb.QuerySketch(ctx, hs, list(range(40)))], fragments=True)
            got[sparse] = (got[sparse].tobytes(), frags.tobytes())
            _check_path(_paths(ctx, "rank %d cgi_sparse=%d" % (rank, sparse)), sparse)
        assert got[0] == got[1]
    r = _ok(_cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "g2.txt", "--gpus", "2"], sparse=1))
    assert sorted(open(cfg4_dir / "g2.txt").read().splitlines()) == sorted(_golden("cfg4_40x40.txt").splitlines())
