"""GPU (-m gpu): reference lists built and mapped in chunks.  Budgets are forced small through the switches, so no test
comes near the device's memory: the budgeted index build, the Python chunk loop and the command line against the
goldens of the unmodified reference."""
import os
import subprocess

import numpy as np
import pytest

import fastani_b200 as fb
from conftest import GOLDEN, ROOT
from fastani_b200 import report, workloads as W

pytestmark = pytest.mark.gpu

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")
K, L = 16, 3000


def _golden_lines(name):
    return open(os.path.join(GOLDEN, name)).read().splitlines()


@pytest.fixture(scope="module")
def cfg4():
    specs = W.config4(clusters=2)
    ctx = fb.Context(fb.Parameters())
    contigs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs]
    ctx.close()
    return specs, contigs


def _staging_cap(pos, w):
    return min(pos, int(3.0 * pos / (w + 1)) + 65536)


def _spans(contigs):
    """Per genome: (contigs, hashed positions, validity bits), as the index build counts them."""
    out = []
    for cl in contigs:
        lens = [len(s) for _, s in cl]
        out.append((len(lens), sum(x - K + 1 for x in lens if x >= K), sum((x + 31) & ~31 for x in lens)))
    return out


def _predict_taken(spans, rec_end, budget, w):
    """The prefix bani_index_build_budget keeps: the launch takes the longest prefix whose expected build fits (the first
    genome: its staging and tables), then the longest prefix of that whose exact build -- record counts of the full
    index -- fits with the staging and the contig tables of the launch."""
    n, nc, pos, bits = 0, 0, 0, 0
    for g, (c, p, b) in enumerate(spans):
        cap = _staging_cap(pos + p, w)
        m = int(2.0 * (pos + p) / (w + 1))
        need = fb.index_footprint(0, 0, nc + c, bits + b, cap)[0] if g == 0 else fb.index_footprint(m, m, nc + c, bits + b, cap)[0]
        if need > budget:
            break
        n, nc, pos, bits = g + 1, nc + c, pos + p, bits + b
    cap = _staging_cap(pos, w)
    t = 0
    for g in range(n):
        m = rec_end[g]
        if m > cap or fb.index_footprint(m, m, nc, bits, cap)[0] > budget:      # tables of every launched genome
            break
        t = g + 1
    return t


def test_budgeted_build_takes_the_predicted_prefix(cfg4):
    specs, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    w = ctx.windowSize
    hs = ctx.genomes(contigs)
    full = fb.Sketch(ctx, hs)
    rec = full.minimizerIndex()
    sbf = full.sequencesByFileInfo
    counts = np.bincount(rec["seqId"], minlength=sbf[-1])
    rec_end = [int(counts[:e].sum()) for e in sbf]
    spans = _spans(contigs)

    def budget_for(n):                            # the smallest budget that admits n genomes, by bisection
        lo, hi = 1 << 20, 1 << 36
        while hi - lo > (1 << 16):
            mid = (lo + hi) // 2
            if _predict_taken(spans, rec_end, mid, w) >= n:
                hi = mid
            else:
                lo = mid
        return hi

    for n in (1, 7, 40):
        budget = budget_for(n)
        want = _predict_taken(spans, rec_end, budget, w)
        assert want == n
        live0 = ctx.mem_stats()["live"]
        sk, taken, peak = fb.Sketch.build_budget(ctx, hs, budget)
        st = ctx.mem_stats()
        assert taken == want
        assert 0 < peak <= budget and st["peak_live"] - live0 == peak
        ref = fb.Sketch(ctx, hs[:taken])
        assert sk.stats() == ref.stats() and (sk.minimizerIndex() == ref.minimizerIndex()).all()
        assert sk.sequencesByFileInfo == ref.sequencesByFileInfo
        # the cut index maps like the one built from exactly those genomes, with hashed query sketches and with sketches
        # derived from the index (stage A': they read the validity bitmap the cut shrinks)
        r1, _ = fb.compute_cgi_sketched(ctx, sk, [fb.QuerySketch(ctx, hs[:3], [0, 1, 2])])
        r2, _ = fb.compute_cgi_sketched(ctx, ref, [fb.QuerySketch(ctx, hs[:3], [0, 1, 2])])
        assert r1.tobytes() == r2.tobytes()
        members = list(range(min(taken, 5)))
        d1 = fb.QuerySketch.from_index(ctx, sk, members)
        d2 = fb.QuerySketch.from_index(ctx, ref, members)
        nh = min(taken + 1, len(hs))                 # the members, and one genome that is not (hashed) where there is one
        h1 = fb.QuerySketch(ctx, hs[:nh], list(range(nh)), hint=sk)
        h2 = fb.QuerySketch(ctx, hs[:nh], list(range(nh)), hint=ref)
        assert d1.info() == d2.info() and h1.info() == h2.info()
        assert fb.compute_cgi_sketched(ctx, sk, [d1, h1])[0].tobytes() == fb.compute_cgi_sketched(ctx, ref, [d2, h2])[0].tobytes()
        assert fb.compute_cgi_sketched(ctx, sk, [d1])[0].tobytes() == fb.compute_cgi_sketched(ctx, ref, [fb.QuerySketch(ctx, hs[:len(members)], members)])[0].tobytes()
        sk.close(); ref.close()
    with pytest.raises(fb.BaniError) as e:
        fb.Sketch.build_budget(ctx, hs, budget_for(1) // 4)
    assert e.value.code == -4 and "does not fit" in str(e.value)


def _budget_for_chunks(lens, conts, n, w):
    """A budget whose plan has n chunks, near the top of the range that gives n (slack for record counts above the expected
    density)."""
    def chunks(b):
        try:
            return len(fb.plan_chunks(lens, conts, K, w, b))
        except fb.BaniError:
            return 1 << 30
    def smallest(m):                              # smallest budget with at most m chunks
        lo, hi = 1 << 20, 1 << 40
        while hi - lo > (1 << 16):
            mid = (lo + hi) // 2
            if chunks(mid) <= m:
                hi = mid
            else:
                lo = mid
        return hi
    top = smallest(n - 1) - (1 << 16) if n > 1 else 1 << 40
    assert chunks(top) == n
    bot = smallest(n)
    return bot + (top - bot) * 3 // 4


@pytest.mark.parametrize("n_chunks,query_budget_blocks", [(1, 1), (2, 1), (5, 1), (40, 1), (5, 3)])
def test_python_chunk_loop_equals_one_index_and_the_golden(cfg4, n_chunks, query_budget_blocks):
    specs, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    w = ctx.windowSize
    hs = ctx.genomes(contigs)
    want, _, _ = fb.compute_cgi(ctx, fb.Sketch(ctx, hs), hs)
    want = want[np.lexsort((want["refGenomeId"], want["qryGenomeId"]))]
    qs = [fb.QuerySketch(ctx, hs[i:i + 4], list(range(i, i + 4))) for i in range(0, 40, 4)]     # hashed, 10 sketches
    for h in hs:
        h.close()
    qbytes = [q.info()["export_bytes"] for q in qs]
    qbudget = None if query_budget_blocks == 1 else sum(qbytes) // 3 + max(qbytes)
    lens = [sum(len(s) for _, s in cl) for cl in contigs]
    budget = _budget_for_chunks(lens, [len(cl) for cl in contigs], n_chunks, w)
    got, plan = fb.compute_cgi_chunked(ctx, contigs, qs, index_budget=budget, query_budget=qbudget)
    assert len(plan["chunks"]) == n_chunks and len(plan["blocks"]) == query_budget_blocks
    assert plan["chunks"][0][0] == 0 and plan["chunks"][-1][1] == 40
    assert got.tobytes() == want.tobytes()
    names = [s.name + ".fna" for s in specs]
    glen = [report.genome_length(s.contig_lengths(), L) for s in specs]
    rows = [(int(x["qryGenomeId"]), int(x["refGenomeId"]), int(x["countSeq"]), int(x["totalQueryFragments"]), x["identity"]) for x in got]
    assert sorted(report.output_lines(rows, names, names, glen, glen, L)) == sorted(_golden_lines("cfg4_40x40.txt"))
    if n_chunks > 1:
        # every chunk hands its index and the cached blocks back: the device holds the same bytes at every boundary
        assert len(set(plan["device_bytes"])) == 1, plan["device_bytes"]


def test_budget_switches_and_environment(cfg4):
    """The switches replace the derived budgets; a small run plans into one chunk with the derived ones."""
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    lens = [sum(len(s) for _, s in cl) for cl in contigs]
    conts = [len(cl) for cl in contigs]
    chunks, blocks, ib = ctx.plan_run(lens, conts, lens)
    assert chunks == [(0, 40)] and blocks == [(0, 40)] and ib > 0
    ctx.set_flag("index_bytes_budget", 300 << 20)
    ctx.set_flag("query_sketch_budget", 4 << 20)
    chunks, blocks, ib = ctx.plan_run(lens, conts, lens)
    assert ib == 300 << 20 and len(chunks) > 1 and len(blocks) > 1
    assert chunks == fb.plan_chunks(lens, conts, K, ctx.windowSize, ib)
    assert ctx.plan_run(lens, conts, lens, index_budget=1 << 40)[0] == [(0, 40)]      # an explicit budget overrides the switch
    ctx.set_flag("index_bytes_budget", 0)
    ctx.set_flag("query_sketch_budget", 0)
    assert ctx.plan_run(lens, conts, lens)[:2] == ([(0, 40)], [(0, 40)])
    with pytest.raises(fb.BaniError):
        ctx.set_flag("index_bytes_budget", -1)


@pytest.fixture(scope="module")
def cfg4_dir(tmp_path_factory, cfg4):
    specs, contigs = cfg4
    d = tmp_path_factory.mktemp("cfg4")
    for s, c in zip(specs, contigs):
        W.write_fasta(str(d / (s.name + ".fna")), c)
    open(d / "all.txt", "w").write("\n".join(s.name + ".fna" for s in specs) + "\n")
    return d


def _cli(d, args, budget=None, qbudget=None):
    env = dict(os.environ)
    env.pop("BANI_INDEX_BUDGET", None); env.pop("BANI_QUERY_BUDGET", None)
    if budget:
        env["BANI_INDEX_BUDGET"] = str(budget)
    if qbudget:
        env["BANI_QUERY_BUDGET"] = str(qbudget)
    return subprocess.run([EXE] + args + ["-t", "8"], cwd=d, capture_output=True, text=True, timeout=900, env=env)


def _chunk_counts(stderr):
    return [int(l.split("reference chunks : ")[1].split(",")[0]) for l in stderr.splitlines() if "reference chunks : " in l]


def _block_counts(stderr):
    return [int(l.split("query blocks : ")[1].split(" ")[0]) for l in stderr.splitlines() if "query blocks : " in l]


def test_cli_chunked_cfg4_equals_the_golden(cfg4_dir):
    r = _cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "c.txt", "--gpus", "1"], budget="300M", qbudget="4M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert _chunk_counts(r.stderr)[0] > 1 and _block_counts(r.stderr)[0] > 1
    assert sorted(open(cfg4_dir / "c.txt").read().splitlines()) == sorted(_golden_lines("cfg4_40x40.txt"))
    # refused when more than one chunk is needed
    for extra, msg in ((["--visualize"], "--visualize"), (["--saveIndex", "db"], "--saveIndex")):
        r = _cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "v.txt", "--gpus", "1"] + extra, budget="300M")
        assert r.returncode == 1 and msg in r.stderr and "chunk" in r.stderr, r.stderr[-2000:]
    # without the variable: one chunk, and the same commands run
    r = _cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "v.txt", "--gpus", "1", "--saveIndex", "db"])
    assert r.returncode == 0 and _chunk_counts(r.stderr) == [1], r.stderr[-2000:]
    # a bad value is refused where the context is created
    r = _cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "v.txt", "--gpus", "1"], budget="lots")
    assert r.returncode == 1 and "BANI_INDEX_BUDGET" in r.stderr


@pytest.mark.parametrize("partition", ["interleave", "block"])
def test_cli_chunked_two_gpus(cfg4_dir, partition):
    import ctypes as C
    cnt = C.c_int32()
    fb.load_library().bani_device_count(C.byref(cnt))
    if cnt.value < 2:
        pytest.skip("needs two GPUs")
    r = _cli(cfg4_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "p.txt", "--gpus", "2", "--partition", partition], budget="300M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert all(c > 1 for c in _chunk_counts(r.stderr)) and len(_chunk_counts(r.stderr)) == 2
    assert sorted(open(cfg4_dir / "p.txt").read().splitlines()) == sorted(_golden_lines("cfg4_40x40.txt"))


@pytest.fixture(scope="module")
def cfg5_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("cfg5")
    specs = W.config3(clusters=2, strains=10)
    ctx = fb.Context(fb.Parameters())
    for s in specs:
        W.write_fasta(str(d / (s.name + ".fna")), s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)))
    open(d / "all.txt", "w").write("\n".join(s.name + ".fna" for s in specs) + "\n")
    ctx.close()
    return d


def test_cli_chunked_cfg5_matrix_equals_the_golden(cfg5_dir):
    r = _cli(cfg5_dir, ["--ql", "all.txt", "--rl", "all.txt", "-o", "m.txt", "-k", "16", "--fragLen", "3000", "--minFraction", "0.2",
                        "--matrix", "--gpus", "1", "-s"], budget="400M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert _chunk_counts(r.stderr)[0] > 1
    assert sorted(open(cfg5_dir / "m.txt").read().splitlines()) == sorted(_golden_lines("cfg5_20x20.k16.L3000.txt"))
    assert open(cfg5_dir / "m.txt.matrix").read() == open(os.path.join(GOLDEN, "cfg5_20x20.k16.L3000.txt.matrix")).read()
