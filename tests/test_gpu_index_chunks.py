"""GPU (-m gpu): saved indexes loaded in runs of genomes that fit a budget, and shard files mapped on fewer GPUs than they
were saved with.  Budgets are forced small, so no test comes near the device's memory: the range load against the index
built from the same genomes, the per-genome checksums, query sketches read from a file, the Python loop and the command
line against the goldens of the unmodified reference."""
import os
import shutil
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


@pytest.fixture(scope="module")
def saved(cfg4, tmp_path_factory):
    """The 40 cfg4 genomes saved as one index file."""
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    path = str(tmp_path_factory.mktemp("ix") / "db.idx")
    fb.Sketch(ctx, ctx.genomes(contigs)).save(path)
    ctx.close()
    return path


def _need(info, first, end):
    """Device bytes of loading genomes [first, end): the build footprint of their exact counts, without sketch staging."""
    m = int(info["genome_records"][first:end].sum())
    return fb.index_footprint(m, m, int(info["genome_contigs"][first:end].sum()), int(info["genome_bits"][first:end].sum()), 0)[0]


def _predict_taken(info, first, budget):
    t = 0
    while first + t < info["n_genomes"] and _need(info, first, first + t + 1) <= budget:
        t += 1
    return t


def _predict_runs(info, budget):
    runs, first = [], 0
    while first < info["n_genomes"]:
        t = _predict_taken(info, first, budget)
        if t == 0:
            return None
        runs.append((first, first + t))
        first += t
    return runs


def test_range_loads_equal_builds(cfg4, saved):
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    hs = ctx.genomes(contigs)
    info = fb.index_file_info(saved)
    assert info["version"] == 3 and info["n_genomes"] == 40 and info["w"] == ctx.windowSize
    hashed = lambda: fb.QuerySketch(ctx, hs[:3], [0, 1, 2])
    for first in (0, 7, 39):
        for want in sorted({1, min(5, 40 - first), 40 - first}):
            budget = _need(info, first, first + want)
            assert _predict_taken(info, first, budget) == want
            live0 = ctx.mem_stats()["live"]
            sk, taken, peak = fb.Sketch.load_budget(ctx, saved, first, budget)
            st = ctx.mem_stats()
            assert taken == want
            assert 0 < peak <= budget and st["peak_live"] - live0 == peak
            ref = fb.Sketch(ctx, hs[first:first + taken])
            assert sk.stats() == ref.stats() and (sk.minimizerIndex() == ref.minimizerIndex()).all()
            assert sk.sequencesByFileInfo == ref.sequencesByFileInfo
            assert [m[1] for m in sk.metadata] == [m[1] for m in ref.metadata]
            assert fb.compute_cgi_sketched(ctx, sk, [hashed()])[0].tobytes() == fb.compute_cgi_sketched(ctx, ref, [hashed()])[0].tobytes()
            members = list(range(min(taken, 4)))
            d1, d2 = fb.QuerySketch.from_index(ctx, sk, members), fb.QuerySketch.from_index(ctx, ref, members)
            assert d1.info() == d2.info()
            assert fb.compute_cgi_sketched(ctx, sk, [d1])[0].tobytes() == fb.compute_cgi_sketched(ctx, ref, [d2])[0].tobytes()
            sk.close(); ref.close()
    with pytest.raises(fb.BaniError) as e:
        fb.Sketch.load_budget(ctx, saved, 7, _need(info, 7, 8) - 1)
    assert e.value.code == -4 and "does not fit" in str(e.value)
    with pytest.raises(fb.BaniError):
        fb.Sketch.load_budget(ctx, saved, 40, 1 << 40)


def _offsets(info):
    n_c, n_g, m = info["n_contigs"], info["n_genomes"], info["n_minimizers"]
    off_hash = 128 + 4 * n_c + 4 * n_g + 4 * (n_c + 1)
    return off_hash, off_hash + 4 * m


def test_per_genome_checksums_and_version_2(cfg4, saved, tmp_path):
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    hs = ctx.genomes(contigs)
    info = fb.index_file_info(saved)
    blob = open(saved, "rb").read()
    _, off_wpos = _offsets(info)
    rec0 = np.concatenate([[0], np.cumsum(info["genome_records"])]).astype(int)
    j = 7
    bad = bytearray(blob)
    bad[off_wpos + 4 * (rec0[j] + 5) + 1] ^= 0x01              # one byte inside genome 7's wpos slice
    path = str(tmp_path / "bad.idx")
    open(path, "wb").write(bytes(bad))
    big = 1 << 40
    with pytest.raises(fb.BaniError) as e:                       # a range that covers genome 7
        fb.Sketch.load_budget(ctx, path, 5, big)
    assert "genome 7" in str(e.value)
    with pytest.raises(fb.BaniError):
        fb.QuerySketch.from_index_file(ctx, path, [3, 7])
    with pytest.raises(fb.BaniError):                            # and the whole load
        fb.Sketch.load(ctx, path)
    # ranges that do not cover it load and map as the index of their genomes
    q = lambda: fb.QuerySketch(ctx, hs[:2], [0, 1])
    sk, taken, _ = fb.Sketch.load_budget(ctx, path, 0, _need(info, 0, j))
    assert taken == j
    assert fb.compute_cgi_sketched(ctx, sk, [q()])[0].tobytes() == fb.compute_cgi_sketched(ctx, fb.Sketch(ctx, hs[:j]), [q()])[0].tobytes()
    sk, taken, _ = fb.Sketch.load_budget(ctx, path, j + 1, big)
    assert taken == 40 - j - 1
    assert fb.compute_cgi_sketched(ctx, sk, [q()])[0].tobytes() == fb.compute_cgi_sketched(ctx, fb.Sketch(ctx, hs[j + 1:]), [q()])[0].tobytes()
    # the same file in version 2: no table or genome checksums, version 2, the whole-file checksum recomputed
    n_g = info["n_genomes"]
    v2 = bytearray(blob[:len(blob) - 8 - 8 - 8 * n_g])
    v2[8:16] = np.array([2], "<u8").tobytes()
    v2 += np.array([int(np.frombuffer(bytes(v2), "<u4").astype(np.uint64).sum())], "<u8").tobytes()
    p2 = str(tmp_path / "v2.idx")
    open(p2, "wb").write(bytes(v2))
    assert fb.index_file_info(p2)["version"] == 2
    whole, full = fb.Sketch.load(ctx, p2), fb.Sketch(ctx, hs)
    assert (whole.minimizerIndex() == full.minimizerIndex()).all()
    assert fb.compute_cgi_sketched(ctx, whole, [q()])[0].tobytes() == fb.compute_cgi_sketched(ctx, full, [q()])[0].tobytes()
    for call in (lambda: fb.Sketch.load_budget(ctx, p2, 0, big), lambda: fb.QuerySketch.from_index_file(ctx, p2, [0])):
        with pytest.raises(fb.BaniError) as e:
            call()
        assert e.value.code == -1 and "save it again" in str(e.value)


def test_query_sketches_from_the_file_equal_those_of_the_loaded_index(cfg4, saved):
    ctx = fb.Context(fb.Parameters())
    whole = fb.Sketch.load(ctx, saved)
    ords = [12, 0, 39, 5, 12, 21]
    a = fb.QuerySketch.from_index_file(ctx, saved, ords)
    b = fb.QuerySketch.from_index(ctx, whole, ords)
    assert a.info() == b.info()
    assert fb.compute_cgi_sketched(ctx, whole, [a])[0].tobytes() == fb.compute_cgi_sketched(ctx, whole, [b])[0].tobytes()
    ids = [100 + i for i in range(len(ords))]
    a = fb.QuerySketch.from_index_file(ctx, saved, ords, ids)
    b = fb.QuerySketch.from_index(ctx, whole, ords, ids)
    assert fb.compute_cgi_sketched(ctx, whole, [a])[0].tobytes() == fb.compute_cgi_sketched(ctx, whole, [b])[0].tobytes()
    for o in ([40], [-1]):
        with pytest.raises(fb.BaniError):
            fb.QuerySketch.from_index_file(ctx, saved, o)


def _budget_for_runs(info, n):
    """A budget whose loads take the file in n > 1 runs, three quarters up the range that gives n (the run plan, which
    counts expected minimizers and sketch staging, must not find a genome too large for it)."""
    count = lambda b: len(_predict_runs(info, b) or [0] * (1 << 30))

    def smallest(m):                              # smallest budget with at most m runs
        lo, hi = 1 << 20, 1 << 40
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if count(mid) <= m:
                hi = mid
            else:
                lo = mid
        return hi
    bot, top = smallest(n), smallest(n - 1) - 1
    budget = bot + (top - bot) * 3 // 4
    assert count(budget) == n
    return budget


@pytest.mark.parametrize("n_chunks,query_blocks", [(1, 1), (2, 1), (5, 1), (40, 1), (5, 3)])
def test_python_loop_from_the_file_equals_one_index_and_the_golden(cfg4, saved, n_chunks, query_blocks):
    specs, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    hs = ctx.genomes(contigs)
    want, _, _ = fb.compute_cgi(ctx, fb.Sketch(ctx, hs), hs)
    want = want[np.lexsort((want["refGenomeId"], want["qryGenomeId"]))]
    qs = [fb.QuerySketch(ctx, hs[i:i + 4], list(range(i, i + 4))) for i in range(0, 40, 4)]
    for h in hs:
        h.close()
    info = fb.index_file_info(saved)
    qbytes = [q.info()["export_bytes"] for q in qs]
    qbudget = None if query_blocks == 1 else sum(qbytes) // 3 + max(qbytes)
    budget = None if n_chunks == 1 else _budget_for_runs(info, n_chunks)
    got, plan = fb.compute_cgi_from_index_file(ctx, saved, qs, index_budget=budget, query_budget=qbudget)
    assert len(plan["blocks"]) == query_blocks
    assert plan["chunks"] == (_predict_runs(info, budget) if budget else [(0, 40)])
    assert got.tobytes() == want.tobytes()
    names = [s.name + ".fna" for s in specs]
    glen = [report.genome_length(s.contig_lengths(), L) for s in specs]
    rows = [(int(x["qryGenomeId"]), int(x["refGenomeId"]), int(x["countSeq"]), int(x["totalQueryFragments"]), x["identity"]) for x in got]
    assert sorted(report.output_lines(rows, names, names, glen, glen, L)) == sorted(_golden_lines("cfg4_40x40.txt"))
    if n_chunks > 1:
        assert len(set(plan["device_bytes"])) == 1, plan["device_bytes"]


# ---------------------------------------------------------------------------------------- command line
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


def test_cli_chunked_load_equals_the_golden(cfg4_dir, tmp_path):
    d = cfg4_dir
    r = _cli(d, ["--ql", "all.txt", "--rl", "all.txt", "-o", "s.txt", "--gpus", "1", "--saveIndex", "db"])
    assert r.returncode == 0 and _chunk_counts(r.stderr) == [1], r.stderr[-2000:]
    golden = sorted(_golden_lines("cfg4_40x40.txt"))
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "db", "-o", "c.txt"], budget="300M", qbudget="4M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert _chunk_counts(r.stderr)[0] > 1 and _block_counts(r.stderr)[0] > 1
    assert sorted(open(d / "c.txt").read().splitlines()) == golden
    # a chunked load refuses --visualize as a chunked build does
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "db", "-o", "v.txt", "--visualize"], budget="300M")
    assert r.returncode == 1 and "--visualize" in r.stderr and "chunk" in r.stderr, r.stderr[-2000:]
    # no FASTA at all: every query is a genome of the (one-shard) index, its sketch is read from the file
    for f in ("db.meta", "db.0of1.idx", "all.txt"):
        shutil.copy(d / f, tmp_path / f)
    r = _cli(tmp_path, ["--ql", "all.txt", "--loadIndex", "db", "-o", "c.txt"], budget="300M", qbudget="4M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert "reading 0 genome files" in r.stderr and _chunk_counts(r.stderr)[0] > 1
    assert open(tmp_path / "c.txt").read() == open(d / "c.txt").read()


def _write_shards(d, specs, contigs, prefix, block):
    """A 2-shard index as --saveIndex --gpus 2 writes it: one Sketch.save file per shard and the metadata file (version 1:
    interleaved, 2: blocks of the list)."""
    n = len(specs)
    shards = [list(range(n // 2)), list(range(n // 2, n))] if block else [list(range(0, n, 2)), list(range(1, n, 2))]
    ctx = fb.Context(fb.Parameters(kmerSize=K, minReadLength=L))
    for s, sh in enumerate(shards):
        fb.Sketch(ctx, ctx.genomes([contigs[j] for j in sh])).save(str(d / ("%s.%dof2.idx" % (prefix, s))))
    lines = ["BANI_INDEX_META\t%d" % (2 if block else 1), "%d\t%d\t%d\t2\t%d" % (K, L, ctx.windowSize, n)]
    lines += [s.name + ".fna" for s in specs]
    for sh in shards:
        names = [nm for j in sh for nm, _ in contigs[j]]
        lines += [str(len(names))] + names
    open(d / (prefix + ".meta"), "w").write("\n".join(lines) + "\n")
    ctx.close()


@pytest.mark.parametrize("block", [False, True])
def test_cli_two_shards_on_one_gpu(cfg4, cfg4_dir, block):
    specs, contigs = cfg4
    d = cfg4_dir
    prefix = "two_block" if block else "two"
    _write_shards(d, specs, contigs, prefix, block)
    golden = sorted(_golden_lines("cfg4_40x40.txt"))
    for budget in (None, "300M"):
        r = _cli(d, ["--ql", "all.txt", "--loadIndex", prefix, "-o", "t.txt", "--gpus", "1"], budget=budget)
        assert r.returncode == 0, r.stderr[-3000:]
        counts = _chunk_counts(r.stderr)
        assert len(counts) == 2 and (all(c > 1 for c in counts) if budget else counts == [1, 1])
        assert sorted(open(d / "t.txt").read().splitlines()) == golden


@pytest.mark.parametrize("block", [False, True])
def test_cli_two_shards_on_two_gpus(cfg4, cfg4_dir, block):
    import ctypes as C
    cnt = C.c_int32()
    fb.load_library().bani_device_count(C.byref(cnt))
    if cnt.value < 2:
        pytest.skip("needs two GPUs")
    specs, contigs = cfg4
    d = cfg4_dir
    prefix = "two2_block" if block else "two2"
    _write_shards(d, specs, contigs, prefix, block)
    golden = sorted(_golden_lines("cfg4_40x40.txt"))
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", prefix, "-o", "t2.txt", "--gpus", "2"], budget="300M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert sorted(open(d / "t2.txt").read().splitlines()) == golden


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


def test_cli_chunked_load_cfg5_matrix_equals_the_golden(cfg5_dir):
    d = cfg5_dir
    common = ["-k", "16", "--fragLen", "3000", "--minFraction", "0.2", "--matrix", "--gpus", "1", "-s"]
    r = _cli(d, ["--ql", "all.txt", "--rl", "all.txt", "-o", "s.txt", "--saveIndex", "db"] + common)
    assert r.returncode == 0, r.stderr[-3000:]
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "db", "-o", "m.txt"] + common, budget="400M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert _chunk_counts(r.stderr)[0] > 1
    assert sorted(open(d / "m.txt").read().splitlines()) == sorted(_golden_lines("cfg5_20x20.k16.L3000.txt"))
    assert open(d / "m.txt.matrix").read() == open(os.path.join(GOLDEN, "cfg5_20x20.k16.L3000.txt.matrix")).read()
