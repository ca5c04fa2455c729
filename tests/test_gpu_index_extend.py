"""GPU (-m gpu): genomes added to a saved index file (bani_index_file_extend, and --loadIndex with -r/--rl and --saveIndex on
the command line).  The extended file must equal, byte for byte, the file saved from a fresh build of the whole list, so
every check here compares SHA-256 digests or whole files with that fresh save; the command line is also checked against the
golden of the unmodified reference.  Budgets are forced small, so no test comes near the device's memory."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

import fastani_b200 as fb
from conftest import GOLDEN, ROOT
from fastani_b200 import workloads as W

pytestmark = pytest.mark.gpu

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")
K, L = 16, 3000


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


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
def fresh(cfg4, tmp_path_factory):
    """Sketch(all 40 genomes).save(): what every extension must equal."""
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    path = str(tmp_path_factory.mktemp("fresh") / "all.idx")
    fb.Sketch(ctx, ctx.genomes(contigs)).save(path)
    ctx.close()
    return path


def _save(ctx, contigs, path):
    sk = fb.Sketch(ctx, ctx.genomes(contigs))
    sk.save(path)
    sk.close()
    return path


def test_extensions_equal_the_fresh_save(cfg4, fresh, tmp_path):
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    want = _sha(fresh)
    for n in (1, 7, 25, 39):
        old = _save(ctx, contigs[:n], str(tmp_path / ("first%d.idx" % n)))
        added = fb.Sketch(ctx, ctx.genomes(contigs[n:]))
        out = str(tmp_path / ("ext%d.idx" % n))
        fb.index_file_extend(ctx, old, added, out)
        assert _sha(out) == want, n
        assert fb.index_file_info(out)["n_genomes"] == 40
    # two extensions in a row: 25 -> 32 -> 40
    mid = str(tmp_path / "mid.idx")
    fb.index_file_extend(ctx, str(tmp_path / "first25.idx"), fb.Sketch(ctx, ctx.genomes(contigs[25:32])), mid)
    assert _sha(mid) == _sha(_save(ctx, contigs[:32], str(tmp_path / "first32.idx")))
    end = str(tmp_path / "end.idx")
    fb.index_file_extend(ctx, mid, fb.Sketch(ctx, ctx.genomes(contigs[32:])), end)
    assert _sha(end) == want
    # the extended file loads and maps as the index built from all 40
    whole, full = fb.Sketch.load(ctx, end), fb.Sketch(ctx, ctx.genomes(contigs))
    assert (whole.minimizerIndex() == full.minimizerIndex()).all()
    q = lambda: fb.QuerySketch.from_index_file(ctx, end, [0, 24, 25, 39])
    assert fb.compute_cgi_sketched(ctx, whole, [q()])[0].tobytes() == fb.compute_cgi_sketched(ctx, full, [q()])[0].tobytes()


def _acgt(rng, n):
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()


def _bitmap_words(path, first_genome):
    """The validity bitmap words of genomes [first_genome, end) of a saved file, trailing word excluded."""
    info = fb.index_file_info(path)
    n_c, n_g, m = info["n_contigs"], info["n_genomes"], info["n_minimizers"]
    off_bits = 128 + 4 * n_c + 4 * n_g + 4 * (n_c + 1) + 8 * m
    w0 = int(info["genome_bits"][:first_genome].sum()) // 32
    w1 = int(info["genome_bits"].sum()) // 32
    blob = open(path, "rb").read()
    return np.frombuffer(blob[off_bits + 4 * w0:off_bits + 4 * w1], "<u4")


@pytest.mark.parametrize("kind", ["shorter_than_k", "no_full_window"])
def test_added_genomes_without_records(cfg4, tmp_path, kind):
    """Genomes that add no record: contigs shorter than k have no position (the added index has no bitmap, its words are
    zero); contigs of k .. k + w - 2 bases have valid positions but no full window (the bitmap holds bits, no record)."""
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    w = ctx.windowSize
    rng = np.random.default_rng(7)
    lens = [[1, K - 1, 5], [K - 2]] if kind == "shorter_than_k" else [[K, K + w - 2, K + 3], [K + w // 2]]
    small = [[("s%d_%d" % (g, i), _acgt(rng, n)) for i, n in enumerate(ls)] for g, ls in enumerate(lens)]
    old = _save(ctx, contigs[:5], str(tmp_path / "old.idx"))
    added = fb.Sketch(ctx, ctx.genomes(small))
    assert added.stats()["n_minimizers"] == 0
    out = str(tmp_path / "ext.idx")
    fb.index_file_extend(ctx, old, added, out)
    fresh = _save(ctx, contigs[:5] + small, str(tmp_path / "fresh.idx"))
    assert _sha(out) == _sha(fresh)
    bits = _bitmap_words(fresh, 5)
    assert len(bits) > 0 and (bits.any() if kind == "no_full_window" else not bits.any())
    # and followed by genomes with records again
    out2 = str(tmp_path / "ext2.idx")
    fb.index_file_extend(ctx, out, fb.Sketch(ctx, ctx.genomes(contigs[5:8])), out2)
    assert _sha(out2) == _sha(_save(ctx, contigs[:5] + small + contigs[5:8], str(tmp_path / "fresh2.idx")))


def _refused(call, out, code, words):
    with pytest.raises(fb.BaniError) as e:
        call()
    assert e.value.code == code and all(w in str(e.value) for w in words), str(e.value)
    assert not os.path.exists(out)


def test_refusals_leave_no_file(cfg4, tmp_path):
    _, contigs = cfg4
    ctx = fb.Context(fb.Parameters())
    old = _save(ctx, contigs[:10], str(tmp_path / "old.idx"))
    added = fb.Sketch(ctx, ctx.genomes(contigs[10:12]))
    out = str(tmp_path / "out.idx")
    # an old file without records saved no bitmap
    empty = _save(ctx, [[("tiny", b"ACGTACGT")]], str(tmp_path / "empty.idx"))
    _refused(lambda: fb.index_file_extend(ctx, empty, added, out), out, -1, ["build it again"])
    # one flipped byte in genome 7's wpos slice: found while the file is copied, named, and nothing is left
    info = fb.index_file_info(old)
    n_c, n_g, m = info["n_contigs"], info["n_genomes"], info["n_minimizers"]
    off_wpos = 128 + 4 * n_c + 4 * n_g + 4 * (n_c + 1) + 4 * m
    rec0 = int(info["genome_records"][:7].sum())
    blob = open(old, "rb").read()
    bad = bytearray(blob)
    bad[off_wpos + 4 * (rec0 + 3) + 1] ^= 0x01
    badp = str(tmp_path / "bad.idx")
    open(badp, "wb").write(bytes(bad))
    _refused(lambda: fb.index_file_extend(ctx, badp, added, out), out, -1, ["genome 7"])
    # version 2: no per-genome sums
    v2 = bytearray(blob[:len(blob) - 8 - 8 - 8 * n_g])
    v2[8:16] = np.array([2], "<u8").tobytes()
    v2 += np.array([int(np.frombuffer(bytes(v2), "<u4").astype(np.uint64).sum())], "<u8").tobytes()
    p2 = str(tmp_path / "v2.idx")
    open(p2, "wb").write(bytes(v2))
    _refused(lambda: fb.index_file_extend(ctx, p2, added, out), out, -1, ["save it again"])
    # contexts of other parameters
    for prm in (fb.Parameters(kmerSize=21), fb.Parameters(minReadLength=2000)):
        c2 = fb.Context(prm)
        a2 = fb.Sketch(c2, c2.genomes(contigs[10:12]))
        _refused(lambda: fb.index_file_extend(c2, old, a2, out), out, -1, ["other parameters"])
        a2.close(); c2.close()
    # the file being extended as the output: refused before anything is written, the file intact
    _refused(lambda: fb.index_file_extend(ctx, old, added, old), str(tmp_path / "never"), -1, ["another path"])
    assert open(old, "rb").read() == blob
    fb.index_file_extend(ctx, old, added, out)                  # and the intact file extends
    assert _sha(out) == _sha(_save(ctx, contigs[:12], str(tmp_path / "fresh12.idx")))


# ---------------------------------------------------------------------------------------- command line
@pytest.fixture(scope="module")
def cfg4_dir(tmp_path_factory, cfg4):
    specs, contigs = cfg4
    d = tmp_path_factory.mktemp("cfg4x")
    for s, c in zip(specs, contigs):
        W.write_fasta(str(d / (s.name + ".fna")), c)
    names = [s.name + ".fna" for s in specs]
    for f, sel in (("all.txt", names), ("first25.txt", names[:25]), ("last15.txt", names[25:])):
        open(d / f, "w").write("\n".join(sel) + "\n")
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


def _same_files(d, a, b, names):
    for n in names:
        assert open(d / (a + n), "rb").read() == open(d / (b + n), "rb").read(), a + n


def test_cli_one_shard(cfg4_dir):
    d = cfg4_dir
    golden = sorted(_golden_lines("cfg4_40x40.txt"))
    r = _cli(d, ["--ql", "all.txt", "--rl", "first25.txt", "--saveIndex", "a", "-o", "a.txt", "--gpus", "1"])
    assert r.returncode == 0, r.stderr[-3000:]
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "a", "--rl", "last15.txt", "--saveIndex", "b", "-o", "b.txt", "--gpus", "1"])
    assert r.returncode == 0, r.stderr[-3000:]
    assert "reading 15 genome files" in r.stderr and "15 genome(s) and" in r.stderr, r.stderr[-3000:]
    assert sorted(open(d / "b.txt").read().splitlines()) == golden
    r = _cli(d, ["--ql", "all.txt", "--rl", "all.txt", "--saveIndex", "c", "-o", "c.txt", "--gpus", "1"])
    assert r.returncode == 0, r.stderr[-3000:]
    _same_files(d, "b", "c", [".meta", ".0of1.idx"])
    # the extended index is an index like any other: loaded in chunks, its member queries read from it
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "b", "-o", "bc.txt"], budget="300M", qbudget="4M")
    assert r.returncode == 0, r.stderr[-3000:]
    assert _chunk_counts(r.stderr)[0] > 1
    assert sorted(open(d / "bc.txt").read().splitlines()) == golden


def _write_shards(d, specs, contigs, prefix):
    """A 2-shard interleaved index as --saveIndex --gpus 2 writes it: one Sketch.save file per shard and the metadata."""
    n = len(specs)
    shards = [list(range(0, n, 2)), list(range(1, n, 2))]
    ctx = fb.Context(fb.Parameters(kmerSize=K, minReadLength=L))
    for s, sh in enumerate(shards):
        fb.Sketch(ctx, ctx.genomes([contigs[j] for j in sh])).save(str(d / ("%s.%dof2.idx" % (prefix, s))))
    lines = ["BANI_INDEX_META\t1", "%d\t%d\t%d\t2\t%d" % (K, L, ctx.windowSize, n)]
    lines += [s.name + ".fna" for s in specs]
    for sh in shards:
        names = [nm for j in sh for nm, _ in contigs[j]]
        lines += [str(len(names))] + names
    open(d / (prefix + ".meta"), "w").write("\n".join(lines) + "\n")
    ctx.close()


def test_cli_two_interleaved_shards_on_one_gpu(cfg4, cfg4_dir):
    specs, contigs = cfg4
    d = cfg4_dir
    _write_shards(d, specs[:25], contigs[:25], "i25")
    _write_shards(d, specs, contigs, "i40")
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "i25", "--rl", "last15.txt", "--saveIndex", "i25x", "-o", "i.txt", "--gpus", "1"])
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stderr.count("minimizers added to") == 2
    _same_files(d, "i25x", "i40", [".meta", ".0of2.idx", ".1of2.idx"])
    assert sorted(open(d / "i.txt").read().splitlines()) == sorted(_golden_lines("cfg4_40x40.txt"))


def test_cli_added_genomes_larger_than_the_budget(cfg4_dir):
    d = cfg4_dir
    r = _cli(d, ["--ql", "all.txt", "--rl", "first25.txt", "--saveIndex", "t", "-o", "t.txt", "--gpus", "1"])
    assert r.returncode == 0, r.stderr[-3000:]
    r = _cli(d, ["--ql", "all.txt", "--loadIndex", "t", "--rl", "last15.txt", "--saveIndex", "tx", "-o", "tx.txt", "--gpus", "1"],
             budget="1M")
    assert r.returncode == 1, r.stderr[-3000:]
    assert "shard 0" in r.stderr and "add fewer genomes per run" in r.stderr, r.stderr[-3000:]
    assert not [f for f in os.listdir(d) if f.startswith("tx.")]
