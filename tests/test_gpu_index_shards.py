"""GPU (-m gpu): --loadIndex runs against saved indexes of several shard files whose queries are genomes of the index
(member queries).  Their sketches are derived from the shard file that holds each genome, so no FASTA is read.  Every run
is made in a directory that holds only the index and the list, and its outputs are compared with the goldens of the
unmodified reference and, byte for byte, with the same run where every query is read and hashed (BANI_CLI_HOST_CGI=1,
with the files present).  Budgets are forced small where chunks are wanted, so no test comes near the device's memory."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

import fastani_b200 as fb
from conftest import GOLDEN, ROOT
from fastani_b200 import workloads as W

pytestmark = pytest.mark.gpu

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")
K, L = 16, 3000


def _golden_lines(name):
    return open(os.path.join(GOLDEN, name)).read().splitlines()


def _split(n, S, block):
    """The saved partition: list position j goes to shard j mod S, or (block) to the contiguous range that holds it."""
    return [list(range(n * s // S, n * (s + 1) // S)) for s in range(S)] if block else [list(range(s, n, S)) for s in range(S)]


def _write_shards(d, names, contigs, prefix, S, block):
    """An S-shard index as --saveIndex on S GPUs writes it: one Sketch.save file per shard and the metadata file (version 1:
    interleaved, 2: blocks of the list)."""
    shards = _split(len(names), S, block)
    ctx = fb.Context(fb.Parameters(kmerSize=K, minReadLength=L))
    for s, sh in enumerate(shards):
        sk = fb.Sketch(ctx, ctx.genomes([contigs[j] for j in sh]))
        sk.save(str(d / ("%s.%dof%d.idx" % (prefix, s, S))))
        sk.close()
    lines = ["BANI_INDEX_META\t%d" % (2 if block else 1), "%d\t%d\t%d\t%d\t%d" % (K, L, ctx.windowSize, S, len(names))]
    lines += names
    for sh in shards:
        cn = [nm for j in sh for nm, _ in contigs[j]]
        lines += [str(len(cn))] + cn
    open(d / (prefix + ".meta"), "w").write("\n".join(lines) + "\n")
    ctx.close()
    return prefix


def _index_only(src, dst, prefix, lists=("all.txt",)):
    """A fresh directory with the index and the query list, and no genome file."""
    dst.mkdir(exist_ok=True)
    for f in os.listdir(src):
        if f == prefix + ".meta" or (f.startswith(prefix + ".") and f.endswith(".idx")) or f in lists:
            shutil.copy(src / f, dst / f)
    assert not [f for f in os.listdir(dst) if f.endswith(".fna")]
    return dst


def _cli(d, args, budget=None, qbudget=None, hashed=False):
    env = dict(os.environ)
    for v in ("BANI_CLI_HOST_CGI", "BANI_INDEX_BUDGET", "BANI_QUERY_BUDGET", "BANI_CGI_SPARSE"):
        env.pop(v, None)
    if budget:
        env["BANI_INDEX_BUDGET"] = str(budget)
    if qbudget:
        env["BANI_QUERY_BUDGET"] = str(qbudget)
    if hashed:
        env["BANI_CLI_HOST_CGI"] = "1"
    return subprocess.run([EXE] + args + ["-t", "8"], cwd=d, capture_output=True, text=True, timeout=900, env=env)


def _ok(r):
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _reading(stderr):
    return [int(l.split("Time spent reading ")[1].split(" ")[0]) for l in stderr.splitlines() if "Time spent reading " in l]


def _chunk_counts(stderr):
    return [int(l.split("reference chunks : ")[1].split(",")[0]) for l in stderr.splitlines() if "reference chunks : " in l]


def _block_counts(stderr):
    return [int(l.split("query blocks : ")[1].split(" ")[0]) for l in stderr.splitlines() if "query blocks : " in l]


def _n_gpus():
    cnt = C.c_int32()
    fb.load_library().bani_device_count(C.byref(cnt))
    return cnt.value


def _same(a, b, exts=("",)):
    for ext in exts:
        assert open(str(a) + ext, "rb").read() == open(str(b) + ext, "rb").read(), ext


@pytest.fixture(scope="module")
def cfg4(tmp_path_factory):
    """The config-4 slice (40 genomes of 2 clusters) written as FASTA, with its list files."""
    specs = W.config4(clusters=2)
    ctx = fb.Context(fb.Parameters())
    contigs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs]
    ctx.close()
    d = tmp_path_factory.mktemp("cfg4s")
    names = [s.name + ".fna" for s in specs]
    for nm, c in zip(names, contigs):
        W.write_fasta(str(d / nm), c)
    for f, sel in (("all.txt", names), ("first25.txt", names[:25]), ("last15.txt", names[25:])):
        open(d / f, "w").write("\n".join(sel) + "\n")
    return d, names, contigs


def _cfg4_index(cfg4, S, block):
    d, names, contigs = cfg4
    prefix = "s%d%s" % (S, "b" if block else "i")
    if not os.path.exists(d / (prefix + ".meta")):
        _write_shards(d, names, contigs, prefix, S, block)
    return prefix


CASES = [(2, False), (2, True), (3, False), (3, True)]


@pytest.mark.parametrize("S,block", CASES)
def test_shards_on_one_gpu_read_no_fasta(cfg4, tmp_path, S, block):
    d = cfg4[0]
    prefix = _cfg4_index(cfg4, S, block)
    e = _index_only(d, tmp_path / "ix", prefix)
    args = ["--ql", "all.txt", "--loadIndex", prefix, "-o", "t.txt", "--gpus", "1"]
    r = _ok(_cli(e, args))
    assert _reading(r.stderr) == [0] and _chunk_counts(r.stderr) == [1] * S, r.stderr[-3000:]
    assert sorted(open(e / "t.txt").read().splitlines()) == sorted(_golden_lines("cfg4_40x40.txt"))
    r = _ok(_cli(d, args, hashed=True))
    assert _reading(r.stderr) == [40]
    _same(e / "t.txt", d / "t.txt")


@pytest.mark.parametrize("S,block", CASES)
def test_chunked_shards_read_no_fasta(cfg4, tmp_path, S, block):
    d = cfg4[0]
    prefix = _cfg4_index(cfg4, S, block)
    e = _index_only(d, tmp_path / "ix", prefix)
    args = ["--ql", "all.txt", "--loadIndex", prefix, "-o", "c.txt", "--gpus", "1"]
    r = _ok(_cli(e, args, budget="300M", qbudget="4M"))
    assert _reading(r.stderr) == [0], r.stderr[-3000:]
    assert len(_chunk_counts(r.stderr)) == S and all(c > 1 for c in _chunk_counts(r.stderr)) and all(b > 1 for b in _block_counts(r.stderr))
    assert sorted(open(e / "c.txt").read().splitlines()) == sorted(_golden_lines("cfg4_40x40.txt"))
    r = _ok(_cli(d, args, budget="300M", qbudget="4M", hashed=True))
    assert _reading(r.stderr) == [40]
    _same(e / "c.txt", d / "c.txt")


def test_cfg5_matrix_and_sanity_check_from_two_shards(tmp_path):
    specs = W.config3(clusters=2, strains=10)
    ctx = fb.Context(fb.Parameters())
    contigs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs]
    ctx.close()
    names = [s.name + ".fna" for s in specs]
    _write_shards(tmp_path, names, contigs, "db", 2, False)
    open(tmp_path / "all.txt", "w").write("\n".join(names) + "\n")
    r = _ok(_cli(tmp_path, ["--ql", "all.txt", "--loadIndex", "db", "-o", "m.txt", "-k", "16", "--fragLen", "3000", "--minFraction", "0.2",
                            "--matrix", "--gpus", "1", "-s"]))
    assert _reading(r.stderr) == [0] and "exceeds maximum thresholds" not in r.stderr
    assert sorted(open(tmp_path / "m.txt").read().splitlines()) == sorted(_golden_lines("cfg5_20x20.k16.L3000.txt"))
    assert open(tmp_path / "m.txt.matrix").read() == open(os.path.join(GOLDEN, "cfg5_20x20.k16.L3000.txt.matrix")).read()


def test_visualize_from_two_shards(cfg4, tmp_path):
    d = cfg4[0]
    prefix = _cfg4_index(cfg4, 2, False)
    e = _index_only(d, tmp_path / "ix", prefix)
    args = ["--ql", "all.txt", "--loadIndex", prefix, "-o", "v.txt", "--gpus", "1", "--matrix", "--visualize"]
    r = _ok(_cli(e, args))
    assert _reading(r.stderr) == [0]
    r = _ok(_cli(d, args, hashed=True))
    assert _reading(r.stderr) == [40]
    _same(e / "v.txt", d / "v.txt", ("", ".matrix", ".visual"))
    assert len(open(e / "v.txt.visual").read().splitlines()) > 40 * 900


def test_members_of_one_shard_and_a_renamed_copy(cfg4, tmp_path):
    d, names, _ = cfg4
    prefix = _cfg4_index(cfg4, 2, False)
    e = _index_only(d, tmp_path / "ix", prefix)
    shutil.copy(d / names[4], e / "copy.fna")                   # the same genome under another path: not a member
    open(e / "q.txt", "w").write("\n".join(names[0::2] + ["copy.fna"]) + "\n")
    r = _ok(_cli(e, ["--ql", "q.txt", "--loadIndex", prefix, "-o", "q.out", "--gpus", "1"]))
    assert _reading(r.stderr) == [1], r.stderr[-3000:]
    lines = [l.split("\t") for l in open(e / "q.out").read().splitlines()]
    member = [l[1:] for l in lines if l[0] == names[4]]
    copy = [l[1:] for l in lines if l[0] == "copy.fna"]
    assert len(member) > 1 and copy == member
    golden = [l for l in _golden_lines("cfg4_40x40.txt") if l.split("\t")[0] in names[0::2]]
    assert sorted("\t".join(l) for l in lines if l[0] != "copy.fna") == sorted(golden)


def test_extended_index_loads_without_fasta(cfg4, tmp_path):
    d, names, contigs = cfg4
    if not os.path.exists(d / "e25.meta"):
        _write_shards(d, names[:25], contigs[:25], "e25", 2, False)
    r = _ok(_cli(d, ["--ql", "all.txt", "--loadIndex", "e25", "--rl", "last15.txt", "--saveIndex", "e40", "-o", "e.txt", "--gpus", "1"]))
    assert _reading(r.stderr) == [15], r.stderr[-3000:]
    golden = sorted(_golden_lines("cfg4_40x40.txt"))
    assert sorted(open(d / "e.txt").read().splitlines()) == golden
    e = _index_only(d, tmp_path / "ix", "e40")
    r = _ok(_cli(e, ["--ql", "all.txt", "--loadIndex", "e40", "-o", "x.txt", "--gpus", "1"]))
    assert _reading(r.stderr) == [0]
    assert sorted(open(e / "x.txt").read().splitlines()) == golden
    _same(e / "x.txt", d / "e.txt")


def test_corrupt_member_fails_and_names_it(cfg4, tmp_path):
    d, names, _ = cfg4
    prefix = _cfg4_index(cfg4, 2, False)
    e = _index_only(d, tmp_path / "ix", prefix)
    path = e / (prefix + ".1of2.idx")
    info = fb.index_file_info(str(path))
    n_c, n_g, m = info["n_contigs"], info["n_genomes"], info["n_minimizers"]
    off_wpos = 128 + 4 * n_c + 4 * n_g + 4 * (n_c + 1) + 4 * m
    o = 3                                                        # ordinal 3 of shard 1 is list position 7
    rec0 = int(info["genome_records"][:o].sum())
    assert int(info["genome_records"][o]) > 10
    blob = bytearray(open(path, "rb").read())
    blob[off_wpos + 4 * (rec0 + 5) + 1] ^= 0x01
    open(path, "wb").write(bytes(blob))
    r = _cli(e, ["--ql", "all.txt", "--loadIndex", prefix, "-o", "bad.txt", "--gpus", "1"])
    assert r.returncode == 1, r.stderr[-3000:]
    assert names[7] in r.stderr and "genome 3" in r.stderr, r.stderr[-3000:]
    assert not [f for f in os.listdir(e) if f.startswith("bad.txt")]


def test_three_shards_on_two_gpus(cfg4, tmp_path):
    if _n_gpus() < 2:
        pytest.skip("needs two GPUs")
    d = cfg4[0]
    prefix = _cfg4_index(cfg4, 3, False)
    e = _index_only(d, tmp_path / "ix", prefix)
    args = ["--ql", "all.txt", "--loadIndex", prefix, "-o", "g.txt", "--gpus", "2"]
    r = _ok(_cli(e, args))
    assert _reading(r.stderr) == [0]
    assert sorted(open(e / "g.txt").read().splitlines()) == sorted(_golden_lines("cfg4_40x40.txt"))
    _ok(_cli(d, args, hashed=True))
    _same(e / "g.txt", d / "g.txt")
