"""Adding genomes to a saved index from the command line (--loadIndex with -r/--rl and --saveIndex), without a GPU: the
combinations the command line refuses are refused with exit 1 and their message.  The CLI parses its options and reads the
index's .meta before it looks for a device, so hand-written .meta files are enough."""
import os
import subprocess

import pytest

import fastani_b200 as fb
from conftest import ROOT

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")


def _meta(d, prefix, version=1, k=16, frag_len=3000, shards=1, refs=("old0.fa", "old1.fa")):
    w = fb.Parameters(kmerSize=k, minReadLength=frag_len).recommendedWindowSize()
    lines = ["BANI_INDEX_META\t%d" % version, "%d\t%d\t%d\t%d\t%d" % (k, frag_len, w, shards, len(refs))] + list(refs)
    for s in range(shards):
        names = ["c%d" % j for j in range(s, len(refs), shards)]
        lines += [str(len(names))] + names
    open(os.path.join(d, prefix + ".meta"), "w").write("\n".join(lines) + "\n")


@pytest.fixture
def work(tmp_path):
    d = str(tmp_path)
    for name in ("q.fa", "new.fa"):
        open(os.path.join(d, name), "w").write(">x\n" + "ACGT" * 100 + "\n")
    open(os.path.join(d, "q.txt"), "w").write("q.fa\n")
    open(os.path.join(d, "new.txt"), "w").write("new.fa\n")
    _meta(d, "db")
    return d


def _run(d, args):
    return subprocess.run([EXE] + args, cwd=d, capture_output=True, text=True, timeout=120)


def _refused(r, text):
    assert r.returncode == 1, (r.returncode, r.stderr[-2000:])
    assert text in r.stderr, r.stderr[-2000:]
    assert "no CUDA device" not in r.stderr


def test_same_prefix_is_refused(work):
    r = _run(work, ["--ql", "q.txt", "--loadIndex", "db", "--rl", "new.txt", "--saveIndex", "db", "-o", "out.txt"])
    _refused(r, "is the index given to --loadIndex")


def test_block_partitioned_index_of_two_shards_is_refused(work):
    _meta(work, "blk", version=2, shards=2)
    r = _run(work, ["--ql", "q.txt", "--loadIndex", "blk", "-r", "new.fa", "--saveIndex", "blk2", "-o", "out.txt"])
    _refused(r, "blocks of the reference list")
    assert not [f for f in os.listdir(work) if f.startswith("blk2")]


def test_added_genomes_without_save_index_are_refused(work):
    r = _run(work, ["--ql", "q.txt", "--loadIndex", "db", "--rl", "new.txt", "-o", "out.txt"])
    _refused(r, "--loadIndex replaces -r/--rl")


def test_save_index_without_added_genomes_stays_refused(work):
    r = _run(work, ["--ql", "q.txt", "--loadIndex", "db", "--saveIndex", "db2", "-o", "out.txt"])
    _refused(r, "--saveIndex and --loadIndex exclude each other")


def test_index_of_another_k_is_refused(work):
    _meta(work, "k21", k=21)
    r = _run(work, ["--ql", "q.txt", "--loadIndex", "k21", "--rl", "new.txt", "--saveIndex", "db2", "-o", "out.txt"])
    _refused(r, "the saved index was built with k 21")
    assert not [f for f in os.listdir(work) if f.startswith("db2")]


def test_missing_added_genome_file_is_refused(work):
    open(os.path.join(work, "gone.txt"), "w").write("gone.fa\n")
    r = _run(work, ["--ql", "q.txt", "--loadIndex", "db", "--rl", "gone.txt", "--saveIndex", "db2", "-o", "out.txt"])
    _refused(r, "Could not open gone.fa")
