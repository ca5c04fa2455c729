"""GPU (-m gpu): the fragment-row mode of the identity reduction (bani_map_cgi_sketch_frags) -- the 2-way fragment
mappings behind every ANI value -- against the host rule (pyoracle.cgi over the mapping rows), the reference's .visual
goldens, and the command line's per-query host path (BANI_CLI_HOST_CGI=1)."""
import ctypes as C
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


def _expected_frags(ctx, sk, genomes, qids, frag_len):
    """What the host rule makes of the device's mapping rows, query by query, in the order given."""
    parts = []
    for g, q in zip(genomes, qids):
        _, (vr, vq, vs, vi) = po.cgi(fb.Map(ctx, sk, g).rows, sk.sequencesByFileInfo, frag_len, want_visual=True)
        f = np.zeros(len(vr), fb.FRAG_DTYPE)
        f["qryGenomeId"], f["querySeqId"], f["refSeqId"], f["refStartPos"], f["identity"] = q, vq, vr, vs, vi
        parts.append(f)
    return np.concatenate(parts) if parts else np.empty(0, fb.FRAG_DTYPE)


def _check_invariants(res, frags, sbf):
    """Per (query, genome) pair: countSeq frags, whose float32 sum in order over countSeq is the identity."""
    gen = np.searchsorted(np.asarray(sbf), frags["refSeqId"], side="right")
    assert int(res["countSeq"].sum()) == len(frags)
    for r in res:
        sel = frags[(frags["qryGenomeId"] == r["qryGenomeId"]) & (gen == r["refGenomeId"])]
        assert len(sel) == r["countSeq"]
        s = np.float32(0)
        for x in sel["identity"]:
            s = np.float32(s + x)
        assert np.float32(s / np.float32(len(sel))).view(np.uint32) == np.float32(r["identity"]).view(np.uint32)


def _map_both(ctx, sk, sketches):
    """compute_cgi_sketched with and without fragments: the results must be the same bytes."""
    want, ctr0 = fb.compute_cgi_sketched(ctx, sk, sketches)
    res, ctr, frags = fb.compute_cgi_sketched(ctx, sk, sketches, fragments=True)
    assert res.tobytes() == want.tobytes()
    assert ctr.as_dict() == ctr0.as_dict()
    _check_invariants(res, frags, sk.sequencesByFileInfo)
    return res, frags


@pytest.fixture(scope="module")
def real():
    return fb.read_fasta(EC), fb.read_fasta(SH)


def test_real_pair_frags_equal_the_host_rule_and_the_visual_goldens(real):
    ec, sh = real
    ctx = fb.Context(fb.Parameters())
    ge, gs = ctx.genomes([ec, sh])
    names = {"e": "data/Escherichia_coli_str_K12_MG1655.fna", "s": "data/Shigella_flexneri_2a_01.fna"}
    for tag, (q, gq, qn), (r, gr, rn) in (("e2s", (ec, ge, "e"), (sh, gs, "s")), ("s2e", (sh, gs, "s"), (ec, ge, "e"))):
        sk = fb.Sketch(ctx, [gr])
        qs = fb.QuerySketch(ctx, [gq], [0], hint=sk)
        res, frags = _map_both(ctx, sk, [qs])
        assert frags.tobytes() == _expected_frags(ctx, sk, [gq], [0], 3000).tobytes(), tag
        lines = report.visual_lines(frags, [names[qn]], [names[rn]],
                                    [report.fragment_lengths([len(s) for _, s in q], 3000, 16, ctx.windowSize)],
                                    [l for _, l in sk.metadata], sk.sequencesByFileInfo, 3000)
        assert "\n".join(lines) + "\n" == open(os.path.join(GOLDEN, tag + ".txt.visual")).read(), tag


def test_edge_contigs_member_and_hashed_queries(real):
    """edge_mixed.fa (short contigs, N runs, lower case) at fragLen 1000: hashed and index-derived query sketches of the
    same genome, several sketches in one call."""
    ec, _ = real
    edge = fb.read_fasta(os.path.join(GOLDEN, "edge_mixed.fa"))
    other = [("ec_a", ec[0][1][:40000]), ("ec_b", edge[3][1] + ec[0][1][50000:52000].lower())]
    ctx = fb.Context(fb.Parameters(minReadLength=1000))
    ga, gb = ctx.genomes([edge, other])
    sk = fb.Sketch(ctx, [ga, gb])
    hashed = fb.QuerySketch(ctx, [ga, gb], [0, 1])                  # no hint: every fragment hashed
    derived = fb.QuerySketch.from_index(ctx, sk, [1, 0], [2, 3])    # stage A'
    res, frags = _map_both(ctx, sk, [hashed, derived])
    assert len(frags) > 10
    assert frags.tobytes() == _expected_frags(ctx, sk, [ga, gb, gb, ga], [0, 1, 2, 3], 1000).tobytes()


@pytest.fixture(scope="module")
def cfg4_slice():
    specs = W.config4(clusters=2)
    pick = list(range(0, 6)) + list(range(20, 26))                 # both clusters, multi-contig 3 Mbp drafts
    ctx = fb.Context(fb.Parameters())
    contigs = [specs[i].contigs(ctx.synth_genome(specs[i].seed, specs[i].ancestor, specs[i].strain, specs[i].ppm, specs[i].length))
               for i in pick]
    ctx.close()
    return [specs[i] for i in pick], contigs


def _cfg4_run(contigs, flags):
    ctx = fb.Context(fb.Parameters())
    for k, v in flags.items():
        ctx.set_flag(k, v)
    hs = ctx.genomes(contigs)
    refs = hs[:8]
    sk = fb.Sketch(ctx, refs)
    members = fb.QuerySketch.from_index(ctx, sk, [1, 6, 3], [10, 11, 12])          # members, derived from the index
    others = fb.QuerySketch(ctx, hs[8:] + [hs[0]], [20, 21, 22, 23, 24], hint=sk)   # non-members hashed, a member hinted
    res, frags = _map_both(ctx, sk, [members, others])
    want = _expected_frags(ctx, sk, [hs[1], hs[6], hs[3]] + hs[8:] + [hs[0]], [10, 11, 12, 20, 21, 22, 23, 24], 3000)
    assert frags.tobytes() == want.tobytes()
    return res, frags, ctx


def test_cfg4_slice_sketches_pieces_and_passes(cfg4_slice):
    _, contigs = cfg4_slice
    res, frags, _ = _cfg4_run(contigs, {})
    assert len(np.unique(frags["qryGenomeId"])) == 8 and len(frags) > 5000
    # one query per reduction pass and pieces of 700 fragments (a 3 Mbp draft has about 1000): same results and frags
    res2, frags2, ctx = _cfg4_run(contigs, {"cgi_table_queries": 1, "frags_per_piece": 700, "count_paths": 1})
    pc = ctx.path_counts()
    assert pc["piece.mapped"] > 8 and pc["cgi.passes"] >= 8
    assert res2.tobytes() == res.tobytes() and frags2.tobytes() == frags.tobytes()


def test_identity_tie_goes_to_the_largest_query_fragment():
    """Query fragments 3 and 7 are the same 3 kb: both win the same bin of the reference with the same identity, and
    computeCGI's stable sort keeps the later one."""
    base = synth_genome(31, 1, 0, 0, 60000).tobytes()
    x = base[9000:12000]
    qseq = base[:21000] + x + base[24000:30000]
    rseq = synth_genome(31, 1, 1, 20000, 60000).tobytes()          # a 2 % strain of the same ancestor
    ctx = fb.Context(fb.Parameters())
    gq, gr = ctx.genomes([[("q", qseq)], [("r", rseq)]])
    sk = fb.Sketch(ctx, [gr])
    rows = fb.Map(ctx, sk, gq).rows
    r3, r7 = rows[rows["querySeqId"] == 3], rows[rows["querySeqId"] == 7]
    assert len(r3) and len(r7)
    best3, best7 = r3[np.argmax(r3["nucIdentity"])], r7[np.argmax(r7["nucIdentity"])]
    assert best3["nucIdentity"] == best7["nucIdentity"] and best3["refStartPos"] == best7["refStartPos"]
    res, frags = _map_both(ctx, sk, [fb.QuerySketch(ctx, [gq], [0], hint=sk)])
    assert frags.tobytes() == _expected_frags(ctx, sk, [gq], [0], 3000).tobytes()
    at = frags[(frags["refSeqId"] == best3["refSeqId"]) & (frags["refStartPos"] // 2980 == best3["refStartPos"] // 2980)]
    assert len(at) == 1 and at[0]["querySeqId"] == 7 and at[0]["identity"] == best3["nucIdentity"]
    assert 3 not in frags["querySeqId"].tolist()


# ---------------------------------------------------------------------------------------- the command line
@pytest.fixture(scope="module")
def cfg4_dir(tmp_path_factory):
    specs = W.config4(clusters=2)
    d = tmp_path_factory.mktemp("cfg4v")
    ctx = fb.Context(fb.Parameters())
    for s in specs:
        W.write_fasta(str(d / (s.name + ".fna")), s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)))
    ctx.close()
    open(d / "all.txt", "w").write("\n".join(s.name + ".fna" for s in specs) + "\n")
    return d


def _cli(d, args, host=False):
    env = dict(os.environ)
    for v in ("BANI_CLI_HOST_CGI", "BANI_INDEX_BUDGET", "BANI_QUERY_BUDGET"):
        env.pop(v, None)
    if host:
        env["BANI_CLI_HOST_CGI"] = "1"
    r = subprocess.run([EXE] + args + ["-t", "8"], cwd=d, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _same_outputs(d, a, b, exts=("", ".matrix", ".visual")):
    for ext in exts:
        assert open(d / (a + ext)).read() == open(d / (b + ext)).read(), ext


def test_cli_visualize_device_equals_host_path(cfg4_dir):
    d = cfg4_dir
    base = ["--ql", "all.txt", "--rl", "all.txt", "--matrix", "--visualize", "--gpus", "1"]
    _cli(d, base + ["-o", "dev.txt"])
    _cli(d, base + ["-o", "host.txt"], host=True)
    _same_outputs(d, "dev.txt", "host.txt")
    assert sorted(open(d / "dev.txt").read().splitlines()) == sorted(open(os.path.join(GOLDEN, "cfg4_40x40.txt")).read().splitlines())
    vis = open(d / "dev.txt.visual").read().splitlines()
    assert len(vis) > 40 * 900
    # query-list order: the queries' first lines come in the order of all.txt
    order = list(dict.fromkeys(l.split("\t")[0] for l in vis))
    assert order == [l for l in open(d / "all.txt").read().split() if l in order]


def test_cli_visualize_from_a_loaded_index_reads_no_member_query(cfg4_slice, tmp_path):
    specs, contigs = cfg4_slice
    names = []
    for s, c in zip(specs, contigs):
        W.write_fasta(str(tmp_path / (s.name + ".fna")), c)
        names.append(s.name + ".fna")
    open(tmp_path / "all.txt", "w").write("\n".join(names) + "\n")
    _cli(tmp_path, ["--ql", "all.txt", "--rl", "all.txt", "-o", "a.txt", "--matrix", "--visualize", "--gpus", "1", "--saveIndex", "db"])
    for n in names:
        os.unlink(tmp_path / n)
    r = _cli(tmp_path, ["--ql", "all.txt", "--loadIndex", "db", "-o", "b.txt", "--matrix", "--visualize"])
    assert "reading 0 genome files" in r.stderr
    _same_outputs(tmp_path, "a.txt", "b.txt")
    assert len(open(tmp_path / "b.txt.visual").read()) > 0


@pytest.mark.parametrize("partition", ["interleave", "block"])
def test_cli_visualize_two_gpus(cfg4_dir, partition):
    cnt = C.c_int32()
    fb.load_library().bani_device_count(C.byref(cnt))
    if cnt.value < 2:
        pytest.skip("needs two GPUs")
    d = cfg4_dir
    base = ["--ql", "all.txt", "--rl", "all.txt", "--matrix", "--visualize", "--gpus", "2", "--partition", partition]
    _cli(d, base + ["-o", "dev2%s.txt" % partition])
    _cli(d, base + ["-o", "host2%s.txt" % partition], host=True)
    _same_outputs(d, "dev2%s.txt" % partition, "host2%s.txt" % partition)
    assert sorted(open(d / ("dev2%s.txt" % partition)).read().splitlines()) == \
        sorted(open(os.path.join(GOLDEN, "cfg4_40x40.txt")).read().splitlines())
