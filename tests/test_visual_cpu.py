"""CPU: report.visual_lines, the Python form of outputVisualizationFile -- query offsets from the per-fragment metadata
lengths, reference offsets from the contig table of the index, identity digits and the column layout."""
import os

import numpy as np

import pyoracle as po
from conftest import GOLDEN
from fastani_b200.api import FRAG_DTYPE
from fastani_b200.report import fragment_lengths, visual_lines

EC = os.path.join(GOLDEN, "Escherichia_coli_str_K12_MG1655.fna.gz")
SH = os.path.join(GOLDEN, "Shigella_flexneri_2a_01.fna.gz")
E, S = "data/Escherichia_coli_str_K12_MG1655.fna", "data/Shigella_flexneri_2a_01.fna"


def _frags(q, vis):
    vr, vq, vs, vi = vis
    f = np.zeros(len(vr), FRAG_DTYPE)
    f["qryGenomeId"], f["refSeqId"], f["querySeqId"], f["refStartPos"], f["identity"] = q, vr, vq, vs, vi
    return f


def test_fragment_lengths_follow_map_metadata():
    # a contig shorter than a fragment (or than a window / k-mer) is one entry; the last fragment takes the remainder
    assert fragment_lengths([9500, 2999, 3000, 6001], 3000, 16, 24) == [3000, 3000, 3500, 2999, 3000, 3000, 3001]
    assert fragment_lengths([20, 10], 10, 16, 5) == [10, 10, 10]      # 10 < k: one entry
    assert fragment_lengths([20], 10, 16, 25) == [20]                 # 20 < w: one entry
    assert fragment_lengths([], 3000, 16, 24) == []


def test_offsets_and_layout_on_a_constructed_set():
    # query: contigs of 7000 (fragments 3000, 4000) and 500 (one entry); index: genome 0 = contigs 0, 1; genome 1 = contig 2
    f = np.zeros(3, FRAG_DTYPE)
    f[0] = (4, 1, 0, 20, np.float32(99.5))
    f[1] = (4, 2, 1, 100, np.float32(97.25))
    f[2] = (4, 0, 2, 7, np.float32(80.123456))
    lines = visual_lines(f, {4: "q.fa"}, ["r0.fa", "r1.fa"], {4: fragment_lengths([7000, 500], 3000, 16, 24)},
                         [5000, 4000, 3000], [2, 3], 3000)
    assert lines == [
        "q.fa\tr0.fa\t99.5\tNA\tNA\tNA\t3000\t5999\t20\t3019\tNA\tNA",
        "q.fa\tr0.fa\t97.25\tNA\tNA\tNA\t7000\t9999\t5100\t8099\tNA\tNA",
        "q.fa\tr1.fa\t80.1235\tNA\tNA\tNA\t0\t2999\t9007\t12006\tNA\tNA"]
    # offsets past 2^31 stay exact (int64, as the CLI's offset adders)
    big = visual_lines(f[2:], {4: "q.fa"}, ["r0.fa", "r1.fa"], {4: [3000]}, [2 ** 31, 2 ** 31, 3000], [2, 3], 3000)
    assert big[0].split("\t")[8:10] == [str(2 ** 32 + 7), str(2 ** 32 + 7 + 2999)]


def test_the_real_pair_against_the_reference_golden():
    """The 2-way rows of the oracle (E. coli -> Shigella) written by visual_lines against e2s.txt.visual."""
    ec, sh = po.read_fasta(EC), po.read_fasta(SH)
    rec, sbf, lens = po.sketch_genomes([sh], 16, 24)
    rows, _, _ = po.map_genome(po.Index(rec), ec, 16, 24, 3000)
    _, vis = po.cgi(rows, sbf, 3000, want_visual=True)
    got = visual_lines(_frags(0, vis), [E], [S], [fragment_lengths([len(s) for _, s in ec], 3000, 16, 24)], lens, sbf, 3000)
    gold = open(os.path.join(GOLDEN, "e2s.txt.visual")).read().splitlines()
    assert len(got) == len(gold) == 1322
    for g, w in zip(got, gold):
        gf, wf = g.split("\t"), w.split("\t")
        assert len(gf) == 12
        # names, identity digits and NA columns line by line: both files are in (contig, bin) order, and a tied bin
        # holds the same identity whichever fragment won it
        assert [gf[i] for i in (0, 1, 2, 3, 4, 5, 10, 11)] == [wf[i] for i in (0, 1, 2, 3, 4, 5, 10, 11)]
        assert int(gf[7]) - int(gf[6]) == int(gf[9]) - int(gf[8]) == 2999
    # ties on identity inside one (ref contig, bin) are broken arbitrarily by std::sort in the reference:
    # coordinates must agree wherever the winner is unique (the tolerance of test_oracle.py)
    assert len(set(got) & set(gold)) >= 1300
