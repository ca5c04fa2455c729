#!/usr/bin/env python
"""Generates the reference-side golden of a collection of many small genomes by running the UNMODIFIED reference
(oracle/_ref/fastANI_ref, built by oracle/Makefile from /root/reference) on workloads.small_genomes: 3000 genomes of
10 - 40 kbp, all vs all with --matrix.  It uses the helpers of make_bench_golden.py (same directory), so the lines keep
the reference's text verbatim except that the directory of the FASTA paths is stripped.

  small_3000.txt.gz            the output lines
  small_3000.txt.matrix.gz     the --matrix file (3000 x 3000, mostly "NA")

Both are gzipped with mtime 0, so the same reference output gives the same bytes.  The reference's threads may order
lines of one query with equal identity differently from run to run (the matrix does not change), so the tests compare
the lines as sets.  The reference needs 19 - 23 s for the run on 8 CPU cores.

  python tests/golden/make_small_golden.py
"""
import gzip
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_bench_golden as B     # noqa: E402
from make_bench_golden import W   # noqa: E402


def small():
    specs = W.small_genomes()
    d = os.path.join(B.TMP, "bani_fasta_" + W.spec_key(specs))
    paths = W.materialize(specs, d)
    out = os.path.join(d, "golden_out.txt")
    B.run(paths, paths, out, ["--matrix"])
    m = open(out + ".matrix").read().splitlines()
    mat = "\n".join([m[0]] + ["\t".join([os.path.basename(x) if x.endswith(".fna") else x for x in ln.split("\t")]) for ln in m[1:]]) + "\n"
    for name, text in (("small_3000.txt.gz", B.strip_dirs(open(out).read())), ("small_3000.txt.matrix.gz", mat)):
        with open(os.path.join(B.GOLDEN, name), "wb") as f, gzip.GzipFile(fileobj=f, mode="wb", mtime=0, filename="") as z:
            z.write(text.encode())


if __name__ == "__main__":
    small()
