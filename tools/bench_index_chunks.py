"""Cost of mapping against a saved index loaded in chunks (Sketch.load_budget) on one GPU.

Config 3's 1000 references (50 clusters x 20 strains of synthetic 5 Mbp genomes, k 16, fragLen 3000) are sketched once and
saved to one index file in a temporary directory.  The 8 sample queries of tests/golden/bench_cfg3_q8.txt get their
fragment sketches from that file (QuerySketch.from_index_file: no FASTA is read).  The file is then loaded and mapped with
the index budget forced to 1, 2 and 4 runs of genomes.  Per run count, one JSON line: the load time (disk read, checks and
index_finish, with a device synchronise), the index_finish device time (profile stages index_sort + index_compact), the
mapping time, the bytes the loads read from the file, a hash of the sorted results (equal for every run count) and the
parity with the golden.  The card's name and power limit are printed in the same run.  The disk reads go through the
page cache: after the first pass the file is usually cached, so the load time is mostly copies and index_finish.

    python tools/bench_index_chunks.py [--runs 1,2,4] [--clusters 50] [--strains 20]
"""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fastani_b200 as fb  # noqa: E402
from fastani_b200 import report, workloads as W  # noqa: E402

FRAG_LEN = 3000
GOLDEN_Q8 = os.path.join(ROOT, "tests", "golden", "bench_cfg3_q8.txt")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def need(info, first, end):
    """Device bytes of loading genomes [first, end) (what Sketch.load_budget compares with the budget)."""
    m = int(info["genome_records"][first:end].sum())
    return fb.index_footprint(m, m, int(info["genome_contigs"][first:end].sum()), int(info["genome_bits"][first:end].sum()), 0)[0]


def runs_for(info, budget):
    out, first, n = [], 0, info["n_genomes"]
    while first < n:
        lo, hi = first, n                          # the largest end whose load fits (need grows with the end)
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if need(info, first, mid) <= budget else (lo, mid - 1)
        if lo == first:
            return None
        out.append((first, lo))
        first = lo
    return out


def budget_for_runs(info, n):
    """An index budget whose loads take the file in n runs (the middle of the range of budgets that give n)."""
    count = lambda b: len(runs_for(info, b) or [0] * (1 << 30))

    def smallest(m):
        lo, hi = 1 << 20, 1 << 42
        while hi - lo > (1 << 20):
            mid = (lo + hi) // 2
            lo, hi = (lo, mid) if count(mid) <= m else (mid, hi)
        return hi
    if n == 1:
        return need(info, 0, info["n_genomes"]) + (1 << 20)
    bot, top = smallest(n), smallest(n - 1) - (1 << 20)
    return (bot + top) // 2


def bytes_read(info, first, end):
    """Bytes one Sketch.load_budget of genomes [first, end) reads from the file: header, tables and checksums, the run's
    records (hash + wpos) and bitmap words, and the trailing bitmap word with the last genome."""
    nc, ng = info["n_contigs"], info["n_genomes"]
    tables = 128 + 4 * (nc + ng + nc + 1) + 8 + 8 * ng
    return tables + 8 * int(info["genome_records"][first:end].sum()) + int(info["genome_bits"][first:end].sum()) // 8 + (4 if end == ng else 0)


def parse(lines):
    rows = {}
    for ln in lines:
        f = ln.split("\t")
        rows[(f[0], f[1])] = (float(f[2]), int(f[3]), int(f[4]))
    return rows


def parity(got_lines, golden_lines):
    got, want = parse(got_lines), parse(golden_lines)
    bad = [k for k in set(got) | set(want)
           if k not in got or k not in want or got[k][1:] != want[k][1:] or abs(got[k][0] - want[k][0]) > 1e-4]
    return {"golden_rows": len(want), "mismatches": len(bad), "example": sorted(bad)[0] if bad else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", type=int, default=50)
    ap.add_argument("--strains", type=int, default=20)
    ap.add_argument("--runs", default="1,2,4")
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    specs = W.config3(clusters=a.clusters, strains=a.strains)
    names = [s.name + ".fna" for s in specs]
    ctx = fb.Context(fb.Parameters())
    tmp = tempfile.mkdtemp(prefix="bani_ix_")
    try:
        path = os.path.join(tmp, "cfg3.idx")
        t0 = time.perf_counter()
        hs = []
        for i in range(0, len(specs), 50):                   # synthesised and uploaded 50 at a time: host memory stays small
            hs += ctx.genomes([s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs[i:i + 50]])
        sk = fb.Sketch(ctx, hs)
        sk.save(path)
        sk.close()
        for h in hs:
            h.close()
        ctx.trim()
        print(json.dumps({"genomes": len(specs), "sketch_and_save_s": round(time.perf_counter() - t0, 1),
                          "file_bytes": os.path.getsize(path)}), flush=True)
        info = fb.index_file_info(path)
        sample = W.sample_queries(a.clusters, a.strains, 8)
        qs = fb.QuerySketch.from_index_file(ctx, path, sample, sample)
        glen = [report.genome_length([s.length], FRAG_LEN) for s in specs]
        default = (a.clusters, a.strains) == (50, 20)
        golden = open(GOLDEN_Q8).read().splitlines() if default else None
        digests = set()
        for n in [int(x) for x in a.runs.split(",")]:
            budget = budget_for_runs(info, n)
            runs = runs_for(info, budget)
            ctx.profile(True)
            ctx.profile_read()
            load_ms = map_ms = 0.0
            parts, first, nbytes = [], 0, 0
            while first < info["n_genomes"]:
                ctx.sync()
                t0 = time.perf_counter()
                sk, taken, _ = fb.Sketch.load_budget(ctx, path, first, budget)
                ctx.sync()
                t1 = time.perf_counter()
                res, _ = fb.compute_cgi_sketched(ctx, sk, [qs])
                ctx.sync()
                t2 = time.perf_counter()
                load_ms += (t1 - t0) * 1e3
                map_ms += (t2 - t1) * 1e3
                nbytes += bytes_read(info, first, first + taken)
                res["refGenomeId"] += first
                parts.append(res)
                sk.close()
                ctx.trim()
                first += taken
            prof = ctx.profile_read()
            ctx.profile(False)
            finish_ms = sum(prof[k][0] for k in ("index_sort", "index_compact") if k in prof)
            out = np.concatenate(parts)
            out = out[np.lexsort((out["refGenomeId"], out["qryGenomeId"]))]
            digest = hashlib.sha256(out.tobytes()).hexdigest()
            digests.add(digest)
            line = {"runs_forced": n, "runs_loaded": len(parts), "runs_predicted": len(runs), "index_budget": budget,
                    "load_ms": round(load_ms, 1), "index_finish_ms": round(finish_ms, 1), "map_ms": round(map_ms, 1),
                    "bytes_read": nbytes, "result_sha256": digest}
            if golden is not None:
                rows = [(int(x["qryGenomeId"]), int(x["refGenomeId"]), int(x["countSeq"]), int(x["totalQueryFragments"]), x["identity"]) for x in out]
                line["parity_vs_golden"] = parity(report.output_lines(rows, names, names, glen, glen, FRAG_LEN), golden)
            print(json.dumps(line), flush=True)
        print(json.dumps({"same_result_for_every_run_count": len(digests) == 1}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
