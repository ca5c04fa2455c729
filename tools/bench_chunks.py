"""Cost of building and mapping a reference list in chunks (fastani_b200.compute_cgi_chunked) on one GPU.

Config 3 (clusters x strains synthetic 5 Mbp genomes, all vs all, k 16, fragLen 3000) is run with its reference list
forced into 1, 2 and 4 chunks through the index budget.  Queries are hashed once into one sketch per 50 genomes; every
timed step uploads the references, builds each chunk's index and maps every query against it.  Prints one JSON line per
chunk count: ms per step, the per-chunk overhead against one chunk, and a hash of the sorted results, which must be equal
for every chunk count.  The card's name and power limit are printed in the same run.

    python tools/bench_chunks.py [--clusters 50] [--strains 20] [--steps 2] [--warmup 1] [--chunks 1,2,4]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import fastani_b200 as fb  # noqa: E402
from fastani_b200 import workloads as W  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def budget_for_chunks(lens, conts, n, w):
    """An index budget whose plan has n chunks (the middle of the range of budgets that give n)."""
    def chunks(b):
        try:
            return len(fb.plan_chunks(lens, conts, 16, w, b))
        except fb.BaniError:
            return 1 << 30

    def smallest(m):
        lo, hi = 1 << 20, 1 << 42
        while hi - lo > (1 << 20):
            mid = (lo + hi) // 2
            lo, hi = (lo, mid) if chunks(mid) <= m else (mid, hi)
        return hi
    if n == 1:
        return smallest(1) + (1 << 20)
    bot, top = smallest(n), smallest(n - 1) - (1 << 20)
    return (bot + top) // 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", type=int, default=50)
    ap.add_argument("--strains", type=int, default=20)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chunks", default="1,2,4")
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    specs = W.config3(clusters=a.clusters, strains=a.strains)
    ctx = fb.Context(fb.Parameters())
    w = ctx.windowSize
    contigs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs]
    qs = []
    for i in range(0, len(contigs), 50):
        hs = ctx.genomes(contigs[i:i + 50])
        qs.append(fb.QuerySketch(ctx, hs, list(range(i, i + len(hs)))))
        for h in hs:
            h.close()
    lens = [sum(len(x) for _, x in cl) for cl in contigs]
    conts = [len(cl) for cl in contigs]
    base = None
    for n in [int(x) for x in a.chunks.split(",")]:
        budget = budget_for_chunks(lens, conts, n, w)
        times, digest, plan = [], None, None
        for step in range(a.warmup + a.steps):
            ctx.sync()
            t0 = time.perf_counter()
            res, plan = fb.compute_cgi_chunked(ctx, contigs, qs, index_budget=budget, query_budget=1 << 40)
            ctx.sync()
            if step >= a.warmup:
                times.append((time.perf_counter() - t0) * 1e3)
            digest = hashlib.sha256(res.tobytes()).hexdigest()
        ms = sum(times) / len(times)
        if n == 1:
            base = ms
        print(json.dumps({"genomes": len(specs), "chunks_forced": n, "chunks_run": len(plan["chunks"]), "index_budget": budget,
                          "ms_per_step": round(ms, 1),
                          "ms_per_extra_chunk": round((ms - base) / (len(plan["chunks"]) - 1), 1) if base is not None and len(plan["chunks"]) > 1 else None,
                          "result_sha256": digest}), flush=True)


if __name__ == "__main__":
    main()
