"""The identity reduction on collections of many small genomes: the sparse path of stage H against the dense one.

Collections of 50 kbp genomes (clusters of 10 strains at 0.8 % * strain substitutions) are generated on the device
(bani_synth_genome) and mapped all vs all through the Python API (compute_cgi, k16, fragLen 3000), one GPU:

  0. --sweep (500 .. 6000 genomes, one query piece each): dense forced against sparse forced, alternating, around the
     selection threshold of 2^22 dense pairs (n x n pairs against the piece's rows, printed with each line).
  1. --n (20,000 genomes, 1 Gbp): dense forced and sparse forced, alternating, --runs times each (after one warm-up
     run of each).  Per path: median mapping ms (host clock around compute_cgi, which returns after its last device
     synchronisation), device peak bytes (mem_stats) and the SHA-256 of the results, which must be equal.
  2. --scale-n (100,000 genomes, 5 Gbp): the sparse path once.  The dense path runs there only with --scale-dense and
     only if its per-piece tables (count + identity for 16,384 queries x every genome, on the device and on the host)
     fit the free device and host memory; otherwise the line says why it did not run.
  3. config 3 (1000 x 1000 x 5 Mbp): automatic choice against dense forced, alternating, --runs times each, then one
     run of each with the path counters on: cgi.sparse must be 0 and the result hashes equal.

The card's name and power limit are read in the same run.  One JSON line per measurement.

    python tools/bench_small_genomes.py [--n 20000] [--scale-n 100000] [--scale-dense] [--runs 3] [--skip-config3]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fastani_b200 as fb  # noqa: E402
from fastani_b200 import workloads as W  # noqa: E402

LENGTH = 50_000
STRAINS = 10
PIECE_QUERIES = (1 << 18) // (LENGTH // 3000)       # whole genomes of 16 fragments in a piece of 2^18 fragments


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,memory.free", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def free_device_bytes():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=memory.free", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.split()
        return int(out[0]) << 20
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        return 0


def free_host_bytes():
    try:
        for ln in open("/proc/meminfo"):
            if ln.startswith("MemAvailable:"):
                return int(ln.split()[1]) << 10
    except OSError:
        pass
    return 0


def emit(**kw):
    print(json.dumps(kw), flush=True)


def collection(ctx, n, length=LENGTH, seed=9, batch=5000):
    """n genomes of `length` bases in clusters of STRAINS strains, synthesised on the device into one host buffer."""
    seq = np.empty(n * length, np.uint8)
    for g in range(n):
        ctx.synth_genome(seed, g // STRAINS + 1, g % STRAINS, 8000 * (g % STRAINS), length, out=seq[g * length:(g + 1) * length])
    hs = []
    for a in range(0, n, batch):
        b = min(n, a + batch)
        off = np.arange(a, b + 1, dtype=np.int64) * length - a * length
        hs += ctx.genomes_from_buffer(seq[a * length:b * length], off, np.arange(b - a + 1, dtype=np.int32))
    return hs


def specs_genomes(ctx, specs):
    return [ctx.genome(s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length))) for s in specs]


def run(ctx, sk, hs, sparse, count_paths=False):
    ctx.set_flag("cgi_sparse", sparse)
    ctx.set_flag("count_paths", 1 if count_paths else 0)
    ctx.sync()
    ctx.mem_stats()                                   # resets the peak
    t0 = time.perf_counter()
    res, _, ctr = fb.compute_cgi(ctx, sk, hs)
    ms = (time.perf_counter() - t0) * 1e3
    peak = ctx.mem_stats()["peak_live"]
    paths = ctx.path_counts() if count_paths else None
    run.mappings = ctr.as_dict()["mappings"]
    return ms, peak, hashlib.sha256(res.tobytes()).hexdigest(), len(res), paths


def alternate(ctx, sk, hs, modes, runs, workload, **extra):
    for m in modes:                                   # warm-up: module loads, scratch slots, CUB temp sizes
        run(ctx, sk, hs, m)
    got = {m: [] for m in modes}
    for _ in range(runs):
        for m in modes:
            got[m].append(run(ctx, sk, hs, m))
    hashes = set()
    for m in modes:
        rs = got[m]
        hashes |= {r[2] for r in rs}
        emit(workload=workload, cgi_sparse=m, runs=runs, mapping_ms=[round(r[0], 1) for r in rs],
             median_ms=round(statistics.median(r[0] for r in rs), 1), peak_gb=round(max(r[1] for r in rs) / 1e9, 2),
             results=rs[0][3], sha256=rs[0][2][:16], **extra)
    emit(workload=workload, results_equal=len(hashes) == 1)
    return len(hashes) == 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000)
    ap.add_argument("--scale-n", type=int, default=100_000)
    ap.add_argument("--scale-dense", action="store_true")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-config3", action="store_true")
    ap.add_argument("--sweep", type=int, nargs="*", default=[500, 1000, 1500, 2048, 3000, 4000, 6000],
                    help="collection sizes (at most 16,384: one piece) timed dense against sparse around the threshold")
    a = ap.parse_args()
    emit(gpu=gpu_info())
    ok = True
    ctx = fb.Context(fb.Parameters())

    # 0. the threshold: collections whose one piece has about 2^22 dense (query, genome) pairs, dense against sparse
    for n in a.sweep:
        hs = collection(ctx, n)
        sk = fb.Sketch(ctx, hs)
        run(ctx, sk, hs, 1)
        ok &= alternate(ctx, sk, hs, (0, 1), a.runs, "sweep %d x 50 kbp" % n, pairs=n * n, rows=run.mappings)
        sk.close()
        for g in hs:
            g.close()
        ctx.trim()

    # 1. dense against sparse on the 1 Gbp collection
    hs = collection(ctx, a.n)
    sk = fb.Sketch(ctx, hs)
    ok &= alternate(ctx, sk, hs, (0, 1), a.runs, "small %d x 50 kbp" % a.n)
    ms, peak, h, n, p = run(ctx, sk, hs, -1, count_paths=True)
    emit(workload="small %d x 50 kbp" % a.n, cgi_sparse=-1, mapping_ms=round(ms, 1), sha256=h[:16],
         paths={k: v for k, v in p.items() if k.startswith(("cgi.", "piece."))})
    sk.close()
    for g in hs:
        g.close()
    ctx.trim()

    # 2. the 5 Gbp collection
    if a.scale_n:
        hs = collection(ctx, a.scale_n)
        sk = fb.Sketch(ctx, hs)
        wl = "small %d x 50 kbp" % a.scale_n
        ms, peak, h, n, p = run(ctx, sk, hs, 1, count_paths=True)
        emit(workload=wl, cgi_sparse=1, mapping_ms=round(ms, 1), peak_gb=round(peak / 1e9, 2), results=n, sha256=h[:16],
             paths={k: v for k, v in p.items() if k.startswith(("cgi.", "piece."))})
        dense = 8 * min(PIECE_QUERIES, a.scale_n) * a.scale_n
        fd, fh = free_device_bytes(), free_host_bytes()
        fits = dense + (3 << 30) < fd and dense < fh
        if a.scale_dense and fits:
            ms0, peak0, h0, _, _ = run(ctx, sk, hs, 0)
            emit(workload=wl, cgi_sparse=0, mapping_ms=round(ms0, 1), peak_gb=round(peak0 / 1e9, 2), sha256=h0[:16])
            ok &= h0 == h
        else:
            emit(workload=wl, cgi_sparse=0, skipped="dense tables %.1f GB per piece (device + host each); free %.1f GB device, %.1f GB host%s"
                 % (dense / 1e9, fd / 1e9, fh / 1e9, "" if a.scale_dense else "; --scale-dense not given"))
        sk.close()
        for g in hs:
            g.close()
        ctx.trim()

    # 3. config 3, where the dense path is the right one
    if not a.skip_config3:
        hs = specs_genomes(ctx, W.config3())
        sk = fb.Sketch(ctx, hs)
        ok &= alternate(ctx, sk, hs, (-1, 0), a.runs, "config3 1000 x 1000")
        for m in (-1, 0):
            ms, _, h, _, p = run(ctx, sk, hs, m, count_paths=True)
            emit(workload="config3 1000 x 1000", cgi_sparse=m, counted=True, sha256=h[:16],
                 paths={k: v for k, v in p.items() if k.startswith(("cgi.", "piece."))})
            ok &= p["cgi.sparse"] == 0
    emit(gpu=gpu_info(), ok=bool(ok))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
