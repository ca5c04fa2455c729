"""Cost of `fastANI --visualize` on the device reduction against the per-query host path (BANI_CLI_HOST_CGI=1).

An all-vs-all synthetic set is written to a temporary directory: the config 4 slice (2 clusters x 20 multi-contig 3 Mbp
drafts, 40 x 40) by default, or config 3 at 5 clusters x 20 strains of 5 Mbp (100 x 100) with --config3.  The command
line then runs with `--matrix --visualize --gpus 1`, the two paths alternating, `--repeats` times each.  Prints one JSON
line per path: the median wall time of the whole process and the median of the mapping time the command line logs (GPU
0, "Time spent mapping"), both in ms; then one line saying whether .txt, .matrix and .visual were byte-identical in every
run.  The card's name and power limit are printed in the same run.

    python tools/bench_visual.py [--config3] [--repeats 3] [--threads 8]
"""
import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fastani_b200 as fb  # noqa: E402
from fastani_b200 import workloads as W  # noqa: E402

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(d, out, host, threads):
    env = dict(os.environ)
    for v in ("BANI_CLI_HOST_CGI", "BANI_INDEX_BUDGET", "BANI_QUERY_BUDGET"):
        env.pop(v, None)
    if host:
        env["BANI_CLI_HOST_CGI"] = "1"
    t0 = time.perf_counter()
    r = subprocess.run([EXE, "--ql", "all.txt", "--rl", "all.txt", "-o", out, "--matrix", "--visualize", "--gpus", "1", "-t", str(threads)],
                       cwd=d, capture_output=True, text=True, env=env)
    wall = (time.perf_counter() - t0) * 1e3
    if r.returncode != 0:
        raise SystemExit(r.stderr[-3000:])
    mapping = [float(l.split(" : ")[1].split()[0]) * 1e3 for l in r.stderr.splitlines() if "Time spent mapping" in l]
    return wall, mapping[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config3", action="store_true")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--threads", type=int, default=8)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    specs = W.config3(clusters=5, strains=20) if a.config3 else W.config4(clusters=2)
    ctx = fb.Context(fb.Parameters())
    with tempfile.TemporaryDirectory() as d:
        W.materialize(specs, d, gen=lambda s: ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length))
        ctx.close()
        open(os.path.join(d, "all.txt"), "w").write("\n".join(s.name + ".fna" for s in specs) + "\n")
        times = {"device": [], "host": []}
        identical = True
        for i in range(a.repeats):
            for path in ("device", "host"):
                times[path].append(run(d, "%s%d.txt" % (path, i), path == "host", a.threads))
            for ext in ("", ".matrix", ".visual"):
                identical &= filecmp.cmp(os.path.join(d, "device%d.txt%s" % (i, ext)), os.path.join(d, "host%d.txt%s" % (i, ext)), shallow=False)
        n_lines = sum(1 for _ in open(os.path.join(d, "device0.txt.visual")))
        for path in ("device", "host"):
            print(json.dumps({"workload": "config3 100x100" if a.config3 else "config4 40x40", "path": path, "runs": a.repeats,
                              "wall_ms": round(statistics.median(t[0] for t in times[path]), 1),
                              "mapping_ms": round(statistics.median(t[1] for t in times[path]), 1),
                              "visual_lines": n_lines}), flush=True)
        print(json.dumps({"outputs_identical": identical}), flush=True)
        if not identical:
            sys.exit(1)


if __name__ == "__main__":
    main()
