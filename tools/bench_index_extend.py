"""Cost of adding genomes to a saved index (index_file_extend) against sketching and saving the whole list again.

Config 3's 1000 references (50 clusters x 20 strains of synthetic 5 Mbp genomes, k 16, fragLen 3000) are synthesised and
uploaded once.  The first 990 are sketched and saved to an index file in a temporary directory (set-up, not timed).  Then,
one after the other, with a device synchronise around each:
  extend : sketch the last 10 (Sketch) and write old file + their records to a new file (index_file_extend)
  fresh  : sketch all 1000 (Sketch) and save them (Sketch.save)
Both files must have the same SHA-256.  One JSON line per arm (wall seconds, bytes read from and written to disk), then one
with the digests.  The card's name and power limit are printed in the same run.  The old file was written just before the
extension, so its read usually comes from the page cache: the extension's time is mostly copies and checksums.

    python tools/bench_index_extend.py [--clusters 50] [--strains 20] [--added 10]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fastani_b200 as fb  # noqa: E402
from fastani_b200 import workloads as W  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def sha256(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            h.update(block)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", type=int, default=50)
    ap.add_argument("--strains", type=int, default=20)
    ap.add_argument("--added", type=int, default=10)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    specs = W.config3(clusters=a.clusters, strains=a.strains)
    n_old = len(specs) - a.added
    ctx = fb.Context(fb.Parameters())
    tmp = tempfile.mkdtemp(prefix="bani_extend_")
    try:
        hs = []
        for i in range(0, len(specs), 50):                   # synthesised and uploaded 50 at a time: host memory stays small
            hs += ctx.genomes([s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs[i:i + 50]])
        old, ext, fresh = (os.path.join(tmp, n) for n in ("old.idx", "ext.idx", "fresh.idx"))
        sk = fb.Sketch(ctx, hs[:n_old])
        sk.save(old)
        sk.close()
        ctx.trim()

        ctx.sync()
        t0 = time.perf_counter()
        added = fb.Sketch(ctx, hs[n_old:])
        ctx.sync()
        t1 = time.perf_counter()
        fb.index_file_extend(ctx, old, added, ext)
        t2 = time.perf_counter()
        added.close()
        ctx.trim()
        print(json.dumps({"arm": "extend", "genomes_saved": n_old, "genomes_added": a.added, "wall_s": round(t2 - t0, 2),
                          "sketch_added_s": round(t1 - t0, 2), "extend_file_s": round(t2 - t1, 2),
                          "bytes_read": os.path.getsize(old), "bytes_written": os.path.getsize(ext)}), flush=True)
        digest_ext = sha256(ext)
        os.unlink(ext)

        ctx.sync()
        t0 = time.perf_counter()
        sk = fb.Sketch(ctx, hs)
        ctx.sync()
        t1 = time.perf_counter()
        sk.save(fresh)
        t2 = time.perf_counter()
        sk.close()
        ctx.trim()
        print(json.dumps({"arm": "fresh", "genomes": len(specs), "wall_s": round(t2 - t0, 2), "sketch_s": round(t1 - t0, 2),
                          "save_s": round(t2 - t1, 2), "bytes_read": 0, "bytes_written": os.path.getsize(fresh)}), flush=True)
        digest_fresh = sha256(fresh)
        print(json.dumps({"sha256_extend": digest_ext, "sha256_fresh": digest_fresh, "identical": digest_ext == digest_fresh}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
