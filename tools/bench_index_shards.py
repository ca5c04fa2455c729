"""Cost of an all-vs-all --loadIndex run against a saved index of several shard files: member query sketches derived from
the shard files against every query file read and hashed.

Config 3's 1000 genomes (50 clusters x 20 strains of synthetic 5 Mbp genomes, k 16, fragLen 3000) are synthesised, written
as FASTA files to a temporary directory, and saved as S interleaved shard files (one Sketch.save per shard plus the .meta
file, as --saveIndex on S GPUs writes them; set-up, not timed).  Then, for each S, the command line runs
`--ql <list> --loadIndex db<S> --gpus 1` in two arms, alternating:
  derived : the list names the genomes of the index, so no query file is read (their sketches come from the shard files)
  hashed  : the list names symlinks to the same files; they are not genomes of the index, so every file is read and
            hashed, as every multi-shard load did before member queries were derived from any shard count
One JSON line per run: the whole-process wall time and the phases the command line logs (reading, loading the reference,
mapping; summed over the shard files).  Then one line per S comparing the two arms' output rows after the symlink names
are mapped back (they must be identical).  The card's name and power limit are printed in the same run.  The files were
written just before, so the reads usually come from the page cache.

    python tools/bench_index_shards.py [--shards 2,4] [--reps 2] [--threads 16] [--clusters 50] [--strains 20]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fastani_b200 as fb  # noqa: E402
from fastani_b200 import workloads as W  # noqa: E402

EXE = os.path.join(ROOT, "fastani_b200", "bin", "fastANI")
K, FRAG_LEN = 16, 3000


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def phases(stderr):
    """Seconds of each phase the command line logs, summed over the shard files."""
    out = {}
    for key, pat in (("read_s", r"Time spent reading \d+ genome files : ([\d.e+-]+)"),
                     ("load_s", r"Time spent loading the reference : ([\d.e+-]+)"),
                     ("map_s", r"Time spent mapping \d+ query genome\(s\) : ([\d.e+-]+)"),
                     ("load_and_map_chunked_s", r"Time spent loading and mapping in chunks : ([\d.e+-]+)"),
                     ("total_s", r"Total time : ([\d.e+-]+)")):
        v = [float(x) for x in re.findall(pat, stderr)]
        if v:
            out[key] = round(sum(v), 3)
    m = re.search(r"Time spent reading (\d+) genome files", stderr)
    out["files_read"] = int(m.group(1)) if m else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", type=int, default=50)
    ap.add_argument("--strains", type=int, default=20)
    ap.add_argument("--shards", default="2,4")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--threads", type=int, default=16)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    specs = W.config3(clusters=a.clusters, strains=a.strains)
    names = [s.name + ".fna" for s in specs]
    ctx = fb.Context(fb.Parameters(kmerSize=K, minReadLength=FRAG_LEN))
    tmp = tempfile.mkdtemp(prefix="bani_shards_")
    try:
        t0 = time.perf_counter()
        hs, contig_names = [], []
        os.mkdir(os.path.join(tmp, "h"))
        for i in range(0, len(specs), 50):                   # synthesised, written and uploaded 50 at a time
            cs = [s.contigs(ctx.synth_genome(s.seed, s.ancestor, s.strain, s.ppm, s.length)) for s in specs[i:i + 50]]
            for nm, c in zip(names[i:i + 50], cs):
                W.write_fasta(os.path.join(tmp, nm), c)
                os.symlink(os.path.join("..", nm), os.path.join(tmp, "h", nm))
                contig_names.append([n for n, _ in c])
            hs += ctx.genomes(cs)
        open(os.path.join(tmp, "members.txt"), "w").write("\n".join(names) + "\n")
        open(os.path.join(tmp, "links.txt"), "w").write("\n".join("h/" + n for n in names) + "\n")
        print(json.dumps({"genomes": len(specs), "synth_and_write_s": round(time.perf_counter() - t0, 1)}), flush=True)
        counts = [int(x) for x in a.shards.split(",")]
        index_bytes = {}
        for S in counts:                                      # every index is saved before the command line runs
            shards = [list(range(s, len(names), S)) for s in range(S)]
            index_bytes[S] = 0
            for s, sh in enumerate(shards):
                sk = fb.Sketch(ctx, [hs[j] for j in sh])
                path = os.path.join(tmp, "db%d.%dof%d.idx" % (S, s, S))
                sk.save(path)
                sk.close()
                ctx.trim()
                index_bytes[S] += os.path.getsize(path)
            lines = ["BANI_INDEX_META\t1", "%d\t%d\t%d\t%d\t%d" % (K, FRAG_LEN, ctx.windowSize, S, len(names))] + names
            for sh in shards:
                cn = [n for j in sh for n in contig_names[j]]
                lines += [str(len(cn))] + cn
            open(os.path.join(tmp, "db%d.meta" % S), "w").write("\n".join(lines) + "\n")
        for h in hs:                                          # the device is the command line's alone while it runs
            h.close()
        ctx.close()
        for S in counts:
            outs = {}
            for rep in range(a.reps):
                for arm in (("derived", "hashed") if rep % 2 == 0 else ("hashed", "derived")):
                    out = "%s_%d.txt" % (arm, S)
                    env = {k: v for k, v in os.environ.items() if not k.startswith("BANI_")}
                    cmd = [EXE, "--ql", "members.txt" if arm == "derived" else "links.txt", "--loadIndex", "db%d" % S, "--gpus", "1",
                           "-t", str(a.threads), "-o", out]
                    t1 = time.perf_counter()
                    r = subprocess.run(cmd, cwd=tmp, capture_output=True, text=True, env=env)
                    wall = time.perf_counter() - t1
                    if r.returncode != 0:
                        raise SystemExit("%s failed:\n%s" % (" ".join(cmd), r.stderr[-3000:]))
                    line = {"shards": S, "arm": arm, "rep": rep, "wall_s": round(wall, 3)}
                    line.update(phases(r.stderr))
                    print(json.dumps(line), flush=True)
                    outs[arm] = open(os.path.join(tmp, out)).read()
            hashed = "".join(l[2:] + "\n" if l.startswith("h/") else l + "\n" for l in outs["hashed"].splitlines())
            print(json.dumps({"shards": S, "index_bytes": index_bytes[S], "rows": outs["derived"].count("\n"),
                              "identical_rows": hashed == outs["derived"]}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
