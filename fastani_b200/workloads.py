"""The synthetic inputs of BASELINE.json's configs (SURVEY.md section 8d), as pure numpy/host code.

Nothing here touches the CUDA library: the reference arm of bench.py, the golden generators under
tests/golden/ and the parity tests all describe their genomes with these functions, and the device generator
(csrc/synth.cu, bani_synth_genome) produces the same bytes for the same (seed, ancestor, strain, ppm, length).

    config 2   1 query x 100 references, 5 Mbp, reference j = ancestor with substitutions at 0.2 % * j
    config 3   50 clusters x 20 strains, 5 Mbp, strain m = cluster ancestor with substitutions at 0.6 % * m
    config 4   500 clusters x 20 strains, 3 Mbp, cut into contigs (N50 ~ 50 kbp, minimum 2 kbp)
    config 5   the first 200 genomes of config 3 at k in {16, 21} x fragLen in {1000, 3000, 5000}
    small      300 clusters x 10 strains of 10 - 40 kbp, some drafts, some shorter than a fragment (small_genomes)
"""
import hashlib
import os

import numpy as np

from .synth import synth_genome


class GenomeSpec:
    """One synthetic genome: synth_genome(seed, ancestor, strain, ppm, length) cut at `cuts` (contig ends)."""
    __slots__ = ("name", "seed", "ancestor", "strain", "ppm", "length", "cuts")

    def __init__(self, name, seed, ancestor, strain, ppm, length, cuts=None):
        self.name, self.seed, self.ancestor, self.strain, self.ppm, self.length = name, seed, ancestor, strain, ppm, length
        self.cuts = cuts if cuts is not None else [length]

    def contig_lengths(self):
        return list(np.diff([0] + list(self.cuts)))

    def bases(self):
        return synth_genome(self.seed, self.ancestor, self.strain, self.ppm, self.length)

    def contigs(self, seq=None):
        """[(contig name, bytes)] -- one contig: the genome name; several: name_0, name_1, ..."""
        s = self.bases() if seq is None else seq
        if len(self.cuts) == 1:
            return [(self.name, s.tobytes())]
        out, a = [], 0
        for i, b in enumerate(self.cuts):
            out.append(("%s_%d" % (self.name, i), s[a:b].tobytes()))
            a = b
        return out


def config3(clusters=50, strains=20, length=5_000_000, seed=3):
    """Many-to-many clusters; genome index g = cluster * strains + strain."""
    return [GenomeSpec("c%d_s%d" % (c, s), seed, c + 1, s, 6000 * s, length)
            for c in range(clusters) for s in range(strains)]


def config2(n_refs=100, length=5_000_000, seed=2):
    """(query, references): the query is the ancestor, reference j diverges by 0.2 % * j."""
    q = GenomeSpec("q_anc", seed, 1, 0, 0, length)
    refs = [GenomeSpec("r%03d" % j, seed, 1, j, 2000 * j, length) for j in range(n_refs)]
    return q, refs


def contig_cuts(length, rng, mean=28000, minimum=2000):
    """Contig ends of a draft assembly: lengths = minimum + exponential(mean), N50 ~ 50 kbp; the last piece is
    merged into its predecessor when it would fall below the minimum."""
    cuts, pos = [], 0
    while pos < length:
        pos += minimum + int(rng.exponential(mean))
        cuts.append(min(pos, length))
    if len(cuts) > 1 and cuts[-1] - cuts[-2] < minimum:
        cuts.pop(-2)
    return cuts


def config4(clusters=500, strains=20, length=3_000_000, seed=4):
    out = []
    for c in range(clusters):
        for s in range(strains):
            rng = np.random.default_rng([seed, c, s])
            out.append(GenomeSpec("d%d_s%d" % (c, s), seed, c + 1, s, 6000 * s, length, contig_cuts(length, rng)))
    return out


def small_genomes(clusters=300, strains=10, seed=6, min_len=10_000, max_len=40_000):
    """A collection of many small genomes (plasmids, phages, MAG bins of a few tens of kbp): `clusters` ancestors of
    min_len .. max_len bases, each with `strains` strains at 0.8 % * strain substitutions.  Strain 2 of every third
    cluster is a draft cut into contigs of at least 2 kbp; the last strain of every fifth cluster is cut to 2500 bases,
    shorter than a 3 kbp fragment.  Genome index g = cluster * strains + strain.

    All vs all at the default parameters (k16, fragLen 3000) the default 3000 genomes make one query piece of about
    24,000 fragments against 3000 genomes: 9e6 dense (query, genome) pairs, far more than the piece's rows, so the
    identity reduction takes its sparse path.  The reference CLI needs 23 s for it (with --matrix) on 8 CPU cores."""
    out = []
    for c in range(clusters):
        rng = np.random.default_rng([seed, c])
        length = int(rng.integers(min_len, max_len + 1))
        for s in range(strains):
            n, cuts = length, None
            if s == strains - 1 and c % 5 == 0:
                n = 2500
            elif s == 2 and c % 3 == 0:
                cuts = contig_cuts(n, rng, mean=8000, minimum=2000)
            out.append(GenomeSpec("m%d_s%d" % (c, s), seed, c + 1, s, 8000 * s, n, cuts))
    return out


def n50(lengths):
    ls = sorted(lengths, reverse=True)
    half, acc = sum(ls) / 2.0, 0
    for x in ls:
        acc += x
        if acc >= half:
            return x
    return 0


def sample_queries(clusters, strains, n=8):
    """Indices (into config3 order) of the bounded query sample of the CPU arm: n queries spread over the clusters
    and over the divergence ladder (strain 1, 4, 7, ...)."""
    n = max(1, min(n, clusters * strains))
    out = []
    for i in range(n):
        c = (i * clusters) // n
        s = (1 + 3 * i) % strains
        out.append(c * strains + s)
    return out


# ----------------------------------------------------------------------------------------- FASTA on disk
def write_fasta(path, contigs, width=80):
    """80-column FASTA, written through a temporary name so that concurrent writers never expose a partial file."""
    tmp = "%s.%d.tmp" % (path, os.getpid())
    with open(tmp, "wb") as f:
        for name, seq in contigs:
            f.write((">%s\n" % name).encode())
            mv = np.frombuffer(seq, np.uint8)
            n = len(mv)
            full = n // width
            body = np.empty(n + (n + width - 1) // width, np.uint8)
            if full:
                blk = body[:full * (width + 1)].reshape(full, width + 1)
                blk[:, :width] = mv[:full * width].reshape(full, width)
                blk[:, width] = 10
            rest = n - full * width
            if rest:
                body[full * (width + 1):full * (width + 1) + rest] = mv[full * width:]
                body[-1] = 10
            f.write(body.tobytes())
    os.replace(tmp, path)


def spec_key(specs):
    h = hashlib.sha256()
    for g in specs:
        h.update(("%s,%d,%d,%d,%d,%d,%s;" % (g.name, g.seed, g.ancestor, g.strain, g.ppm, g.length,
                                             ",".join(map(str, g.cuts)) if len(g.cuts) > 1 else "")).encode())
    return h.hexdigest()[:16]


def _write_one(args):
    g, path = args
    if not os.path.exists(path):
        write_fasta(path, g.contigs())
    return path


def materialize(specs, directory, gen=None, procs=0):
    """Writes every genome of `specs` to directory/<name>.fna (skipping files that exist) and returns the paths.
    gen(spec) -> uint8 bases may replace the numpy generator (the GPU arm passes the device generator); without it
    the numpy generator runs in `procs` worker processes (0 = one per available core)."""
    os.makedirs(directory, exist_ok=True)
    paths = [os.path.join(directory, g.name + ".fna") for g in specs]
    todo = [(g, p) for g, p in zip(specs, paths) if not os.path.exists(p)]
    if not todo:
        return paths
    if gen is not None:
        for g, p in todo:
            write_fasta(p, g.contigs(gen(g)))
        return paths
    procs = procs or available_cores()
    if procs > 1 and len(todo) > 1:
        import multiprocessing as mp
        with mp.get_context("fork").Pool(min(procs, len(todo))) as pool:
            list(pool.imap_unordered(_write_one, todo, chunksize=1))
    else:
        for t in todo:
            _write_one(t)
    return paths


def available_cores():
    """Host threads this process may really use: the affinity mask capped by the cgroup CPU quota."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    for p in ("/sys/fs/cgroup/cpu.max",):
        try:
            q, per = open(p).read().split()[:2]
            if q != "max":
                n = max(1, min(n, int(float(q) / float(per) + 0.5)))
        except Exception:
            pass
    try:        # cgroup v1
        q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
        per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
        if q > 0 and per > 0:
            n = max(1, min(n, int(q / per + 0.5)))
    except Exception:
        pass
    return n
