"""Build libfastani_b200.so in-tree with nvcc for sm_90a (H100; no GPU needed: nvcc cross-compiles)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "lib")
LIB = os.path.join(OUT, "libfastani_b200.so")
STAMP = os.path.join(OUT, "flags.txt")
SOURCES = ["capi.cu", "pack.cu", "sketch.cu", "index.cu", "map.cu", "cgi.cu", "hits.cu", "synth.cu", "cubops.cu", "stats.cpp", "alloc.cpp", "budget.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17",
                   "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr", "-x", "cu"]


def _deps_mtime():
    m = 0.0
    for root, _, files in os.walk(CSRC):
        for f in files:
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    m = max(m, os.path.getmtime(os.path.join(HERE, "..", "include", "fastani_b200.h")))
    for f in os.listdir(os.path.join(HERE, "host")):
        m = max(m, os.path.getmtime(os.path.join(HERE, "host", f)))
    return m


def _stamp():
    """The flags the objects in OUT were compiled with: objects of other flags (another architecture) are rebuilt."""
    try:
        return open(STAMP).read()
    except OSError:
        return None


def _compile(src, verbose):
    obj = os.path.join(OUT, os.path.splitext(src)[0] + ".o")
    srcp = os.path.join(CSRC, src)
    hdr = max(os.path.getmtime(os.path.join(CSRC, "common.cuh")),
              os.path.getmtime(os.path.join(HERE, "..", "include", "fastani_b200.h")))
    if os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(srcp), hdr):
        return obj
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", srcp, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force=False, verbose=False):
    os.makedirs(OUT, exist_ok=True)
    if _stamp() != " ".join(FLAGS):
        force = True
        for f in os.listdir(OUT):
            if f.endswith(".o"):
                os.unlink(os.path.join(OUT, f))
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _deps_mtime():
        return LIB
    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), SOURCES))
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"]
    # link cudart statically so the library has no dependency on the loader's CUDA runtime version
    r = subprocess.run([NVCC] + GENCODE + ["-shared", "-Xcompiler", "-fPIC",
                        "-o", LIB] + objs + ["-cudart", "static"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(STAMP, "w") as f:
        f.write(" ".join(FLAGS))
    build_cli()
    return LIB


def build_cli():
    """The fastANI command line (C++ host above the C ABI): fastani_b200/bin/fastANI."""
    bindir = os.path.join(HERE, "bin")
    os.makedirs(bindir, exist_ok=True)
    exe = os.path.join(bindir, "fastANI")
    src = os.path.join(HERE, "host", "fastani_main.cpp")
    cmd = ["g++", "-O2", "-std=c++17", "-Wall", src, "-o", exe, "-L" + OUT, "-lfastani_b200", "-lz", "-lpthread",
           "-Wl,-rpath,$ORIGIN/../lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("CLI build failed:\n%s\n%s" % (r.stdout, r.stderr))
    return exe


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
