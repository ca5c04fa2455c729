"""CPU: where a genome of a saved index lives.  host/ani_host.hpp referenceShardOrdinal, the inverse of splitReferenceGenomes,
must give every list position the (shard file, ordinal in that file) the partition put it at, for both partitions, any
shard count and lists shorter than the shard count (empty shards)."""
import os
import subprocess

from conftest import ROOT


def test_shard_ordinal_inverts_the_split(tmp_path):
    src = tmp_path / "s.cpp"
    src.write_text(r'''#include "ani_host.hpp"
#include <cstdio>
int main() {
  long checked = 0;
  for (int block = 0; block < 2; block++)
    for (int G = 1; G <= 9; G++)
      for (int n = 0; n <= 60; n++) {
        const auto s = cgi::splitReferenceGenomes(n, G, block != 0);
        for (int g = 0; g < G; g++)
          for (size_t i = 0; i < s[g].size(); i++) {
            const auto at = cgi::referenceShardOrdinal(s[g][i], n, G, block != 0);
            if (at.first != g || at.second != (int)i) {
              printf("block %d G %d n %d: position %d is ordinal %zu of shard %d, got (%d, %d)\n", block, G, n, s[g][i], i, g, at.first, at.second);
              return 1;
            }
            checked++;
          }
      }
  printf("ok %ld\n", checked);
}
''')
    exe = tmp_path / "s"
    libdir = os.path.join(ROOT, "fastani_b200", "lib")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "fastani_b200", "host"), "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-lfastani_b200", "-lz", "-lpthread", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("ok "), (r.stdout, r.stderr)
    assert int(r.stdout.split()[1]) == 2 * 9 * sum(range(61))
