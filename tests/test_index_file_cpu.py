"""Saved index files without a GPU: bani_index_file_info reads and checks the header and tables of the version-3 layout
(DESIGN.md section 3, "Sketch cache on disk"), written here by hand from that description."""
import numpy as np
import pytest

import fastani_b200 as fb

MAGIC = 0x32584449494e4142


def _sum(*arrays):
    """64-bit sum of the 32-bit little-endian words of the arrays' bytes."""
    return sum(int(np.frombuffer(np.ascontiguousarray(a).tobytes(), "<u4").astype(np.uint64).sum()) for a in arrays) & (2 ** 64 - 1)


def _layout(contig_len, seqs_by_file, rec_per_contig, k=16, w=24, frag_len=3000, seed=0):
    """The sections of a version-3 file with random records: header, tables, hash, wpos, bitmap."""
    rng = np.random.default_rng(seed)
    contig_len = np.asarray(contig_len, "<i4")
    sbf = np.asarray(seqs_by_file, "<i4")
    rec_off = np.zeros(len(contig_len) + 1, "<u4")
    rec_off[1:] = np.cumsum(rec_per_contig)
    m = int(rec_off[-1])
    bits = int(sum((int(x) + 31) & ~31 for x in contig_len))
    valid_words = bits // 32 + 1 if m else 0
    hdr = np.zeros(16, "<u8")
    hdr[:9] = [MAGIC, 3, k, w, frag_len, m, len(contig_len), len(sbf), valid_words]
    hsh = rng.integers(0, 2 ** 32, m, dtype=np.uint64).astype("<u4")
    wpos = rng.integers(0, 1000, m).astype("<i4")
    vb = rng.integers(0, 2 ** 32, valid_words, dtype=np.uint64).astype("<u4")
    if valid_words:
        vb[-1] = 0
    return dict(hdr=hdr, contig_len=contig_len, sbf=sbf, rec_off=rec_off, hash=hsh, wpos=wpos, bits=vb)


def _write(path, s, table_sum=None):
    """A version-3 file of the sections: the table checksum (recomputed unless given), one checksum per genome over its
    hash and wpos slices and its bitmap words, and the whole-file checksum."""
    tables = [s["hdr"], s["contig_len"], s["sbf"], s["rec_off"]]
    ts = _sum(*tables) if table_sum is None else table_sum
    c0 = np.concatenate([[0], s["sbf"][:-1]]).astype(int) if len(s["sbf"]) else np.zeros(0, int)
    bit_off = np.concatenate([[0], np.cumsum([(int(x) + 31) & ~31 for x in s["contig_len"]])]).astype(int)
    gsum = []
    for a, b in zip(c0, s["sbf"].astype(int)):
        r0, r1 = int(s["rec_off"][a]), int(s["rec_off"][b])
        w0, w1 = bit_off[a] // 32, bit_off[b] // 32
        gsum.append(_sum(s["hash"][r0:r1], s["wpos"][r0:r1], s["bits"][w0:w1] if len(s["bits"]) else s["bits"]))
    body = tables + [s["hash"], s["wpos"], s["bits"], np.array([ts], "<u8"), np.array(gsum, "<u8")]
    blob = b"".join(np.ascontiguousarray(a).tobytes() for a in body)
    blob += np.array([_sum(np.frombuffer(blob, "<u4"))], "<u8").tobytes()
    open(path, "wb").write(blob)
    return blob


def _small():
    # 3 genomes: 2 contigs (one shorter than a word of bits), 1 contig, 3 contigs
    return _layout([100, 20, 5000, 40, 33, 64], [2, 3, 6], [7, 0, 300, 2, 1, 4])


def test_index_file_info_reads_counts_and_lengths(tmp_path):
    s = _small()
    path = str(tmp_path / "db.idx")
    _write(path, s)
    info = fb.index_file_info(path)
    assert (info["version"], info["k"], info["w"], info["frag_len"]) == (3, 16, 24, 3000)
    assert (info["n_genomes"], info["n_contigs"], info["n_minimizers"]) == (3, 6, 314)
    assert info["genome_contigs"].tolist() == [2, 1, 3]
    assert info["genome_length"].tolist() == [120, 5000, 137]
    assert info["genome_records"].tolist() == [7, 300, 7]
    assert info["genome_bits"].tolist() == [128 + 32, 5024, 64 + 64 + 64]
    assert info["contig_length"].tolist() == [100, 20, 5000, 40, 33, 64]


def test_index_file_info_empty_index(tmp_path):
    s = _layout([], [], [])
    path = str(tmp_path / "empty.idx")
    _write(path, s)
    info = fb.index_file_info(path)
    assert (info["n_genomes"], info["n_contigs"], info["n_minimizers"]) == (0, 0, 0)


def _refused(path, words):
    with pytest.raises(fb.BaniError) as e:
        fb.index_file_info(path)
    assert e.value.code == -1 and any(w in str(e.value) for w in words), str(e.value)


def test_index_file_info_refuses_corrupt_files(tmp_path):
    s = _small()
    path = str(tmp_path / "db.idx")
    blob = _write(path, s)
    # a flipped byte in the contig table: the table checksum no longer matches
    bad = bytearray(blob)
    bad[128 + 4 * 2 + 1] ^= 0x10
    open(path, "wb").write(bytes(bad))
    _refused(path, ["table checksum"])
    # a wrong table checksum over intact tables
    _write(path, s, table_sum=_sum(s["hdr"], s["contig_len"], s["sbf"], s["rec_off"]) + 1)
    _refused(path, ["table checksum"])
    # truncated
    open(path, "wb").write(blob[:-12])
    _refused(path, ["truncated"])
    # record offsets that go down (the table checksum recomputed: the check itself refuses it)
    t = _small()
    t["rec_off"][2], t["rec_off"][3] = t["rec_off"][3], t["rec_off"][2]
    _write(path, t)
    _refused(path, ["record offsets"])
    # a genome table that does not end at the contig count
    t = _small()
    t["sbf"][-1] = 5
    _write(path, t)
    _refused(path, ["genome table"])
    # not an index file
    open(path, "wb").write(b"\0" * 256)
    _refused(path, ["not a fastani_b200 index"])
