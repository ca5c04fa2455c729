"""Host glue after the hot path: the output filter and text format of cgi::outputCGI
(src/cgi/include/computeCoreIdentity.hpp:307-343), computeGenomeLengths (:48-92) and outputVisualizationFile (:103-153)."""
import numpy as np


def genome_length(contig_lens, frag_len):
    """computeCoreIdentity.hpp:57-61: sum over contigs >= fragLen of floor(len/fragLen)*fragLen."""
    return int(sum((int(L) // frag_len) * frag_len for L in contig_lens if L >= frag_len))


def fmt_float(x):
    """std::ostream << float with default precision (6 significant digits, %g)."""
    return "%g" % float(np.float32(x))


def output_lines(results, query_names, ref_names, query_lens, ref_lens, frag_len, min_fraction=0.2):
    """results: iterable of (qryGenomeId, refGenomeId, countSeq, totalQueryFragments, identity).
    Ordered as outputCGI: query ascending, identity descending (cgid_types.hpp:76-79)."""
    rows = sorted(results, key=lambda r: (r[0], -float(r[4])))
    out = []
    for q, r, cnt, tot, idn in rows:
        min_len = min(query_lens[q], ref_lens[r])
        shared = cnt * frag_len
        if shared >= np.float32(min_len) * np.float32(min_fraction):        # uint64 * float -> float (:326-332)
            out.append("%s\t%s\t%s\t%d\t%d" % (query_names[q], ref_names[r], fmt_float(idn), cnt, tot))
    return out


def fragment_lengths(contig_lens, frag_len, kmer_size, window_size):
    """Map::metadata of one query genome (computeMap.hpp:138-167): a contig too short to map counts as one entry of
    its length; any other contig gives len // frag_len fragments of frag_len, the last one extended by len % frag_len.
    Entry i belongs to querySeqId i."""
    out = []
    for L in contig_lens:
        L = int(L)
        if L < window_size or L < kmer_size or L < frag_len:
            out.append(L)
            continue
        fc = L // frag_len
        out += [frag_len] * (fc - 1) + [frag_len + L % frag_len]
    return out


def _offsets(lens):
    off = np.zeros(len(lens) + 1, np.int64)
    if len(lens):
        off[1:] = np.cumsum(np.asarray(lens, np.int64))
    return off


def visual_lines(frags, query_names, ref_names, query_frag_lens, ref_contig_lens, seqs_by_file, frag_len):
    """outputVisualizationFile: one line per 2-way mapping.
    frags: FRAG_DTYPE records (compute_cgi_sketched(..., fragments=True)), written in the order given.
    query_names[q] / query_frag_lens[q]: name and fragment_lengths() of the query with qryGenomeId q (list or dict).
    ref_names[g]: name of genome g of the index; ref_contig_lens: contig lengths of the index in seqId order;
    seqs_by_file: its cumulative contig count per genome (Sketch.sequencesByFileInfo).
    Query and reference coordinates are offsets into the concatenated fragments and contigs (int64)."""
    ref_off = _offsets(ref_contig_lens)
    sbf = np.asarray(seqs_by_file, np.int64)
    q_off = {}
    out = []
    for f in frags:
        q, qs, rs, rp = int(f["qryGenomeId"]), int(f["querySeqId"]), int(f["refSeqId"]), int(f["refStartPos"])
        if q not in q_off:
            q_off[q] = _offsets(query_frag_lens[q])
        g = int(np.searchsorted(sbf, rs, side="right"))               # upper_bound over sequencesByFileInfo
        qa, ra = int(q_off[q][qs]), rp + int(ref_off[rs])
        out.append("%s\t%s\t%s\tNA\tNA\tNA\t%d\t%d\t%d\t%d\tNA\tNA" % (
            query_names[q], ref_names[g], fmt_float(f["identity"]), qa, qa + frag_len - 1, ra, ra + frag_len - 1))
    return out
