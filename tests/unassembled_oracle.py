"""CPU oracle of `autocycler unassembled` (DESIGN.md §21), restated in numpy from the rule, not from the product's code.

`unassembled` is not in the reference, so the oracle pins the rule: the inputs, contig windows, read counts r(key), histogram and valley
as qv's (tests/qv_oracle.py); A = the canonical keys of every input's contigs together; per read, s = its windows whose key has r >= t
and a = those of them whose key is not in A; a read is scored when s >= min_solid and selected when also a >= F s (one f64 multiply);
the absent keys are the distinct keys with r >= t not in A; p* is genome_size's refined peak (tests/genome_size_oracle.py).

    run(reads_path, assembly_args, k, min_count=None, min_solid=100, min_fraction=0.5)
        -> dict(files={name: bytes}, t, valley, s, a, selected=[read index], absent_kmers, ...)
"""
import numpy as np

import depth_oracle as D
import genome_size_oracle as G
import qv_oracle as Q
import subsample_oracle

H = G.H
NoWindows = Q.NoWindows


def read_windows(seqs, k):
    """-> (canonical keys of every read window, in input order, and the read each belongs to)."""
    codes = G._CODE[np.frombuffer(b"\x00".join(seqs) + b"\x00", dtype=np.uint8)] if seqs else np.zeros(0, dtype=np.uint8)
    keys = G.canonical_keys(codes, k)
    n = len(codes) - k + 1
    bad = np.concatenate([[0], np.cumsum(codes == 4, dtype=np.int64)])
    pos = np.nonzero(bad[k:k + max(n, 0)] - bad[:max(n, 0)] == 0)[0] if n > 0 else np.zeros(0, dtype=np.int64)
    assert len(pos) == len(keys)
    starts = np.concatenate([[0], np.cumsum([len(s) + 1 for s in seqs])])
    return keys, np.searchsorted(starts, pos, side="right") - 1


def median_text(absent_bins):
    n = len(absent_bins)
    if n == 0:
        return None
    v = np.sort(absent_bins)
    return (float(v[(n - 1) // 2]) + float(v[n // 2])) / 2.0


def run(reads, args, k, min_count=None, min_solid=100, min_fraction=0.5):
    paths = Q.inputs(args)
    asm_keys = [D.contig_keys(s, h, k) for p in paths for _, h, s in D.load_fasta(p)]
    A = np.unique(np.concatenate(asm_keys)) if asm_keys else np.zeros(0, dtype=np.uint64)
    if len(A) == 0:
        raise NoWindows(", ".join(paths))
    recs = subsample_oracle.parse_fastq(subsample_oracle.read_bytes(reads))
    seqs = [r[1] for r in recs]
    keys, rid = read_windows(seqs, k)
    W = len(keys)
    if W == 0:
        raise NoWindows(reads)
    uk, uc = np.unique(keys, return_counts=True)
    hist = np.bincount(np.minimum(uc, H - 1), minlength=H).astype(np.int64)
    hist[0] = 0
    v = Q.valley(hist)
    t = min_count if min_count is not None else v
    if t is None:
        raise G.NoPeak("no k-mer depth peak")
    r = uc[np.searchsorted(uk, keys)]
    solid = r >= t
    in_a = np.isin(keys, A)
    n = len(recs)
    s = np.bincount(rid[solid], minlength=n).astype(np.int64)
    a = np.bincount(rid[solid & ~in_a], minlength=n).astype(np.int64)
    lengths = np.array([len(x) for x in seqs], dtype=np.int64)
    scored = s >= min_solid
    selected = [i for i in range(n) if scored[i] and float(a[i]) >= min_fraction * float(s[i])]
    frac_reads, frac_bases = np.zeros(101, dtype=np.int64), np.zeros(101, dtype=np.int64)
    for i in np.nonzero(scored)[0]:
        b = (100 * int(a[i])) // int(s[i])
        frac_reads[b] += 1
        frac_bases[b] += int(lengths[i])
    absent_mask = (uc >= t) & ~np.isin(uk, A)
    absent_bins = np.minimum(uc[absent_mask], H - 1)
    absent = np.bincount(absent_bins, minlength=H)
    med = median_text(absent_bins)
    try:
        peak = G.estimate(list(hist), W)["peak_refined"]
    except (G.NoPeak, G.PeakAtCap, ZeroDivisionError):
        peak = None
    if peak is not None and not peak > 0:
        peak = None
    ratio = med / peak if med is not None and peak is not None else None
    fmt = lambda x, d: "" if x is None else f"{x:.{d}f}"    # noqa: E731
    summary = ("reads\tread_windows\tmin_count\tscored_reads\tselected_reads\tselected_bases\tabsent_kmers\tabsent_median\tpeak\t"
               "absent_copy_ratio\n"
               f"{n}\t{W}\t{t}\t{int(scored.sum())}\t{len(selected)}\t{int(lengths[selected].sum())}\t{len(absent_bins)}\t{fmt(med, 1)}\t"
               f"{fmt(peak, 2)}\t{fmt(ratio, 2)}\n")
    table = ["read\tlength\tsolid_kmers\tabsent_kmers\n"]
    for i in selected:
        name = recs[i][0].split(b" ")[0].split(b"\t")[0].decode()
        table.append(f"{name}\t{lengths[i]}\t{s[i]}\t{a[i]}\n")
    files = {
        "unassembled.fastq": b"".join(subsample_oracle.record_bytes(recs[i]) for i in selected),
        "unassembled.tsv": "".join(table).encode(),
        "fraction_histogram.tsv": ("percent\treads\tbases\n" + "".join(f"{b}\t{frac_reads[b]}\t{frac_bases[b]}\n" for b in range(101))).encode(),
        "absent_histogram.tsv": "".join(f"{c}\t{int(absent[c])}\n" for c in range(1, H) if absent[c]).encode(),
        "kmer_histogram.tsv": "".join(f"{c}\t{int(hist[c])}\n" for c in range(1, H) if hist[c]).encode(),
        "summary.tsv": summary.encode(),
    }
    return {"files": files, "t": t, "valley": v, "W": W, "s": s, "a": a, "selected": selected, "absent_kmers": len(absent_bins),
            "absent_median": med, "peak": peak, "ratio": ratio, "hist": hist}
