"""CPU oracle of `autocycler depth` (DESIGN.md §19), restated in numpy from the rule, not from the product's code.

Read-measured depth is not in the reference, so the oracle pins the rule: every contig window of k A/C/G/T bases (a contig whose header
holds "circular=true", any case, and is at least k long also gets the k-1 windows across its end), its canonical key (genome_size's,
tests/genome_size_oracle.py), the keys that occur once over all contigs, the read windows (genome_size's rule) that hit them, and each
contig's median count.  The filter and the header parser restate helper.rs:889-931.

    depths(assembly_path, reads_path, k) -> (records, unique per contig, depth per contig or None)
    run(assembly_path, reads_path, k, min_abs, min_rel) -> dict(fasta=bytes or None, tsv=str, report=str, depths, unique)
"""
import gzip
import math
import re

import numpy as np

import genome_size_oracle as G


def load_fasta(path):
    """misc.rs:248-321 without its error paths: [(name, header, sequence uppercased)]."""
    data = open(path, "rb").read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    recs = []
    for line in data.decode().split("\n"):
        line = line[:-1] if line.endswith("\r") else line
        if not line:
            continue
        if line.startswith(">"):
            recs.append((line[1:], []))
        else:
            recs[-1][1].append(line)
    return [(h.split()[0], h, "".join(s).upper()) for h, s in recs]


_NUM = re.compile(r"[+-]?(inf|infinity|nan|(\d+\.?\d*|\.\d+)(e[+-]?\d+)?)")


def depth_from_header(header):
    """helper.rs:923-931."""
    for key in ("depth=", "depth-", "coverage="):
        i = header.find(key)
        if i >= 0:
            num = re.split(r"[-_ ]", header[i + len(key):])[0]
            return float(num) if _NUM.fullmatch(num.lower()) else None
    return None


def rust_fixed(x, digits):
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    return f"{x:.{digits}f}"


def contig_keys(seq, header, k):
    ext = seq + seq[:k - 1] if "circular=true" in header.lower() and len(seq) >= k else seq
    codes = G._CODE[np.frombuffer(ext.encode() + b"\x00", dtype=np.uint8)]
    return G.canonical_keys(codes, k)


def depths(assembly, reads, k):
    recs = load_fasta(assembly)
    per = [contig_keys(s, h, k) for _, h, s in recs]
    allk = np.concatenate(per) if per else np.zeros(0, dtype=np.uint64)
    keys, counts = np.unique(allk, return_counts=True)
    uniq = keys[counts == 1]
    counts = np.zeros(len(uniq), dtype=np.int64)
    seqs = G.sequences(reads)
    for a in range(0, len(seqs), 2000):                      # the reads' keys in batches, so the memory stays bounded
        batch = seqs[a:a + 2000]
        rk = G.canonical_keys(G._CODE[np.frombuffer(b"\x00".join(batch) + b"\x00", dtype=np.uint8)], k)
        if len(uniq) and len(rk):
            idx = np.minimum(np.searchsorted(uniq, rk), len(uniq) - 1)
            hit = uniq[idx] == rk
            counts += np.bincount(idx[hit], minlength=len(uniq))
    unique, dep = [], []
    for p in per:
        at = np.minimum(np.searchsorted(uniq, p), max(len(uniq) - 1, 0))
        mine = p[uniq[at] == p] if len(uniq) else p[:0]           # np.isin(p, uniq), without a sort of uniq per contig
        unique.append(len(mine))
        if not len(mine):
            dep.append(None)
            continue
        c = counts[np.searchsorted(uniq, mine)]
        c = np.sort(c.astype(np.int64))
        n = len(c)
        dep.append((float(c[(n - 1) // 2]) + float(c[n // 2])) / 2.0)
    return recs, unique, dep


def depth_filter(recs, dep, min_abs, min_rel):
    """helper.rs:889-921 -> (ran, keep flags, report)."""
    if min_abs is None and min_rel is None or any(d is None for d in dep):
        return False, [True] * len(recs), ""
    longest_len, longest_depth = 0, 0.0
    for (_, _, s), d in zip(recs, dep):
        if len(s) > longest_len:
            longest_len, longest_depth = len(s), d
    threshold = 0.0 if min_abs is None else min_abs
    if min_rel is not None:
        t = min_rel * longest_depth
        threshold = t if math.isnan(threshold) else threshold if math.isnan(t) else max(threshold, t)
    report = f"\nAutocycler helper depth filter\nthreshold = {rust_fixed(threshold, 3)}\n"
    keep = []
    for (name, _, _), d in zip(recs, dep):
        keep.append(d >= threshold)
        report += f"{name}: depth={rust_fixed(d, 3)}, {'PASS' if keep[-1] else 'FAIL'}\n"
    return True, keep, report


def run(assembly, reads, k, min_abs=None, min_rel=None):
    recs, unique, dep = depths(assembly, reads, k)
    out = [(n, h + ("" if d is None else f" depth={rust_fixed(d, 2)}"), s) for (n, h, s), d in zip(recs, dep)]
    ran, keep, report = depth_filter(recs, dep, min_abs, min_rel)
    kept = [r for r, x in zip(out, keep) if x]
    fasta = "".join(f">{h}\n{s}\n" for _, h, s in kept).encode() if kept else None
    tsv = "".join(f"{n}\t{len(s)}\t{u}\t{'' if d is None else rust_fixed(d, 2)}\n" for (n, _, s), u, d in zip(recs, unique, dep))
    return {"fasta": fasta, "tsv": tsv, "report": report, "depths": dep, "unique": unique, "filtered": ran}
