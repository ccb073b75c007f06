"""CPU oracle of `autocycler qv` (DESIGN.md §20), restated in numpy from the rule, not from the product's code.

`qv` is not in the reference, so the oracle pins the rule: contig windows and their canonical keys as depth's (tests/depth_oracle.py),
read windows and the histogram as genome_size's (tests/genome_size_oracle.py), r(key) = the read windows with that key, the solid
threshold t (given, or the histogram's valley), each assembly's unsupported windows (r < t), its QV, completeness, BED of unsupported
bases (from a per-base coverage array) and Merqury's copy-number spectrum.

    run(reads_path, assembly_args, k, min_count=None) -> dict(files={relative path: bytes}, hist, W, valley, t, S, assemblies=[...])
"""
import math
import os

import numpy as np

import depth_oracle as D
import genome_size_oracle as G

H = G.H


class NoWindows(ValueError):
    pass


def inputs(args):
    """Each argument a FASTA file, or a directory whose assembly files (.fasta, .fa, .fna, gzipped or not) come in sorted order."""
    out = []
    for a in args:
        if os.path.isdir(a):
            names = sorted(n for n in os.listdir(a) if n.endswith((".fasta", ".fa", ".fna", ".fasta.gz", ".fa.gz", ".fna.gz")))
            out += [a.rstrip("/") + "/" + n for n in names]
        else:
            out.append(a)
    return out


def window_starts(seq, header, k):
    """The start of every contig window (the same order as depth_oracle.contig_keys' keys) in the sequence with its junction bases."""
    ext = seq + seq[:k - 1] if "circular=true" in header.lower() and len(seq) >= k else seq
    bad = np.concatenate([[0], np.cumsum(G._CODE[np.frombuffer(ext.encode(), dtype=np.uint8)] == 4)])
    n = len(ext) - k + 1
    return np.nonzero(bad[k:k + max(n, 0)] - bad[:max(n, 0)] == 0)[0] if n > 0 else np.zeros(0, dtype=np.int64)


def valley(hist):
    h = list(hist)
    s = lambda c: (h[c - 1] if c > 1 else h[1]) + h[c] + h[c + 1]    # noqa: E731
    return next((c for c in range(1, H - 2) if s(c) < s(c + 1)), None)


def qv_text(E, K, k):
    if K == 0:
        return ""
    if E == 0:
        return "inf"
    p = -math.expm1(math.log1p(-E / K) / k)
    return f"{-10.0 * math.log10(p) + 0.0:.2f}"


def read_counts(reads, k):
    """-> (sorted distinct read keys, their counts, W)."""
    seqs = G.sequences(reads)
    codes = G._CODE[np.frombuffer(b"\x00".join(seqs) + b"\x00", dtype=np.uint8)] if seqs else np.zeros(0, dtype=np.uint8)
    keys = G.canonical_keys(codes, k)
    del codes
    uk, uc = np.unique(keys, return_counts=True)
    return uk, uc, len(keys)


def run(reads, args, k, min_count=None):
    paths = inputs(args)
    loaded = []
    for p in paths:
        recs = D.load_fasta(p)
        keys = [D.contig_keys(s, h, k) for _, h, s in recs]
        if sum(len(x) for x in keys) == 0:
            raise NoWindows(p)
        loaded.append((p, recs, keys))
    uk, uc, W = read_counts(reads, k)
    if W == 0:
        raise NoWindows(reads)
    hist = np.bincount(np.minimum(uc, H - 1), minlength=H).astype(np.int64)
    hist[0] = 0
    v = valley(hist)
    t = min_count if min_count is not None else v
    if t is None:
        raise G.NoPeak("no k-mer depth peak")
    S = int(hist[t:].sum())

    def r_of(keys):
        if not len(uk):
            return np.zeros(len(keys), dtype=np.int64)
        idx = np.minimum(np.searchsorted(uk, keys), len(uk) - 1)
        return np.where(uk[idx] == keys, uc[idx], 0)

    files = {}
    qv_rows = ["assembly\tkmers\tunsupported\tqv\tsolid_found\tsolid_kmers\tcompleteness\tmin_count\n"]
    contig_rows = ["assembly\tcontig\tlength\tkmers\tunsupported\tqv\n"]
    summary = []
    for n, (p, recs, keys) in enumerate(loaded, 1):
        bed, K_a, E_a = [], 0, 0
        for (name, header, seq), ck in zip(recs, keys):
            starts = window_starts(seq, header, k)
            assert len(starts) == len(ck)
            bad = r_of(ck) < t
            K, E = len(ck), int(bad.sum())
            K_a += K
            E_a += E
            contig_rows.append(f"{p}\t{name}\t{len(seq)}\t{K}\t{E}\t{qv_text(E, K, k)}\n")
            cover = np.zeros(len(seq) + 1, dtype=np.int64)        # a difference array of the bases each unsupported window covers
            for s in starts[bad]:
                for a, b in ((s, min(s + k, len(seq))), (0, s + k - len(seq))):
                    if b > a:
                        cover[a] += 1
                        cover[b] -= 1
            on = np.concatenate([[0], (np.cumsum(cover)[:len(seq)] > 0).astype(np.int8), [0]])
            edges = np.nonzero(np.diff(on))[0]
            bed += [f"{name}\t{a}\t{b}\n" for a, b in zip(edges[0::2], edges[1::2])]
        allk = np.concatenate(keys)
        ak, am = np.unique(allk, return_counts=True)
        cnt = np.zeros((H, 5), dtype=np.int64)
        np.add.at(cnt, (np.minimum(r_of(ak), H - 1), np.minimum(am, 4)), 1)
        found = int(cnt[t:, 1:].sum())
        spectrum = ["count\tcn0\tcn1\tcn2\tcn3\tcn4+\n"]
        for c in range(H):
            in_asm = int(cnt[c, 1:].sum())
            cn0 = int(hist[c]) - in_asm if c else 0
            assert cn0 >= 0
            if cn0 or in_asm:
                spectrum.append(f"{c}\t{cn0}\t" + "\t".join(str(int(x)) for x in cnt[c, 1:]) + "\n")
        completeness = f"{100.0 * found / S:.2f}" if S else ""
        qv_rows.append(f"{p}\t{K_a}\t{E_a}\t{qv_text(E_a, K_a, k)}\t{found}\t{S}\t{completeness}\t{t}\n")
        files[f"unsupported/{n}.bed"] = "".join(bed).encode()
        files[f"spectra_cn/{n}.tsv"] = "".join(spectrum).encode()
        summary.append({"path": p, "kmers": K_a, "unsupported": E_a, "solid_found": found, "spectrum": cnt})
    files["qv.tsv"] = "".join(qv_rows).encode()
    files["contig_qv.tsv"] = "".join(contig_rows).encode()
    files["kmer_histogram.tsv"] = "".join(f"{c}\t{int(hist[c])}\n" for c in range(1, H) if hist[c]).encode()
    return {"files": files, "hist": hist, "W": W, "valley": v, "t": t, "S": S, "assemblies": summary}
