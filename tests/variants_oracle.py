"""CPU oracle of `autocycler variants` (DESIGN.md §23), restated in numpy from the rule, not from the product's code.

`variants` is not in the reference, so the oracle pins the rule: contig windows, canonical keys, r(key) and the solid threshold t as
polish's (tests/polish_oracle.py) on the input sequence; at every tried position p (linear: p >= k - 1; circular: every p when the contig
is at least 2k + 2L long; and the window that ends at p a window) the screen windows S(p, b), the candidates of polish's enumeration in
their rightmost representation, each evaluated as polish's rule 3 (alt: the minimum r over its checked windows), ref (the minimum r over
the input's windows that start at p - k + 1 .. p + d), PK (checked windows whose key the input holds), the fraction test, and the
left-aligned VCF rows and the summary.

    run(reads_path, assembly_path, k, min_count=None, max_indel=1, min_fraction=0.1, counts=None)
        -> dict(files={name: bytes}, t, valley, W, rows=[row dicts], positions, screened, candidates, passing)
"""
import numpy as np

import depth_oracle as D
import genome_size_oracle as G
import polish_oracle as P
import qv_oracle as Q

NoWindows = Q.NoWindows
BASES = "ACGT"
CHUNK = 1 << 16


def screen(seq, circular, k, L, r, t):
    """-> (tried positions, their bits: bit b set when r(S(p, b)) >= t, as an int array).  A position is tried when it can be polish's
    p0 (see the module docstring) and the window that ends at it has k A/C/G/T bases."""
    n = len(seq)
    cs = P.codes(seq)
    if circular:
        pos = np.arange(n) if n >= 2 * k + 2 * L else np.zeros(0, dtype=np.int64)
    else:
        pos = np.arange(k - 1, n)
    if not len(pos):
        return pos, np.zeros(0, dtype=np.int64)
    ok = np.ones(len(pos), dtype=bool)
    for j in range(k):
        ok &= cs[(pos - j) % n] < 4
    pos = pos[ok]
    bits = np.zeros(len(pos), dtype=np.int64)
    for c0 in range(0, len(pos), CHUNK):
        p = pos[c0:c0 + CHUNK]
        rows = cs[(p[:, None] + np.arange(-k + 1, 1)[None, :]) % n].copy()
        for b in range(4):
            rows[:, -1] = b
            keys, _ = P.keys_of(rows, k)
            bits[c0:c0 + CHUNK] |= (r(keys[:, 0]) >= t).astype(np.int64) << b
    return pos, bits


def first_base(seq, circular, p, mid, skip):
    """The candidate's first base in E at p, or None when that base does not exist or is not A/C/G/T."""
    n = len(seq)
    if mid:
        return mid[0]
    d = skip
    if p + d >= n + (1 if circular else 0):
        return None
    b = seq[(p + d) % n]
    return b if b in BASES else None


def run(reads, assembly, k, min_count=None, max_indel=1, min_fraction=0.1, counts=None):
    L, F = max_indel, min_fraction
    recs = D.load_fasta(assembly)
    if sum(len(D.contig_keys(s, h, k)) for _, h, s in recs) == 0:
        raise NoWindows(assembly)
    if counts is None:
        uk, uc, W = Q.read_counts(reads, k)
        counts = (P.Counts(uk, uc), np.bincount(np.minimum(uc, G.H - 1), minlength=G.H).astype(np.int64), W)
    r, hist, W = counts
    if W == 0:
        raise NoWindows(reads)
    hist = hist.copy()
    hist[0] = 0
    v = Q.valley(hist)
    t = min_count if min_count is not None else v
    if t is None:
        raise G.NoPeak("no k-mer depth peak")
    # the input's own keys, over every contig (PK)
    own = []
    for _, h, s in recs:
        ext = s + s[:k - 1] if P.is_circular(h, s, k) else s
        if len(ext) >= k:
            keys, valid = P.keys_of(P.codes(ext), k)
            own.append(keys[valid])
    own = np.unique(np.concatenate(own)) if own else np.zeros(0, dtype=np.uint64)

    def held(keys):
        keys = np.asarray(keys, dtype=np.uint64)
        if not len(own):
            return np.zeros(len(keys), dtype=bool)
        idx = np.minimum(np.searchsorted(own, keys), len(own) - 1)
        return own[idx] == keys

    positions = screened = n_cand = passing = 0
    rows = []
    for ci_contig, (name, h, raw) in enumerate(recs):
        seq = raw.upper()
        n = len(seq)
        circ = P.is_circular(h, raw, k)
        pos, bits = screen(seq, circ, k, L, r, t)
        positions += len(pos)
        valid, rr = P.contig_windows(h, raw, k, r)
        ext = seq + seq if circ else seq
        evals = []                                           # (p, ci, mid, skip, X)
        for p, b in zip(pos.tolist(), bits.tolist()):
            cur = seq[p]
            alt_bits = b & ~(1 << BASES.index(cur))
            if not alt_bits:
                continue
            screened += 1
            for ci, (mid, skip) in enumerate(P.candidates(cur, L)):
                e = first_base(seq, circ, p, mid, skip)
                if e is None or e == cur or not (alt_bits >> BASES.index(e)) & 1:
                    continue
                n_cand += 1
                d = skip if mid == "" else 0
                s = len(mid) if skip == 0 else 0
                a = p - k + 1
                if p + d > n or (not circ and p + d + k > n):
                    continue
                lo = a + n if (circ and a < 0) else a
                pu = lo + k - 1
                x = ext[lo:pu] + mid + ext[pu + skip:pu + d + k]
                assert len(x) == 2 * k - 1 + s
                evals.append((p, ci, mid, skip, x))
        for p, ci, mid, skip, x in evals:
            keys, ok = P.keys_of(P.codes(x), k)
            cnt = r(keys)
            if not ok.all() or cnt.min() < t:
                continue
            passing += 1
            alt = int(cnt.min())
            d = skip if mid == "" else 0
            starts = np.arange(p - k + 1, p + d + 1)
            ref = int(np.where(valid[starts % n], rr[starts % n], 0).min()) if circ else int(np.where(valid[starts], rr[starts], 0).min())
            hk = held(keys)
            pk = int(hk[:-1].sum()) if ci >= 3 else int(hk.sum())
            if not float(alt) >= F * float(alt + ref):
                continue
            rows.append(dict(contig=ci_contig, name=name, p=p, ci=ci, mid=mid, skip=skip, alt=alt, ref=ref, pk=pk,
                             **vcf_fields(seq, p, ci, mid, skip)))
    rows.sort(key=lambda x: (x["contig"], x["pos"], x["p"], x["ci"]))
    subs = sum(x["ci"] < 3 for x in rows)
    dels = sum(x["ci"] >= 3 and x["mid"] == "" for x in rows)
    ins = len(rows) - subs - dels
    header = "##fileformat=VCFv4.2\n##source=autocycler variants\n"
    for name, _, s in recs:
        header += f"##contig=<ID={name},length={len(s)}>\n"
    header += INFO + "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n"
    body = "".join(f"{x['name']}\t{x['pos']}\t.\t{x['REF']}\t{x['ALT']}\t.\tPASS\t"
                   f"AF={x['alt'] / (x['alt'] + x['ref']):.4f};AK={x['alt']};RK={x['ref']};PK={x['pk']}\n" for x in rows)
    paralog = sum(x["pk"] > 0 for x in rows)
    alt_major = sum(x["alt"] > x["ref"] for x in rows)
    summary = ("contigs\tpositions\tscreened\tcandidates\tvariants\tsubstitutions\tinsertions\tdeletions\tparalog\talt_major\tmin_count\n"
               f"{len(recs)}\t{positions}\t{screened}\t{n_cand}\t{len(rows)}\t{subs}\t{ins}\t{dels}\t{paralog}\t{alt_major}\t{t}\n")
    files = {"variants.vcf": (header + body).encode(), "summary.tsv": summary.encode()}
    return {"files": files, "t": t, "valley": v, "W": W, "rows": rows, "positions": positions, "screened": screened, "candidates": n_cand,
            "passing": passing}


INFO = ('##INFO=<ID=AF,Number=A,Type=Float,Description="Alternative allele fraction AK / (AK + RK)">\n'
        '##INFO=<ID=AK,Number=A,Type=Integer,Description="Least read count of the k-mers that carry the alternative allele">\n'
        '##INFO=<ID=RK,Number=1,Type=Integer,Description="Least read count of the assembly k-mers the alternative allele replaces">\n'
        '##INFO=<ID=PK,Number=A,Type=Integer,Description="Alternative-allele k-mers that occur elsewhere in the assembly">\n')


def vcf_fields(seq, p, ci, mid, skip):
    """POS, REF and ALT of the candidate evaluated at p, indels left-aligned (seq uppercased)."""
    if ci < 3:
        return dict(pos=p + 1, REF=seq[p], ALT=mid)
    if mid == "":                                            # deletion of seq[p:p + d]
        d = skip
        while p > 1 and seq[p - 1] == seq[p + d - 1]:
            p -= 1
        if p == 0:
            return dict(pos=1, REF=seq[:d + 1], ALT=seq[d])
        return dict(pos=p, REF=seq[p - 1:p + d], ALT=seq[p - 1])
    s = mid                                                  # insertion of s before p
    while p > 1 and seq[p - 1] == s[-1]:
        s = s[-1] + s[:-1]
        p -= 1
    if p == 0:
        return dict(pos=1, REF=seq[0], ALT=s + seq[0])
    return dict(pos=p, REF=seq[p - 1], ALT=seq[p - 1] + s)
