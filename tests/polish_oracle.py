"""CPU oracle of `autocycler polish` (DESIGN.md §22), restated in numpy from the rule, not from the product's code.

`polish` is not in the reference, so the oracle pins the rule: contig windows, canonical keys, r(key) and the solid threshold t as qv's
(tests/qv_oracle.py); per round the loci (maximal runs of window starts with r < t, cyclic on a circular contig), the candidate edits at
p0 = a + k - 1 in their fixed order, each scored by the minimum r over the k + s windows of the edited sequence that cover it, the unique
best accepted, the edits whose spans overlap a kept one's deferred, and the kept edits applied together; then the final windows, BED and
summary.  r comes from a lookup of the reads' distinct keys and their counts (`Counts`), which the caller may build once for several runs.

    run(reads_path, assembly_path, k, min_count=None, max_indel=3, rounds=3, counts=None)
        -> dict(files={name: bytes}, t, valley, W, edits=[(round, contig, position, ref, alt, score)], rounds=[row dicts], seqs)
"""
import itertools

import numpy as np

import depth_oracle as D
import genome_size_oracle as G
import qv_oracle as Q

NoWindows = Q.NoWindows
BASES = "ACGT"


class Counts:
    """r(key): the read windows with that canonical key, from the sorted distinct keys uk and their counts uc."""

    def __init__(self, uk, uc):
        self.uk, self.uc = uk, uc

    def __call__(self, keys):
        keys = np.asarray(keys, dtype=np.uint64)
        if not len(self.uk) or not len(keys):
            return np.zeros(len(keys), dtype=np.int64)
        idx = np.minimum(np.searchsorted(self.uk, keys), len(self.uk) - 1)
        return np.where(self.uk[idx] == keys, self.uc[idx], 0).astype(np.int64)


def keys_of(rows, k):
    """rows: uint8 codes (0..3 for A/C/G/T, 4 otherwise), shape (..., m).  -> (the canonical key of every window of k codes along the
    last axis, whether its k codes are all A/C/G/T), shape (..., m - k + 1)."""
    win = np.lib.stride_tricks.sliding_window_view(rows, k, axis=-1)
    fwd = np.zeros(win.shape[:-1], dtype=np.uint64)
    rev = np.zeros(win.shape[:-1], dtype=np.uint64)
    for j in range(k):
        x = (win[..., j] & 3).astype(np.uint64)
        fwd = (fwd << np.uint64(2)) | x
        rev |= (np.uint64(3) - x) << np.uint64(2 * j)
    return np.minimum(fwd, rev), (win < 4).all(axis=-1)


def codes(s):
    return G._CODE[np.frombuffer(s.encode(), dtype=np.uint8)]


def is_circular(header, seq, k):
    return "circular=true" in header.lower() and len(seq) >= k


def contig_windows(header, seq, k, r):
    """-> (valid, r) of every window start: 0 .. n-k on a linear contig, 0 .. n-1 on a circular one (its k-1 junction windows)."""
    ext = seq + seq[:k - 1] if is_circular(header, seq, k) else seq
    if len(ext) < k:
        return np.zeros(0, dtype=bool), np.zeros(0, dtype=np.int64)
    keys, valid = keys_of(codes(ext), k)
    return valid, np.where(valid, r(keys), 0)


def bed(name, n, starts, k):
    """qv's BED lines of one contig: the bases covered by the windows at `starts`, split at a circular contig's end, merged."""
    cover = np.zeros(n + 1, dtype=np.int64)
    for s in starts:
        for a, b in ((s, min(s + k, n)), (0, s + k - n)):
            if b > a:
                cover[a] += 1
                cover[b] -= 1
    on = np.concatenate([[0], (np.cumsum(cover)[:n] > 0).astype(np.int8), [0]])
    edges = np.nonzero(np.diff(on))[0]
    return "".join(f"{name}\t{a}\t{b}\n" for a, b in zip(edges[0::2], edges[1::2]))


def candidates(cur, L):
    """The candidates at p0 in their order, as (bases put at p0, bases of the sequence they replace): the three other bases, the
    deletions of 1..L bases, then every string of 1..L bases inserted before p0, each length in lexicographic order."""
    out = [(b, 1) for b in BASES if b != cur]
    out += [("", d) for d in range(1, L + 1)]
    out += [("".join(p), 0) for s in range(1, L + 1) for p in itertools.product(BASES, repeat=s)]
    return out


def loci(valid, r, t, n, circular, k, L):
    """-> [(a, attempted)] in ascending a."""
    bad = valid & (r < t)
    idx = np.nonzero(bad)[0]
    if not len(idx):
        return []
    cut = np.nonzero(np.diff(idx) != 1)[0]
    runs = [[int(x[0]), int(x[-1])] for x in np.split(idx, cut + 1)]
    whole = circular and len(idx) == n
    if circular and len(runs) > 1 and runs[0][0] == 0 and runs[-1][1] == n - 1:
        runs[0][0] = runs.pop()[0]
    out = []
    for a, _ in runs:
        prev = (a - 1) % n if circular else a - 1
        ok = prev >= 0 and bool(valid[prev]) and r[prev] >= t
        if circular:
            ok = ok and not whole and n >= 2 * k + 2 * L
        out.append((a, ok))
    return sorted(out)


def choose(tried, seqs, k, L, t, r):
    """tried: [(contig, a)] of every attempted locus of the round, with seqs the round's sequences and circular flags.  -> per locus
    (best score or 0, candidates at it, the first of them, its (mid, skip))."""
    rows = {}                        # X length -> [(locus, candidate, X)]
    per = []
    for li, (c, a) in enumerate(tried):
        seq, circ = seqs[c]
        n = len(seq)
        p0 = (a + k - 1) % n
        cands = candidates(seq[p0], L)
        per.append(cands)
        ext = seq + seq if circ else seq
        for ci, (mid, skip) in enumerate(cands):
            d = skip if mid == "" else 0                      # the bases it deletes
            s = len(mid) if skip == 0 else 0                  # the bases it inserts
            if p0 + d > n:                                    # a deletion past the contig's last base
                continue
            if not circ and a + (k + s - 1) + k > n - skip + len(mid):
                continue                                      # the last checked window would pass a linear contig's end
            # E's bases [a, a + 2k - 1 + s): the round's [a, p0), the edit's bases, then the round's from p0 + skip to p0 + d + k
            p = a + k - 1
            x = ext[a:p] + mid + ext[p + skip:p + d + k]
            assert len(x) == 2 * k - 1 + s
            rows.setdefault(len(x), []).append((li, ci, x))
    score = [np.zeros(len(c), dtype=np.int64) for c in per]
    for xs in rows.values():
        arr = codes("".join(x for _, _, x in xs)).reshape(len(xs), -1)
        keys, valid = keys_of(arr, k)
        rr = r(keys.ravel()).reshape(keys.shape)
        m = rr.min(axis=1)
        ok = valid.all(axis=1) & (m >= t)
        for (li, ci, _), good, v in zip(xs, ok, m):
            if good:
                score[li][ci] = v
    out = []
    for li, s in enumerate(score):
        best = int(s.max()) if len(s) else 0
        if best == 0:
            out.append((0, 0, 0, None))
        else:
            at = np.nonzero(s == best)[0]
            out.append((best, len(at), int(at[0]), per[li][int(at[0])]))
    return out


def run(reads, assembly, k, min_count=None, max_indel=3, rounds=3, counts=None):
    L = max_indel
    recs = D.load_fasta(assembly)
    if sum(len(D.contig_keys(s, h, k)) for _, h, s in recs) == 0:
        raise NoWindows(assembly)
    if counts is None:
        uk, uc, W = Q.read_counts(reads, k)
        counts = (Counts(uk, uc), np.bincount(np.minimum(uc, G.H - 1), minlength=G.H).astype(np.int64), W)
    r, hist, W = counts
    if W == 0:
        raise NoWindows(reads)
    hist = hist.copy()
    hist[0] = 0
    v = Q.valley(hist)
    t = min_count if min_count is not None else v
    if t is None:
        raise G.NoPeak("no k-mer depth peak")
    seqs = [s for _, _, s in recs]

    def evaluate():
        return [contig_windows(h, s, k, r) for (_, h, _), s in zip(recs, seqs)]

    def totals(ev):
        return sum(int(va.sum()) for va, _ in ev), sum(int((va & (rr < t)).sum()) for va, rr in ev)

    ev = evaluate()
    K0, E0 = totals(ev)
    edits, round_rows = [], []
    for rnd in range(1, rounds + 1):
        row = dict(unsupported=totals(ev)[1], loci=0, edited=0, ambiguous=0, none=0, edge=0, deferred=0)
        circ = [is_circular(h, s, k) for (_, h, _), s in zip(recs, seqs)]
        per_contig = [loci(va, rr, t, len(s), c, k, L) for (va, rr), s, c in zip(ev, seqs, circ)]
        tried = [(c, a) for c, ls in enumerate(per_contig) for a, ok in ls if ok]
        chosen = iter(choose(tried, list(zip(seqs, circ)), k, L, t, r))
        new = []
        for c, ls in enumerate(per_contig):
            seq, n = seqs[c], len(seqs[c])
            row["loci"] += len(ls)
            kept = []                                        # (a, span length, p0, mid, skip, score)
            for a, ok in ls:
                if not ok:
                    row["edge"] += 1
                    continue
                best, tied, _, cand = next(chosen)
                if best == 0:
                    row["none"] += 1
                    continue
                if tied > 1:
                    row["ambiguous"] += 1
                    continue
                mid, skip = cand
                d = skip if mid == "" else 0
                span = 2 * k - 1 + d                         # the round's bases [a, p0 + d + k)
                if kept:
                    ka = np.array([x[0] for x in kept])
                    kl = np.array([x[1] for x in kept])
                    if circ[c]:
                        hit = ((a - ka) % n < kl) | ((ka - a) % n < span)
                    else:
                        hit = (ka < a + span) & (a < ka + kl)
                    if hit.any():
                        row["deferred"] += 1
                        continue
                kept.append((a, span, (a + k - 1) % n, mid, skip, best))
            kept.sort(key=lambda x: x[2])
            pieces, at = [], 0
            for _, _, p0, mid, skip, best in kept:
                edits.append((rnd, recs[c][0], p0, seq[p0:p0 + skip] if skip else "-", mid or "-", best))
                pieces += [seq[at:p0], mid]
                at = p0 + skip
            new.append("".join(pieces) + seq[at:])
            row["edited"] += len(kept)
        seqs = new
        round_rows.append(row)
        ev = evaluate()
        if row["edited"] == 0:
            break
    K1, E1 = totals(ev)
    remaining = ""
    for (name, h, _), s, (va, rr) in zip(recs, seqs, ev):
        remaining += bed(name, len(s), np.nonzero(va & (rr < t))[0], k)
    files = {
        "polished.fasta": "".join(f">{h}\n{s}\n" for (_, h, _), s in zip(recs, seqs)).encode(),
        "edits.tsv": ("round\tcontig\tposition\tref\talt\tscore\n" + "".join("\t".join(map(str, e)) + "\n" for e in edits)).encode(),
        "rounds.tsv": ("round\tunsupported\tloci\tedited\tambiguous\tnone\tedge\tdeferred\n" + "".join(
            f"{i}\t{x['unsupported']}\t{x['loci']}\t{x['edited']}\t{x['ambiguous']}\t{x['none']}\t{x['edge']}\t{x['deferred']}\n"
            for i, x in enumerate(round_rows, 1))).encode(),
        "remaining.bed": remaining.encode(),
        "summary.tsv": ("contigs\tkmers_before\tunsupported_before\tqv_before\tedits\tkmers_after\tunsupported_after\tqv_after\tmin_count\t"
                        f"rounds\n{len(recs)}\t{K0}\t{E0}\t{Q.qv_text(E0, K0, k)}\t{len(edits)}\t{K1}\t{E1}\t{Q.qv_text(E1, K1, k)}\t{t}\t"
                        f"{len(round_rows)}\n").encode(),
    }
    return {"files": files, "t": t, "valley": v, "W": W, "edits": edits, "rounds": round_rows, "seqs": seqs}
