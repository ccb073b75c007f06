"""CPU oracle of `autocycler helper genome_size` (DESIGN.md §18), restated in numpy from the rule, not from the product's code.

This command departs from the reference on purpose (the reference runs Raven and prints the assembly's length), so the oracle pins the
rule itself: every window of k bases that are all A/C/G/T (any case) inside one read, its canonical 2-bit key min(forward, reverse
complement), the histogram of the distinct keys' counts (the last of H bins holds every count >= H - 1), and the estimate from that
histogram.  The keys are counted by np.unique per partition (a multiplicative hash of the key), each partition spilled to a temporary
file first, so the memory stays bounded by one partition.

    histogram(reads_path, k) -> (hist as a list of H ints, W)
    estimate(hist, W) -> dict(estimate, valley, peak, peak_refined, solid, distinct) or raises NoPeak / PeakAtCap
"""
import math
import os
import tempfile

import numpy as np

import subsample_oracle

H = 16384
CHUNK = 1 << 24                      # windows per numpy chunk
PART_WINDOWS = 1 << 27               # windows per partition file, at most about


class NoPeak(ValueError):
    pass


class PeakAtCap(ValueError):
    pass


_CODE = np.full(256, 4, dtype=np.uint8)
for _i, _c in enumerate(b"ACGT"):
    _CODE[_c] = _i
    _CODE[_c + 32] = _i              # lowercase


def sequences(path):
    """The reads' sequences, as subsample's parser reads them (FastqError on a malformed file)."""
    return [r[1] for r in subsample_oracle.parse_fastq(subsample_oracle.read_bytes(path))]


def canonical_keys(codes, k):
    """codes: uint8, 0..3 for A/C/G/T and 4 for anything else (reads separated by a 4).  -> the canonical keys of its valid windows."""
    n = len(codes) - k + 1
    out = []
    bad = np.concatenate([[0], np.cumsum(codes == 4, dtype=np.int64)])
    for a in range(0, max(n, 0), CHUNK):
        b = min(n, a + CHUNK)
        ok = bad[a + k:b + k] - bad[a:b] == 0
        if not ok.any():
            continue
        c = codes[a:b + k - 1].astype(np.uint64) & np.uint64(3)
        fwd = np.zeros(b - a, dtype=np.uint64)
        rev = np.zeros(b - a, dtype=np.uint64)
        for j in range(k):
            x = c[j:j + b - a]
            fwd = (fwd << np.uint64(2)) | x
            rev |= (np.uint64(3) - x) << np.uint64(2 * j)
        out.append(np.minimum(fwd, rev)[ok])
    return np.concatenate(out) if out else np.zeros(0, dtype=np.uint64)


def histogram(path, k, seqs=None):
    """-> (hist, W): hist[c] = distinct canonical k-mers seen c times (c < H - 1), hist[H - 1] = those seen H - 1 times or more."""
    seqs = sequences(path) if seqs is None else seqs
    total = sum(len(s) + 1 for s in seqs)
    codes = _CODE[np.frombuffer(b"\x00".join(seqs) + b"\x00", dtype=np.uint8)] if seqs else np.zeros(0, dtype=np.uint8)
    assert len(codes) == total
    keys = canonical_keys(codes, k)
    del codes
    W = len(keys)
    parts = max(1, -(-W // PART_WINDOWS))
    hist = np.zeros(H, dtype=np.int64)

    def add(part_keys):
        _, counts = np.unique(part_keys, return_counts=True)
        np.add.at(hist, np.minimum(counts, H - 1), 1)

    if parts == 1:
        add(keys)
    else:
        with tempfile.TemporaryDirectory() as tmp:
            with np.errstate(over="ignore"):
                which = ((keys * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(40)) % np.uint64(parts)
            for p in range(parts):
                keys[which == p].tofile(os.path.join(tmp, f"p{p}"))
            del keys, which
            for p in range(parts):
                add(np.fromfile(os.path.join(tmp, f"p{p}"), dtype=np.uint64))
    hist[0] = 0
    return [int(x) for x in hist], W


def round_half_away(x):
    return math.floor(x + 0.5) if x >= 0 else -math.floor(-x + 0.5)


def estimate(hist, W):
    """The rule of DESIGN.md §18 on hist (H bins, zero-padded) and W."""
    h = [int(x) for x in hist] + [0] * (H - len(hist))
    h[0] = h[1]                                        # the edge bin repeated, for s[1] only
    s = lambda c: h[c - 1] + h[c] + h[c + 1]           # noqa: E731
    v = next((c for c in range(1, H - 2) if s(c) < s(c + 1)), None)
    if v is None:
        raise NoPeak("no k-mer depth peak: the reads are too shallow or too noisy for a k-mer estimate")
    p = max(range(v + 1, H - 1), key=lambda c: (h[c], -c))
    if p >= H - 2:
        raise PeakAtCap(p)
    den = h[p - 1] - 2 * h[p] + h[p + 1]
    ps = float(p) if den == 0 else p + float(h[p - 1] - h[p + 1]) / (2.0 * float(den))
    errors = sum(c * h[c] for c in range(1, v))
    solid = W - errors
    return {"estimate": round_half_away(solid / ps), "valley": v, "peak": p, "peak_refined": ps, "solid": solid,
            "distinct": sum(h[1:])}
