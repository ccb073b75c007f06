"""Exact restatement of how the k-mer table is sized (pipeline.cu local_w: SampleBody, the size estimate, the retry at the safe size),
from the oracle's padded, end-repaired strands.  UnitigGraph.timings().table_capacity is a deterministic function of what the sizing
pass counts, so comparing it with predict_capacity() checks SampleBody<W> and the sample table's upsert exactly."""
import math

import numpy as np

PROBE_LIMIT_LOAD = (0.9, 1.0)      # between these loads a probe chain may or may not pass the 2048-group limit: the route is not certain
_COMP = str.maketrans("ACGT", "TGCA")
_CODE = np.zeros(256, dtype=np.uint32)
for _i, _c in enumerate(b"ACGT"):
    _CODE[_c] = _i


def sampled(c7):
    """SampleBody::sampled: c7 = the 7 bases around the centre, 2 bits each (A=0 C=1 G=2 T=3), first base most significant."""
    if (c7 >> 6) & 2:                  # centre base G or T: the other strand
        r = 0
        for b in range(7):
            r |= ((c7 >> (2 * b)) & 3) << (2 * (6 - b))
        c7 = ~r & 0x3FFF
    return ((c7 * 0x9E3779B1) & 0xFFFFFFFF) >> 26 == 0


SAMPLED = np.array([sampled(c) for c in range(1 << 14)], dtype=bool)
SAMPLED_SET = frozenset(int(c) for c in np.nonzero(SAMPLED)[0])


def heptamer_codes(seq):
    """-> int array: the 7-mer starting at every position of `seq` (len(seq) - 6 entries)."""
    x = _CODE[np.frombuffer(seq.encode(), dtype=np.uint8)]
    n = len(x) - 6
    if n <= 0:
        return np.zeros(0, dtype=np.uint32)
    c = np.zeros(n, dtype=np.uint32)
    for b in range(7):
        c = (c << 2) | x[b:b + n]
    return c


def canonical(w):
    r = w[::-1].translate(_COMP)
    return min(w, r)


def sampled_distinct(padded, k):
    """The count SampleBody leaves in counters[0]: distinct canonical k-mers among the dot-free windows whose centre 7-mer is sampled."""
    h = k // 2
    seen = set()
    for s in padded:
        n_win = len(s) - (k - 1)
        dots = np.frombuffer(s.encode(), dtype=np.uint8) == ord(".")
        cdots = np.concatenate([[0], np.cumsum(dots)])
        starts = np.arange(n_win)
        clean = cdots[starts + k] == cdots[starts]
        hept = heptamer_codes(s)
        centre = starts + h - 3
        ok = clean & SAMPLED[hept[centre]]
        for i in np.nonzero(ok)[0]:
            seen.add(canonical(s[i:i + k]))
    return len(seen)


def distinct_canonical(padded, k):
    """Every distinct canonical k-mer, dotted ones included (they take slots, though the sizing pass skips them)."""
    return len({canonical(s[i:i + k]) for s in padded for i in range(len(s) - k + 1)})


def predict(padded, k, n_distinct=None, load=0.5):
    """-> dict(capacity, safe, estimate_cap, sampled, distinct, retry).  `padded`: the oracle's padded forward strands (oracle_lib.load_sequences);
    `n_distinct`: distinct canonical k-mers if known (the oracle's n_kmers / 2), else counted here; `load`: the table load the estimate is
    sized for (AC_TABLE_LOAD).  Raises when the input's load on the estimated table lies in the band where the route is not certain."""
    n = sum(len(s) - (k - 1) for s in padded)
    safe = (n + n // 2 + 64 + 3) & ~3
    distinct = distinct_canonical(padded, k) if n_distinct is None else n_distinct
    out = dict(safe=safe, distinct=distinct, sampled=None, estimate_cap=None, retry=False, capacity=safe)
    if n <= 65536 or k < 7:
        return out
    s = sampled_distinct(padded, k)
    out["sampled"] = s
    sample_cap = (n // 64 * 4 + 4096) & ~3
    if s > sample_cap:
        return out
    if PROBE_LIMIT_LOAD[0] * sample_cap <= s:
        raise ValueError(f"sample table load {s / sample_cap:.3f}: whether the sizing pass overflows is not certain")
    est = (s + 3 * math.isqrt(s) + 16) * 64 + len(padded) * 2 * k
    cap = min(safe, (int(est / load) + 4096 + 3) & ~3)             # (uint64_t)((double)est / load): est < 2^53, so est / 0.5 == 2 * est
    out["estimate_cap"] = cap
    if distinct > cap:
        out["retry"] = cap != safe
        return out
    if cap != safe and PROBE_LIMIT_LOAD[0] * cap <= distinct:
        raise ValueError(f"table load {distinct / cap:.3f}: whether the insert passes the probe limit is not certain")
    out["capacity"] = cap
    return out
