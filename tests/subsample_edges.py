"""Generators for tests/test_subsample_edges.py: read sets whose n50 edge falls on a chosen statistics row, FASTQ with bad records in
later windows, and gzip input split into many windows.  Every generator returns the shape it claims, computed from how it was built
with plain sums, so that a test can assert the shape as well as parity with tests/subsample_oracle.py.

Subset membership depends only on n, the seed, the count and reads_per_subset (rps), and rps depends on the lengths only through their
total.  With min_read_depth = total_depth / x for x a power of two, rps is exactly n · log2(4x) / (2x) (x = 1: all n reads; x = 4: n/2;
x = 64: n/16), so the row's members are known before any length is chosen: the n50 cases put a built multiset on one row's members
and filler on the rest."""
import gzip
import os

import numpy as np

import subsample_oracle as O
from autocycler_b200 import synth

GENOME = synth.make_genome(synth.SplitMix64(0x5AB5), 40_000)
B = 1 << 16                                     # one level-1 bucket of the device n50: lengths L with the same L >> 16
NO_AT, NO_PLUS, TRUNCATED, UNEQUAL = 1, 2, 3, 4   # SubReason
REASON = {NO_AT: "expected '@' at the start of the header line", NO_PLUS: "expected '+' at the start of the separator line",
          TRUNCATED: "truncated record", UNEQUAL: "sequence and quality lengths differ"}


def reads_of(lengths, seed=1):
    """One read per length, of exactly that length, cut from GENOME (longer reads wrap around it); qualities '!'..'J'."""
    lengths = [int(L) for L in lengths]
    top = max(lengths, default=0)
    g = len(GENOME)
    text = np.resize(GENOME, top + g).tobytes()
    qual = (synth.SplitMix64(seed).u64((top + g + 7) // 8).view(np.uint8)[:top + g] % np.uint8(42) + np.uint8(33)).tobytes()
    out = []
    for i, L in enumerate(lengths):
        o = (i * 7919 + seed) % g
        out.append((f"r{i} len={L}", text[o:o + L], qual[o:o + L]))
    return out


def record_bytes(reads):
    """The LF FASTQ text of each read, as write_reads writes it."""
    return [b"@" + n.encode() + b"\n" + s + b"\n+\n" + q + b"\n" for n, s, q in reads]


# ---- rows ----------------------------------------------------------------------------------------------------------------------
def settings(bases, x):
    """(genome size, min_read_depth) with total_depth / min_read_depth == x exactly."""
    g = 1000
    return str(g), bases / g / x


def rps_of(n, x):
    k = {1: 2, 4: 4, 64: 8}[x]                  # log2(4x)
    assert (n * k) % (2 * x) == 0
    return n * k // (2 * x)


def row_members(n, seed, count, rps, row):
    """The read indices of subset `row` (0-based), or of the input when row is None."""
    if row is None:
        return list(range(n))
    order = O.shuffle_order(n, seed)
    start = O.subset_start(row, n, count)
    return [order[(start + j) % n] for j in range(rps)]


def filler(m, lo=100, span=2900):
    return [lo + (37 * j) % span for j in range(m)]


def spread(total, m, below):
    """m positive lengths, each below `below`, summing to total."""
    assert m > 0 and m <= total <= m * (below - 1), (total, m, below)
    q, r = divmod(total, m)
    return [q + 1] * r + [q] * (m - r)


def edge_lengths(k, z, c, bigs, lows=(), d=1, past=False):
    """k lengths: short reads, `lows`, c reads of length z and `bigs` (all above z), the short reads sized so that the running sum over
    the lengths up to z is exactly floor(bases / 2) (past=False) or one base short of it (past=True).  d = 1 makes bases odd."""
    g = sum(bigs)
    p = g - d - (2 if past else 0)              # the sum of the lengths up to z: exact needs g in {p, p + 1}, past needs {p + 2, p + 3}
    s = p - sum(lows) - c * z
    return spread(s, k - c - len(bigs) - len(lows), min(z, min(lows, default=z))) + list(lows) + [z] * c + list(bigs)


N50_SHAPES = {   # name -> (z, c, bigs, lows, d, past); the n50 is z, or the next length when past
    "bucket0_end": (B - 1, 2, [B] * 3, (), 1, False),
    "bucket1_end": (2 * B - 1, 1, [2 * B] * 2, (), 0, False),
    "first_of_bucket": (3 * B, 1, [200_000] * 2, (), 1, False),
    "run_end": (2 * B + 1234, 4, [2 * B + 1235, 140_000, 150_000, 400_000, 400_000], (2 * B + 5, 132_000), 1, False),
    "run_past": (2 * B + 1234, 4, [2 * B + 1235, 140_000, 150_000, 400_000, 400_000], (2 * B + 5, 132_000), 0, True),
    "bucket10": (10 * B, 1, [700_000, 720_000, 690_000], (), 1, False),
}


def plain_n50(lengths, half):
    """The smallest length present whose running sum over the lengths up to it reaches `half` (the first length when half is 0)."""
    for L in sorted(set(lengths)):
        if sum(x for x in lengths if x <= L) >= half:
            return L
    return 0


def place(n, mem, row_lengths, fill):
    """The lengths of all n reads: row_lengths on the members `mem` in order, `fill` on the others in order."""
    lengths = [None] * n
    for i, L in zip(mem, row_lengths):
        lengths[i] = L
    rest = iter(fill)
    return [next(rest) if L is None else L for L in lengths]


def n50_case(shape, n, count, seed, row, x=4, short=False):
    """-> (lengths of all n reads, settings, claim).  The row's members get the built lengths, the rest filler (of 8-39 bp when
    short)."""
    z, c, bigs, lows, d, past = N50_SHAPES[shape]
    rps = rps_of(n, x)
    mem = row_members(n, seed, count, rps, row)
    row_lengths = edge_lengths(len(mem), z, c, bigs, lows, d, past)
    lengths = place(n, mem, row_lengths, filler(n - len(mem), *((8, 32) if short else ())))
    bases = sum(row_lengths)
    half = bases // 2
    want = min(L for L in row_lengths if L > z) if past else z
    claim = {"row": row, "rps": rps, "bases": bases, "n50": want, "bucket": want >> 16, "cell": want & 0xFFFF,
             "sum_to_z": sum(L for L in row_lengths if L <= z), "half": half,
             "sum_below": sum(L for L in row_lengths if L < want), "sum_to_n50": sum(L for L in row_lengths if L <= want),
             "ceil_n50": plain_n50(row_lengths, (bases + 1) // 2)}
    return lengths, settings(sum(lengths), x), claim


def one_byte_case(path, n=30):
    """rps == n and no final newline: every sample is the input plus the newline its last record lacked.  -> (genome size, depth,
    input bytes)."""
    synth.write_reads(reads_of([100 + 17 * i for i in range(n)]), path, final_newline=False)
    data = open(path, "rb").read()
    return settings(sum(100 + 17 * i for i in range(n)), 1) + (data,)


# ---- windows -----------------------------------------------------------------------------------------------------------------
def windows_of(sizes, w):
    """The window index of each record when windows of w bytes end after their last complete record (no window doubles)."""
    out, start, end, k = [], 0, 0, 0
    for s in sizes:
        assert s <= w, "a record longer than the window"
        if end + s - start > w:
            start, k = end, k + 1
        out.append(k)
        end += s
    return out


def bad_record(rec, why):
    if why == NO_AT:
        return b"x" + rec[1:]
    if why == NO_PLUS:
        return rec.replace(b"\n+\n", b"\n-\n", 1)
    if why == UNEQUAL:
        return rec[:-2] + b"\n"
    if why == TRUNCATED:
        return rec[:rec.index(b"\n+\n") + 3]
    raise KeyError(why)


def with_bad(recs, bad):
    """recs with record j replaced by its bad form for each (j, why) in bad; a truncated record ends the file."""
    out = list(recs)
    for j, why in bad:
        out[j] = bad_record(out[j], why)
        if why == TRUNCATED:
            del out[j + 1:]
    return out


# ---- gzip across windows -------------------------------------------------------------------------------------------------------
def gz_many_windows(path, w):
    """Two gzip members whose boundary falls inside a record, CRLF line ends, no final newline and one record longer than w, with
    short records making the input about 5w.  -> (decompressed bytes, claim)."""
    short = max(40, w // 16)
    lengths = [short + (13 * i) % (short // 2 + 1) for i in range(20)] + [w * 3 // 5] + [short + (7 * i) % 31 for i in range(20)]
    tmp = path + ".plain"
    synth.write_reads(reads_of(lengths, seed=w), tmp, crlf=True, final_newline=False)
    data = open(tmp, "rb").read()
    os.remove(tmp)
    cut = len(data) * 2 // 5 + 7
    with open(path, "wb") as f:
        f.write(gzip.compress(data[:cut], compresslevel=1) + gzip.compress(data[cut:], compresslevel=1))
    long_record = 2 * (w * 3 // 5) + len(f"r20 len={w * 3 // 5}") + 10     # '@', three CRLFs and '+' CRLF
    claim = {"size": len(data), "cut_inside_line": data[cut - 1:cut] != b"\n", "long_record": long_record, "records": len(lengths)}
    return data, claim
