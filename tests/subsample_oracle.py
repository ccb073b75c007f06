"""Python restatement of `autocycler subsample` (subsample.rs, metrics.rs:25-62, misc.rs:98-127 and 197-245), the checker for the
product's sample_XX.fastq files and subsample.yaml.  Every rule below is restated from the published algorithms of the crates the
reference pins (rand 0.9.1, rand_core 0.9.3, rand_chacha 0.9.0, seq_io 0.3.2, serde_yaml 0.9); DESIGN.md §16 lists them.

- parse_genome_size: trim, lowercase, Rust's f64 grammar, round half away from zero, a saturating `as u64`, then k/m/g.
- StdRng::seed_from_u64: eight PCG32 steps give the 32-byte ChaCha12 key; the block counter starts at 0, the stream is 0, and the
  keystream's u32 words are consumed in order.
- SliceRandom::shuffle: `for i in 0..n { swap(i, chooser.next_index()) }` with IncreasingUniform, whose draws are
  `random_range(..bound)` on u32 (a widening multiply, one more word when the low half exceeds `bound.wrapping_neg()`).
- seq_io records: '@' header, sequence, '+' line (its text dropped), quality; LF or CRLF; the last record may lack its newline.  A
  blank line is refused (record N: expected '@'), as the product refuses it.
"""
import gzip
import math
import re

import numpy as np

M32 = 0xFFFFFFFF
M64 = 0xFFFFFFFFFFFFFFFF


# ---- parse_genome_size (subsample.rs:83-101) -------------------------------------------------------------------------------------
_RUST_F64 = re.compile(r"[+-]?(?:inf|infinity|nan|(?:[0-9]+\.?[0-9]*|\.[0-9]+)(?:e[+-]?[0-9]+)?)\Z")


class GenomeSizeError(ValueError):
    pass


def rust_parse_f64(s):
    """str::parse::<f64> on an already lowercased string: None when Rust refuses it."""
    if not _RUST_F64.match(s):
        return None
    return float(s)


def round_half_away(x):
    if x != x or math.isinf(x):
        return x
    f = math.floor(abs(x))
    r = f + 1 if abs(x) - f >= 0.5 else f
    return math.copysign(r, x)


def as_u64(x):
    """Rust's saturating `f64 as u64`."""
    if x != x or x <= 0:
        return 0
    if x >= 18446744073709551616.0:
        return M64
    return int(x)


def parse_genome_size(text):
    s = text.strip(" \t\n\r\x0b\x0c").lower()
    v = rust_parse_f64(s)
    if v is not None:
        return as_u64(round_half_away(v))
    mult = {"k": 1e3, "m": 1e6, "g": 1e9}.get(s[-1:])
    if mult is None:
        raise GenomeSizeError("cannot interpret genome size")
    v = rust_parse_f64(s[:-1])
    if v is None:
        raise GenomeSizeError("cannot interpret genome size")
    return as_u64(round_half_away(v * mult))


# ---- calculate_subsets (subsample.rs:120-144) ------------------------------------------------------------------------------------
class TooShallow(ValueError):
    pass


def reads_per_subset(read_count, read_bases, genome_size, min_depth):
    total_depth = read_bases / float(genome_size)
    if total_depth < min_depth:
        raise TooShallow("input reads are too shallow to subset")
    subset_depth = min_depth * math.log2(4.0 * total_depth / min_depth) / 2.0
    return as_u64(round_half_away(subset_depth / total_depth * float(read_count)))


def subset_start(i, n, count):
    return as_u64(round_half_away(float(i * n) / float(count)))


# ---- StdRng (ChaCha12) and seed_from_u64 -----------------------------------------------------------------------------------------
def pcg32_key(state):
    """rand_core 0.9 SeedableRng::seed_from_u64: the 32-byte seed as eight little-endian u32 words."""
    words = []
    for _ in range(8):
        state = (state * 6364136223846793005 + 11634580027462260723) & M64
        xorshifted = (((state >> 18) ^ state) >> 27) & M32
        rot = state >> 59
        words.append(((xorshifted >> rot) | (xorshifted << ((32 - rot) & 31))) & M32)
    return words


def chacha_blocks(key, first_block, n_blocks, rounds=12, nonce=(0, 0)):
    """n_blocks keystream blocks (16 u32 words each) from block counter first_block (64-bit, words 12-13), stream `nonce` (words 14-15),
    vectorised over the blocks."""
    ctr = np.arange(first_block, first_block + n_blocks, dtype=np.uint64)
    init = [np.full(n_blocks, c, dtype=np.uint32) for c in (0x61707865, 0x3320646E, 0x79622D32, 0x6B206574)]
    init += [np.full(n_blocks, k, dtype=np.uint32) for k in key]
    init += [(ctr & np.uint64(M32)).astype(np.uint32), (ctr >> np.uint64(32)).astype(np.uint32),
             np.full(n_blocks, nonce[0], dtype=np.uint32), np.full(n_blocks, nonce[1], dtype=np.uint32)]
    x = [w.copy() for w in init]

    def rotl(v, c):
        return (v << np.uint32(c)) | (v >> np.uint32(32 - c))

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7)

    with np.errstate(over="ignore"):
        for _ in range(rounds // 2):
            qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
            qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
        out = np.stack([x[i] + init[i] for i in range(16)], axis=1)
    return out.reshape(-1)


class StdRng:
    """rand 0.9 StdRng = ChaCha12Rng: next_u32 returns the keystream's words in order."""
    CHUNK = 4096

    def __init__(self, seed, rounds=12):
        self.key = pcg32_key(seed & M64)
        self.rounds = rounds
        self.block = 0
        self.buf = []
        self.pos = 0

    def next_u32(self):
        if self.pos == len(self.buf):
            self.buf = chacha_blocks(self.key, self.block, self.CHUNK, self.rounds).tolist()
            self.block += self.CHUNK
            self.pos = 0
        v = self.buf[self.pos]
        self.pos += 1
        return v


def random_below_u32(rng, bound):
    """rand 0.9 `random_range(..bound)` on u32 (UniformInt::sample_single_inclusive(0, bound - 1))."""
    rng_range = bound & M32
    if rng_range == 0:
        return rng.next_u32()
    m = rng.next_u32() * rng_range
    hi, lo = m >> 32, m & M32
    if lo > ((-rng_range) & M32):
        new_hi = (rng.next_u32() * rng_range) >> 32
        if lo + new_hi > M32:
            hi += 1
    return hi & M32


def calculate_bound_u32(m):
    product, current = m, m + 1
    while product * current <= M32:
        product *= current
        current += 1
    return product, current - m


def shuffle_order(n, seed):
    """(0..n).shuffle(&mut StdRng::seed_from_u64(seed)) as a list."""
    order = list(range(n))
    if n <= 1:
        return order
    rng = StdRng(seed)
    cn, chunk, remaining = 0, 0, 1        # IncreasingUniform::new(rng, 0)
    for i in range(n):
        next_n = cn + 1
        if remaining == 0:
            bound, count = calculate_bound_u32(next_n)
            chunk = random_below_u32(rng, bound)
            next_remaining = count - 1
        else:
            next_remaining = remaining - 1
        if next_remaining == 0:
            index = chunk
        else:
            index = chunk % next_n
            chunk //= next_n
        remaining, cn = next_remaining, next_n
        order[i], order[index] = order[index], order[i]
    return order


# ---- subsample_indices (subsample.rs:170-196) ------------------------------------------------------------------------------------
def subsample_indices(count, rps, order, i):
    """-> (set of read indices, the "reads a-b [and c-d]" line)."""
    n = len(order)
    start_1 = subset_start(i, n, count)
    end_1 = start_1 + rps
    out = set()
    if end_1 > n:
        end_2 = end_1 - n
        end_1 = n
        line = f"  reads {start_1 + 1}-{end_1} and 1-{end_2}"
        out.update(order[:end_2])
    else:
        line = f"  reads {start_1 + 1}-{end_1}"
    out.update(order[start_1:end_1])
    assert len(out) == rps
    return out, line


# ---- seq_io FASTQ records ------------------------------------------------------------------------------------------------------
class FastqError(ValueError):
    pass


def read_bytes(path):
    """fastq_reader (misc.rs:197-208, 233-245): gunzip (every member) when the file starts with the gzip magic."""
    data = open(path, "rb").read()
    if data[:2] == b"\x1f\x8b":
        return gzip.decompress(data)
    return data


def parse_fastq(data):
    """-> [(head, seq, qual)], or FastqError("record N: reason")."""
    lines = data.split(b"\n")
    if data.endswith(b"\n") or not data:
        lines.pop()                       # the text after the last newline is a line only when it is not empty
    recs = []
    for r in range(0, len(lines), 4):
        rec = lines[r:r + 4]
        num = r // 4 + 1
        strip = [x[:-1] if x.endswith(b"\r") else x for x in rec]
        if not rec[0].startswith(b"@"):
            raise FastqError(f"record {num}: expected '@' at the start of the header line")
        if len(rec) < 2:
            raise FastqError(f"record {num}: truncated record")
        if len(rec) < 3:
            raise FastqError(f"record {num}: truncated record")
        if not rec[2].startswith(b"+"):
            raise FastqError(f"record {num}: expected '+' at the start of the separator line")
        if len(rec) < 4:
            raise FastqError(f"record {num}: truncated record")
        if len(strip[1]) != len(strip[3]):
            raise FastqError(f"record {num}: sequence and quality lengths differ")
        recs.append((strip[0][1:], strip[1], strip[3]))
    return recs


def record_bytes(rec):
    head, seq, qual = rec
    return b"@" + head + b"\n" + seq + b"\n+\n" + qual + b"\n"


# ---- ReadSetDetails (metrics.rs:44-62) and the YAML ----------------------------------------------------------------------------
def read_set_details(lengths):
    lengths = sorted(lengths)
    bases = sum(lengths)
    target, run, n50 = bases // 2, 0, 0
    for x in lengths:
        run += x
        if run >= target:
            n50 = x
            break
    return len(lengths), bases, n50


def yaml_text(inp, outs):
    s = f"input_read_count: {inp[0]}\ninput_read_bases: {inp[1]}\ninput_read_n50: {inp[2]}\noutput_reads:\n"
    for c, b, n in outs:
        s += f"- count: {c}\n  bases: {b}\n  n50: {n}\n"
    return s


# ---- the whole command ---------------------------------------------------------------------------------------------------------
def subsample_data(data, genome_size, count=4, min_read_depth=25.0, seed=0):
    """-> {file name: bytes} for the sample files and subsample.yaml, or GenomeSizeError / FastqError / TooShallow.  Settings are
    checked by the caller (check_settings)."""
    recs = parse_fastq(data)
    n = len(recs)
    inp = read_set_details([len(r[1]) for r in recs])
    rps = reads_per_subset(n, inp[1], genome_size, min_read_depth)
    order = shuffle_order(n, seed)
    rank = [0] * n
    for p, r in enumerate(order):
        rank[r] = p
    files, outs = {}, []
    for i in range(count):
        start = subset_start(i, n, count)
        member = [((rank[r] - start) % n) < rps for r in range(n)] if n else []
        picked = [recs[r] for r in range(n) if member[r]]
        files[f"sample_{i + 1:02}.fastq"] = b"".join(record_bytes(x) for x in picked)
        outs.append(read_set_details([len(x[1]) for x in picked]))
    files["subsample.yaml"] = yaml_text(inp, outs).encode()
    return files


def subsample(reads, genome_size_str, count=4, min_read_depth=25.0, seed=0):
    return subsample_data(read_bytes(reads), parse_genome_size(genome_size_str), count, min_read_depth, seed)
