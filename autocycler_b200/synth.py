"""Deterministic synthetic input assemblies for the BASELINE.json configs (SURVEY.md §8d).

There are no real genomes offline, so every config is a size-matched synthetic: an iid ACGT
"genome" with injected repeat families, from which each "assembly" is derived by a random rotation,
an optional strand flip, per-base substitutions / insertions / deletions, an optional circular end
overlap and an optional split into 2-3 contigs.  All randomness comes from splitmix64 seeded with
0xA07C0C1E00 + config index, so the same inputs are regenerated bit-for-bit anywhere.
"""
import os

import numpy as np

SEED_BASE = 0xA07C0C1E00
_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_COMP = np.zeros(256, dtype=np.uint8)
for _a, _b in zip(b"ACGT", b"TGCA"):
    _COMP[_a] = _b


class SplitMix64:
    """Vectorised splitmix64: stream element i is mix(seed + (i+1)*GAMMA)."""
    GAMMA = np.uint64(0x9E3779B97F4A7C15)

    def __init__(self, seed):
        self.state = np.uint64(seed & 0xFFFFFFFFFFFFFFFF)

    def u64(self, n):
        with np.errstate(over="ignore"):
            idx = np.arange(1, n + 1, dtype=np.uint64)
            z = self.state + idx * self.GAMMA
            self.state = self.state + np.uint64(n) * self.GAMMA
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            return z ^ (z >> np.uint64(31))

    def uniform(self, n):
        return (self.u64(n) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))

    def below(self, bound):
        return int(self.u64(1)[0] % np.uint64(bound))

    def bases(self, n):
        return _ACGT[(self.u64(n) >> np.uint64(62)).astype(np.intp)]


def revcomp(a):
    return _COMP[a[::-1]]


def make_genome(rng, length, repeats=True):
    g = rng.bases(length)
    if repeats and length >= 200_000:
        for copies, rlen in ((7, 5000), (10, 1300)):
            unit = rng.bases(rlen)
            for _ in range(copies):
                at = rng.below(length - rlen)
                g[at:at + rlen] = unit if rng.below(2) else revcomp(unit)
    return g


def mutate(rng, seq, sub=5e-4, ins=2.5e-4, dele=2.5e-4):
    n = len(seq)
    u = rng.uniform(n)
    out = seq.copy()
    is_sub = u < sub
    nsub = int(is_sub.sum())
    if nsub:
        # a different base: rotate by 1..3 in ACGT code space
        code = np.searchsorted(_ACGT, out[is_sub])
        shift = (rng.u64(nsub) % np.uint64(3)).astype(np.intp) + 1
        out[is_sub] = _ACGT[(code + shift) % 4]
    is_del = (u >= sub) & (u < sub + dele)
    is_ins = (u >= sub + dele) & (u < sub + dele + ins)
    nins = int(is_ins.sum())
    if nins:
        out = np.insert(out, np.nonzero(is_ins)[0] + 1, rng.bases(nins))
        keep = np.insert(~is_del, np.nonzero(is_ins)[0] + 1, True)
    else:
        keep = ~is_del
    return out[keep]


def derive_assembly(rng, replicons, sub, ins, dele, p_overlap=0.25, p_split=0.10):
    """-> list of contig byte arrays for one assembly."""
    contigs = []
    for ri, rep in enumerate(replicons):
        n = len(rep)
        rot = rng.below(n)
        s = np.concatenate([rep[rot:], rep[:rot]])
        if rng.below(2):
            s = revcomp(s)
        s = mutate(rng, s, sub, ins, dele)
        if rng.uniform(1)[0] < p_overlap and len(s) > 20_000:
            ov = 50 + rng.below(4951)
            s = np.concatenate([s, s[:ov]])
        if ri == 0 and rng.uniform(1)[0] < p_split and len(s) > 50_000:
            pieces = 2 + rng.below(2)
            cuts = sorted(10_000 + rng.below(len(s) - 20_000) for _ in range(pieces - 1))
            prev = 0
            for c in cuts + [len(s)]:
                if c - prev > 0:
                    contigs.append(s[prev:c])
                prev = c
        else:
            contigs.append(s)
    return contigs


CONFIGS = {
    # name: (config index, replicon lengths, number of assemblies)
    "cfg1": (1, [100_000], 3),
    "cfg2": (2, [4_641_652], 8),
    "cfg3": (3, [5_500_000, 220_000, 110_000, 80_000, 5_000, 3_000], 12),
    "cfg4": (4, [10_000_000], 24),
    "cfg5": (5, [5_000_000], 64),
}


def make_assemblies(config="cfg1", n_assemblies=None, replicon_lengths=None, seed=None,
                    sub=5e-4, ins=2.5e-4, dele=2.5e-4, first=0):
    """-> [(filename, [(header, uint8 array)])], sorted file order == generation order.

    `first` skips the first assemblies without changing the later ones (every assembly has its own
    splitmix64 stream), so a rank can generate only its shard."""
    if config in CONFIGS:
        idx, lens, count = CONFIGS[config]
    else:
        idx, lens, count = 0, [20_000], 4
    lens = replicon_lengths or lens
    count = n_assemblies or count
    seed = SEED_BASE + idx if seed is None else seed
    grng = SplitMix64(seed)
    replicons = [make_genome(grng, L) for L in lens]
    out = []
    for a in range(first, count):
        arng = SplitMix64((seed * 1_000_003 + 7919 * (a + 1)) & 0xFFFFFFFFFFFFFFFF)
        contigs = derive_assembly(arng, replicons, sub, ins, dele)
        recs = [(f"contig_{i + 1} length={len(c)} circular=true", c) for i, c in enumerate(contigs)]
        out.append((f"asm_{a:02d}.fasta", recs))
    return out


def write_assemblies(assemblies, directory, width=0):
    os.makedirs(directory, exist_ok=True)
    for fn, recs in assemblies:
        with open(os.path.join(directory, fn), "wb") as f:
            for header, seq in recs:
                f.write(b">" + header.encode() + b"\n")
                f.write(seq.tobytes())
                f.write(b"\n")


def total_bases(assemblies):
    return sum(len(s) for _, recs in assemblies for _, s in recs)


def make_reads(genome, depth=None, n_reads=None, n50=15_000, sigma=0.5, seed=1, length=None, min_length=0, max_length=None):
    """Seeded long reads cut from a circular genome (make_genome): log-normal lengths whose length-weighted median (the usual N50) is
    about n50, or all of one `length`; either strand; random qualities '!'..'J'.  Stops at `n_reads` reads or at depth x the genome's
    length in bases.  Yields (name, sequence bytes, quality bytes)."""
    rng = SplitMix64(seed)
    glen = len(genome)
    mu = np.log(n50) - sigma * sigma
    target = None if depth is None else int(depth * glen)
    made, bases = 0, 0
    while (n_reads is None or made < n_reads) and (target is None or bases < target):
        if length is not None:
            L = length
        else:
            u1, u2 = rng.uniform(2)
            z = np.sqrt(-2.0 * np.log(max(u1, 1e-300))) * np.cos(2.0 * np.pi * u2)
            L = max(min_length, int(np.exp(mu + sigma * z)))
            if max_length is not None:
                L = min(L, max_length)
        start = rng.below(glen)
        idx = (np.arange(start, start + L) % glen) if start + L > glen else slice(start, start + L)
        seq = genome[idx]
        if rng.below(2):
            seq = revcomp(seq)
        qual = (rng.u64((L + 7) // 8).view(np.uint8)[:L] % np.uint8(42)) + np.uint8(33)
        made += 1
        bases += L
        yield (f"read_{made} length={L}", seq.tobytes(), qual.tobytes())


def make_noisy_reads(genome, depth=None, n_reads=None, n50=15_000, sigma=0.5, seed=1, sub=0.0, ins=0.0, dele=0.0, min_length=0):
    """make_reads' reads (the same seed gives the same positions, strands and lengths before the errors), each then given per-base
    substitutions, insertions and deletions at the given rates from a second seeded stream, with fresh qualities of its new length.
    Stops on make_reads' own rule (depth counts the error-free lengths).  Yields (name, sequence bytes, quality bytes)."""
    rng = SplitMix64(seed ^ 0x6E6F697379)
    for name, seq, _ in make_reads(genome, depth=depth, n_reads=n_reads, n50=n50, sigma=sigma, seed=seed, min_length=min_length):
        out = mutate(rng, np.frombuffer(seq, dtype=np.uint8), sub, ins, dele) if seq else np.zeros(0, dtype=np.uint8)
        qual = (rng.u64((len(out) + 7) // 8).view(np.uint8)[:len(out)] % np.uint8(42)) + np.uint8(33)
        yield (name, out.tobytes(), qual.tobytes())


def write_reads(reads, path, gz=False, crlf=False, plus_header=False, final_newline=True):
    """reads as FASTQ at path (gzipped when gz): CRLF line ends, '+' lines that repeat the header and a last record without its
    newline on request."""
    import gzip
    eol = b"\r\n" if crlf else b"\n"
    out = gzip.open(path, "wb", compresslevel=1) if gz else open(path, "wb")
    with out as f:
        pending = None
        for name, seq, qual in reads:
            if pending is not None:
                f.write(pending + eol)
            head = name.encode() if isinstance(name, str) else name
            f.write(b"@" + head + eol + seq + eol + b"+" + (head if plus_header else b"") + eol)
            pending = qual
        if pending is not None:
            f.write(pending + (eol if final_newline else b""))
