"""Generators for tests/test_spectrum_edges.py: read sets whose k-mer counts are built exactly from the reads rather than from coverage, a
short-read set that packs many reads into each warp's words, an assembly of thousands of short contigs, and repeats whose copies carry
the alleles of chosen polish candidates.  Each generator is seeded (synth.SplitMix64) and returns its input together with the exact
shape it claims to reach, so that a test can assert the shape as well as the parity.

Counts from reads: a homopolymer read of c + k - 1 bases gives the key A^k exactly c windows; a tandem array of an aperiodic unit U
(period p) cut to p c + k - 1 + j bases gives each of its p rotation keys c windows, and the first j rotations one more."""
import numpy as np

import depth_oracle as D
import genome_size_oracle as G
import polish_oracle as P
from autocycler_b200 import synth

H = G.H


def keys_of(seq, k):
    """The canonical keys of a sequence's windows, in order."""
    return G.canonical_keys(G._CODE[np.frombuffer(seq.encode() + b"\x00", dtype=np.uint8)], k)


def genome(seed, n):
    return synth.make_genome(synth.SplitMix64(seed), n, repeats=False).tobytes().decode()


def noisy(seq, depth, seed, n50=2000, err=0.01):
    g = np.frombuffer(seq.encode(), dtype=np.uint8)
    return list(synth.make_noisy_reads(g, depth=depth, n50=n50, seed=seed, sub=err / 2, ins=err / 4, dele=err / 4))


def read(name, seq):
    return (name, seq.encode(), b"I" * len(seq))


def write_fasta(path, records):
    with open(path, "w") as f:
        for header, seq in records:
            f.write(f">{header}\n{seq}\n")


def unit(seed, p, k, avoid):
    """An aperiodic unit of period p whose p rotation keys are distinct canonical keys, none of them in `avoid`."""
    for s in range(seed, seed + 100):
        u = genome(s, p)
        rot = rotation_keys(u, k)
        if len(set(rot.tolist())) == p and not np.isin(rot, avoid).any():
            return u
    raise AssertionError("no aperiodic unit")


def rotation_keys(u, k):
    """Key i: the window of the tandem array of u that starts at rotation i."""
    return keys_of((u * (k // len(u) + 2))[:len(u) + k - 1], k)


def tandem(u, c, k, extra=0):
    """p c + k - 1 + extra bases of u repeated: rotations 0 .. extra-1 get c + 1 windows, the others c."""
    n = len(u) * c + k - 1 + extra
    return (u * (n // len(u) + 1))[:n]


# ---- A. exact high counts -------------------------------------------------------------------------------------------------------------
class Counts:
    """The planted keys and their exact counts, and what every other read adds: nothing to these keys (asserted)."""

    def __init__(self, k):
        self.k, self.reads, self.keys = k, [], {}

    def add(self, name, seq, times=1):
        for i in range(times):
            self.reads.append(read(f"{name}_{i}" if times > 1 else name, seq))
        uk, uc = np.unique(keys_of(seq, self.k), return_counts=True)
        for key, c in zip(uk.tolist(), uc.tolist()):
            self.keys[key] = self.keys.get(key, 0) + c * times

    def add_periodic(self, name, seq, p):
        """The same as add for a sequence of period p, counted from its first p windows: far less memory for a read of 2^25 bases."""
        self.reads.append(read(name, seq))
        w = len(seq) - self.k + 1
        for i, key in enumerate(keys_of(seq[:p + self.k - 1], self.k).tolist()):
            self.keys[key] = self.keys.get(key, 0) + (w - i + p - 1) // p

    def tandem(self, name, u, c, extra=0):
        self.add(name, tandem(u, c, self.k, extra))
        rot = rotation_keys(u, self.k).tolist()
        assert [self.keys[x] for x in rot] == [c + 1] * extra + [c] * (len(u) - extra), name

    def histogram_claim(self):
        """{bin: keys} of the planted keys (the last bin holds every count >= H - 1)."""
        out = {}
        for c in self.keys.values():
            out[min(c, H - 1)] = out.get(min(c, H - 1), 0) + 1
        return out


def background(k, seed, n=20_000, depth=30):
    """An ordinary genome at 30x with 1% errors, so that the valley and peak rules still hold."""
    g = genome(seed, n)
    return g, noisy(g, depth, seed + 1)


def read_keys(reads, k):
    seqs = [r[1] for r in reads]
    return G.canonical_keys(G._CODE[np.frombuffer(b"\x00".join(seqs) + b"\x00", dtype=np.uint8)], k)


def _disjoint(planted, background_keys):
    """No background read window has a planted key, so the planted counts are exact."""
    assert not np.isin(background_keys, np.array(sorted(planted), dtype=np.uint64)).any(), "a background window has a planted key"


def high_counts(k, seed=0x5E01):
    """Reads for genome_size, qv and unassembled: keys counted exactly 255 and 256 (U1), 16,382 and 16,383 (U3), 65,535 and 65,536 (U2),
    a homopolymer key 20,000 times and a dinucleotide's two keys 30,000 times each, mixed into a 30x genome.
    -> (background genome, reads, Counts, units)."""
    g, bg = background(k, seed)
    bk = read_keys(bg, k)
    cnt = Counts(k)
    u1, u2, u3 = unit(seed + 10, 16, k, bk), unit(seed + 200, 16, k, bk), unit(seed + 400, 16, k, bk)
    cnt.tandem("u1", u1, 255, 8)
    cnt.tandem("u3", u3, 16_382, 8)
    cnt.tandem("u2", u2, 65_535, 8)
    cnt.add_periodic("homo", "A" * (20_000 + k - 1), 1)
    cnt.add("di", ("AC" * 40_000)[:2 * 30_000 + k - 1])
    rot = [rotation_keys(u, k).tolist() for u in (u1, u2, u3)]
    assert len(set(sum(rot, []))) == 48
    di = keys_of("AC" * k, k).tolist()
    assert cnt.keys[di[0]] == cnt.keys[di[1]] == 30_000 and cnt.keys[keys_of("A" * k, k)[0]] == 20_000
    _disjoint(cnt.keys, bk)
    reads = bg[:len(bg) // 2] + cnt.reads + bg[len(bg) // 2:]
    return g, reads, cnt, (u1, u2, u3)


def depth_digits(k=11, seed=0x5E02):
    """Depth's contigs at each radix digit boundary, with the median each must get:
      d8:   8 keys at 255 and 8 at 256 -> 255.5          d16: 8 keys at 65,535 and 8 at 65,536 -> 65,535.5
      d24:  the two keys of (AC)^n at 2^24 - 1 and 2^24 -> 16,777,215.5
      dall: 11 keys at 1, 300 (x4), 70,000, 70,001 (x4) and 2^24 + 5 -> 70,000, decided by the upper digits
    and the background genome as a contig of its own.  -> (contigs [(header, seq)], reads, {name: median})."""
    assert k == 11                                    # the (AC)^n contig holds exactly its two keys
    g, bg = background(k, seed)
    bk = read_keys(bg, k)
    cnt = Counts(k)
    u1, u2 = unit(seed + 10, 16, k, bk), unit(seed + 200, 16, k, bk)
    cnt.tandem("u1", u1, 255, 8)
    cnt.tandem("u2", u2, 65_535, 8)
    cnt.add_periodic("ac", "AC" * (2 ** 24) + "ACACACACA", 2)  # 2^25 + 9 bases: 2^24 windows start with A, 2^24 - 1 with C
    allc = "A" * 11 + "C" * 10                          # key i: A^(11-i) C^i
    cnt.add("all_full", allc)
    cnt.add("all_10", allc[:20], 299)
    cnt.add("all_6", allc[:16], 69_700)
    cnt.add("all_5", allc[:15])
    a = 2 ** 24 + 5 - 70_001
    cnt.add_periodic("all_a", "A" * (a + 10), 1)
    want_all = [2 ** 24 + 5] + [70_001] * 4 + [70_000] + [300] * 4 + [1]
    assert [cnt.keys[x] for x in keys_of(allc, k).tolist()] == want_all
    ac = keys_of("ACACACACACAC", k).tolist()
    assert sorted(cnt.keys[x] for x in ac) == [2 ** 24 - 1, 2 ** 24]
    contigs = [("bg circular=true", g), ("d8", (u1 * 3)[:16 + k - 1]), ("d16", (u2 * 3)[:16 + k - 1]), ("d24", "ACACACACACAC"),
               ("dall", allc)]
    every, n = np.unique(np.concatenate([D.contig_keys(s, h, k) for h, s in contigs]), return_counts=True)
    planted = np.concatenate([D.contig_keys(s, h, k) for h, s in contigs[1:]])
    assert (n[np.searchsorted(every, planted)] == 1).all(), "a planted contig key is not unique in the assembly"
    _disjoint(cnt.keys, bk)
    reads = bg[:len(bg) // 2] + cnt.reads + bg[len(bg) // 2:]
    return contigs, reads, {"d8": 255.5, "d16": 65_535.5, "d24": 16_777_215.5, "dall": 70_000.0}


# ---- B. many addresses per warp -------------------------------------------------------------------------------------------------------
def short_reads(k, seed=0x5E03, n_short=8_000):
    """A 40 kbp genome of which the assembly holds the first half; long reads at 25x interleaved with n_short error-free reads of
    0 - 400 bp, lengths at 0, k - 1, k and 32 m - 1, 32 m, 32 m + 1 among them.  -> (genome, held part, reads, short read names)."""
    g = genome(seed, 40_000)
    rng = synth.SplitMix64(seed + 1)
    edge = [0, k - 1, k] + [32 * m + d for m in range(1, 13) for d in (-1, 0, 1)]
    lens = rng.u64(n_short) % np.uint64(401)
    starts = rng.u64(n_short) % np.uint64(len(g) - 400)
    short = []
    for i in range(n_short):
        n = edge[i % len(edge)] if i % 3 == 0 else int(lens[i])
        a = int(starts[i])
        short.append(read(f"s{i}", g[a:a + n]))
    long = noisy(g, 25, seed + 2, n50=3000)
    reads, j = [], 0
    for i, r in enumerate(short):                       # a long read after every few short ones
        reads.append(r)
        if i % (n_short // len(long) + 1) == 0 and j < len(long):
            reads.append(long[j])
            j += 1
    reads += long[j:]
    return g, g[:20_000], reads, {r[0].decode() if isinstance(r[0], bytes) else r[0] for r in short}


def many_contigs(k, seed=0x5E04, n=3_000):
    """n contigs of k - 300 bp and one of 200 kbp, cut from one genome, with reads at 15x over all of it.  -> (contigs, reads)."""
    rng = synth.SplitMix64(seed)
    lens = [k + int(x) for x in rng.u64(n) % np.uint64(301 - k)]
    g = genome(seed + 1, 200_000 + sum(lens))
    contigs, at = [("big circular=true", g[:200_000])], 200_000
    for i, n_ in enumerate(lens):
        contigs.append((f"c{i}", g[at:at + n_]))
        at += n_
    return contigs, noisy(g, 15, seed + 2, n50=2500)


# ---- C. polish ties --------------------------------------------------------------------------------------------------------------------
def apply_edit(s, p0, mid, skip):
    return s[:p0] + mid + s[p0 + skip:]


def tie_case(L, alleles, seed, deep=None, k=21):
    """A circular 4 kbp genome with a 200 bp repeat in len(alleles) copies; copy i carries candidate alleles[i] applied at the repeat's
    base 100, and the assembly's first copy carries the repeat unedited there.  Error-free reads of 120 bp start at every base; with
    deep = i they start twice at every base around copy i, so its allele scores twice the others'.  The repeat's base 100 (the round's
    base at p0) is chosen so that every allele changes the window that ends there.  -> (assembly seq, reads, p0, candidate list)."""
    rep = list(genome(seed + 1, 200))
    cur = next(b for b in "ACGT" if all(P.candidates(b, L)[c][0][:1] != b for c in alleles if P.candidates(b, L)[c][1] == 0))
    rep[100] = cur                                     # a base that no inserted allele starts with
    cands = P.candidates(cur, L)
    for c in alleles:
        mid, skip = cands[c]
        if mid == "" and rep[100 + skip] == cur:       # a deletion of d bases must not leave base 100 unchanged
            rep[100 + skip] = "ACGT"[("ACGT".index(cur) + 1) % 4]
    rep = "".join(rep)
    starts = [500 + 1200 * i for i in range(len(alleles))]
    edited = [apply_edit(rep, 100, *cands[c]) for c in alleles]
    truth, asm, at = [], [], 0
    gs = genome(seed, 4_000)
    for i, s in enumerate(starts):
        truth += [gs[at:s], edited[i]]
        asm += [gs[at:s], rep if i == 0 else edited[i]]
        at = s + 200
    truth, asm = "".join(truth + [gs[at:]]), "".join(asm + [gs[at:]])
    doubled = truth + truth
    reads = [(f"r{i}", doubled[i:i + 120].encode(), b"I" * 120) for i in range(len(truth))]
    if deep is not None:
        shift = sum(len(e) - 200 for e in edited[:deep])
        lo = starts[deep] + shift - 150
        reads += [(f"d{i}", doubled[i:i + 120].encode(), b"I" * 120) for i in range(lo, lo + 200 + 300)]
    return asm, reads, starts[0] + 100, cands
