"""Shared input generators for the parity tests (oracle vs CUDA path, and oracle vs the host-emulated
device logic).  Every case is a list of files: [(filename, [(header, sequence)])]."""
import random


def rc(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def rand_seq(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def mutate(rng, s, rate):
    out = []
    for c in s:
        r = rng.random()
        if r < rate / 3:
            continue
        if r < 2 * rate / 3:
            out.append(rng.choice("ACGT"))
            out.append(c)
        elif r < rate:
            out.append(rng.choice([b for b in "ACGT" if b != c]))
        else:
            out.append(c)
    return "".join(out)


def random_case(seed, k):
    """Adversarial little genomes: rotations, strand flips, shared ends, inverted and tandem repeats,
    homopolymers, low-complexity alphabets, multi-contig files, linear contigs whose ends match nothing."""
    rng = random.Random(seed)
    style = rng.randrange(8)
    n_files = rng.randint(1, 5)
    base_len = rng.randint(k + 1, max(k + 2, rng.choice([30, 60, 150, 400])))
    alphabet = "ACGT" if style != 5 else rng.choice(["AC", "AT", "ACG"])
    genome = rand_seq(rng, base_len, alphabet)
    if style == 1:   # inverted repeat
        unit = rand_seq(rng, rng.randint(k, 2 * k), alphabet)
        genome = genome[:len(genome) // 2] + unit + rand_seq(rng, rng.randint(0, 5)) + rc(unit) + genome[len(genome) // 2:]
    if style == 2:   # tandem repeat
        unit = rand_seq(rng, rng.randint(1, k), alphabet)
        genome = genome[:len(genome) // 3] + unit * rng.randint(2, 3 + (2 * k) // len(unit)) + genome[len(genome) // 3:]
    if style == 3:   # homopolymers
        genome = genome[:len(genome) // 2] + rng.choice("ACGT") * rng.randint(k - 1, 2 * k + 3) + genome[len(genome) // 2:]
    if style == 4:   # dispersed repeat
        unit = rand_seq(rng, rng.randint(k, 3 * k), alphabet)
        genome = unit + genome[:len(genome) // 2] + unit + genome[len(genome) // 2:] + (rc(unit) if rng.random() < 0.5 else unit)
    files = []
    for f in range(n_files):
        recs = []
        n_contigs = 1 if rng.random() < 0.7 else rng.randint(2, 3)
        for c in range(n_contigs):
            s = genome
            if rng.random() < 0.7:
                r = rng.randrange(len(s))
                s = s[r:] + s[:r]
            if rng.random() < 0.5:
                s = rc(s)
            if rng.random() < 0.8:
                s = mutate(rng, s, rng.choice([0.0, 0.01, 0.05]))
            if rng.random() < 0.3:
                s = s + s[:rng.randint(1, min(len(s), 3 * k))]          # circular overlap
            if rng.random() < 0.3 and len(s) > 2 * k + 4:
                a = rng.randrange(len(s) - k - 1)
                s = s[a:a + rng.randint(k, len(s) - a)]                  # linear fragment
            if style == 6 and rng.random() < 0.5:
                s = rand_seq(rng, rng.randint(k, 3 * k))                # unrelated contig: its ends stay dotted
            if style == 7:
                s = s[:k + rng.randint(0, 3)]                           # contigs barely longer than k
            if len(s) < k:
                s = s + rand_seq(rng, k - len(s))
            recs.append((f"c{c + 1} len={len(s)}", s))
        files.append((f"asm_{f:02d}.fasta", recs))
    return files


def _walk_steps(sampled_set):
    """For every 6-mer (2 bits a base, first base most significant): the bases that extend it to an unsampled 7-mer whose own last six
    bases can be extended the same way.  Iterated until no step leads to a dead end."""
    ok = {c6: [b for b in range(4) if ((c6 << 2) | b) not in sampled_set] for c6 in range(1 << 12)}
    while True:
        dead = {c6 for c6, bs in ok.items() if not bs}
        if not dead:
            return ok
        ok = {c6: [b for b in bs if (((c6 << 2) | b) & 0xFFF) not in dead] for c6, bs in ok.items()}


_STEPS = None


def sampled_walk(rng, n, rate=0.0):
    """n bases of a random walk over 7-mers that avoids the 7-mers the table's sizing pass samples (tests/table_sizing.py), except that at
    about `rate` of its steps it writes out a whole sampled 7-mer (the 7-mers across that seam are whatever they happen to be).  The sampled
    set is closed under reverse complement, so at rate 0 neither strand holds a sampled 7-mer: every k-mer's centre is unsampled and the
    size estimate sees nothing of this sequence."""
    global _STEPS
    import table_sizing
    if _STEPS is None:
        _STEPS = _walk_steps(table_sizing.SAMPLED_SET)
    ok = _STEPS
    jumps = [c7 for c7 in sorted(table_sizing.SAMPLED_SET) if ok[c7 & 0xFFF]]
    c6 = rng.choice([c for c, bs in ok.items() if bs])
    out = [(c6 >> (2 * (5 - i))) & 3 for i in range(6)]
    while len(out) < n:
        if rate and rng.random() < rate:
            c7 = rng.choice(jumps)
            out += [(c7 >> (2 * (6 - i))) & 3 for i in range(7)]
            c6 = c7 & 0xFFF
            continue
        b = rng.choice(ok[c6])
        out.append(b)
        c6 = ((c6 << 2) | b) & 0xFFF
    return "".join("ACGT"[b] for b in out[:n])


def homopolymer_case(rng, occurrences, k, base="A", flank=300):
    """One contig holding a run of `base` whose k-mer occurs `occurrences` times (a run of occurrences + k - 1 bases) between random
    flanks (T: the occurrences land on the reverse strand of the canonical all-A k-mer)."""
    stop = "G" if base in "AT" else "A"           # the flanks must not lengthen the run
    a = rand_seq(rng, flank) + stop + base * (occurrences + k - 1) + stop + rand_seq(rng, flank)
    return [("a.fasta", [("c1", a)])]


def write_case(files, directory):
    import os
    os.makedirs(directory, exist_ok=True)
    for fn, recs in files:
        with open(os.path.join(directory, fn), "w") as f:
            for header, seq in recs:
                f.write(f">{header}\n{seq}\n")
