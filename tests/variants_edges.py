"""Generators for tests/test_variants_edges.py: assemblies and read sets for `autocycler variants` (DESIGN.md §23) whose every k-mer
count is known from the construction, with the exact rows (POS, REF, ALT, AK, RK, PK) each case must give.

Counts from tiled reads: a circular sequence of n bases, read as n reads of R bases that start at every one of its bases (the reads run
round the sequence as often as R needs), gives each of its n circular windows exactly R - k + 1 read windows.  A case tiles its truth
contigs c1 times and copies carrying planted events c2 times, so a k-mer's count is (R - k + 1) times the number of copies that hold it.
The expected AK, RK and PK of a planted event are read off those counts with plain string operations: AK the least count over the
edited sequence's k + s windows from a = p - k + 1, RK the least over the truth's windows a .. p + d, PK the edited windows (an indel's
last one left out) that are windows of the assembly.  POS, REF and ALT are given by each generator from where it planted the event.
Each generator is seeded (synth.SplitMix64) and also returns the shape it claims to reach, for the test to assert."""
import polish_oracle as P
from autocycler_b200 import synth

BASES = "ACGT"
COMP = str.maketrans("ACGT", "TGCA")


def canon(w):
    """The canonical form of a window: the smaller of it and its reverse complement (2-bit codes order like the letters)."""
    rc = w.translate(COMP)[::-1]
    return w if w <= rc else rc


def key_int(w):
    """The 2-bit packed key of a canonical window, first base in the top bits."""
    x = 0
    for b in w:
        x = (x << 2) | BASES.index(b)
    return x


M64 = (1 << 64) - 1


def gs_mix(x):
    """The spectrum's key hash (the murmur3 64-bit finaliser of gs_kmers.h)."""
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    return x ^ (x >> 33)


def partition(w, parts):
    """The spectrum partition that holds window w's key: the high word of hash x parts."""
    return (gs_mix(key_int(canon(w))) * parts) >> 64


def windows(seq, k, circular):
    ext = seq + seq[:k - 1] if circular else seq
    return [ext[i:i + k] for i in range(len(ext) - k + 1)]


def genome(seed, n):
    return synth.make_genome(synth.SplitMix64(seed), n, repeats=False).tobytes().decode()


def other(b, i=1):
    return BASES[(BASES.index(b) + i) % 4]


def apply(seq, p, mid, skip):
    """seq with the bases [p, p + skip) replaced by mid; a deletion past the end (circular) also removes the bases it wraps onto."""
    n = len(seq)
    if p + skip > n:
        return seq[p + skip - n:p] + mid
    return seq[:p] + mid + seq[p + skip:]


class Case:
    """One assembly, its tiled reads, and the rows it must give.  k, L: --kmer and --max_indel; R: read length."""

    def __init__(self, k, L, R=150, min_count=2, min_fraction=0.1):
        self.k, self.L, self.R = k, L, R
        self.kw = dict(min_count=min_count, max_indel=L, min_fraction=min_fraction)
        self.contigs = []                                    # (name, header, truth seq, circular)
        self.reads = []
        self.count = {}                                      # canonical window -> exact read windows
        self.events = []                                     # planted events that must give a row
        self.shape = {}

    # ---- construction -----------------------------------------------------------------------------------------------------------------
    def tile(self, name, seq, times, R=None):
        """times copies of the n reads of R bases that start at every base of circular seq."""
        R = R or self.R
        n = len(seq)
        wrap = seq * ((R + n - 1) // n + 1)
        for i in range(n):
            r = wrap[i:i + R].encode()
            for t in range(times):
                self.reads.append((f"{name}_{i}_{t}", r, b"I" * R))
        for w in windows(seq, self.k, True):
            c = canon(w)
            self.count[c] = self.count.get(c, 0) + times * (R - self.k + 1)

    def contig(self, name, seq, circular, times, R=None):
        """A truth contig, tiled `times` times; -> its index."""
        self.contigs.append((name, f"{name} circular=true" if circular else name, seq, circular))
        self.tile(f"{name}_truth", seq, times, R)
        return len(self.contigs) - 1

    def copy(self, ci, edits, times, R=None):
        """A copy of contig ci with edits (p, mid, skip) in descending p (so each p is a truth position), tiled `times` times."""
        seq = self.contigs[ci][2]
        for p, mid, skip in sorted(edits, reverse=True):
            seq = apply(seq, p, mid, skip)
        self.tile(f"{self.contigs[ci][0]}_v{len(self.reads)}", seq, times, R)
        return seq

    def expect(self, ci, p, mid, skip, pos, ref, alt, tag="plain"):
        """A row at POS, REF, ALT from the edit (mid at p, skip truth bases) evaluated at p; tag names what the event is for."""
        self.events.append(dict(ci=ci, p=p, mid=mid, skip=skip, POS=pos, REF=ref, ALT=alt, tag=tag))

    # ---- the rows the construction implies ---------------------------------------------------------------------------------------------
    def own(self):
        return {canon(w) for _, _, s, circ in self.contigs for w in windows(s, self.k, circ)}

    def measure(self, ev):
        """AK, RK and PK of a planted event from the exact counts: the edited sequence's windows from a, the truth's windows a .. p + d."""
        k = self.k
        _, _, s, circ = self.contigs[ev["ci"]]
        p, mid, skip = ev["p"], ev["mid"], ev["skip"]
        d = skip if mid == "" else 0                         # bases deleted, and bases inserted
        sl = len(mid) if skip == 0 else 0
        if circ:                                             # rotate so that a = p - k + 1 is base 0
            r0 = (p - k + 1) % len(s)
            s, p = s[r0:] + s[:r0], k - 1
        a = p - k + 1
        e = apply(s, p, mid, skip)
        e2, s2 = (e + e, s + s) if circ else (e, s)
        checked = [e2[j:j + k] for j in range(a, a + k + sl)]
        ref = [s2[j:j + k] for j in range(a, p + d + 1)]
        assert all(len(w) == k for w in checked + ref), "the event's windows do not fit the contig"
        own = self.own()
        held = [canon(w) in own for w in checked]
        ak = min(self.count.get(canon(w), 0) for w in checked)
        rk = min(self.count.get(canon(w), 0) for w in ref)
        pk = sum(held) if (len(mid), skip) == (1, 1) else sum(held[:-1])
        cur = s[p]
        c = P.candidates(cur, self.L).index((mid, skip))
        return dict(ak=ak, rk=rk, pk=pk, c=c, checked=checked)

    def rows(self, min_fraction=None):
        """The expected VCF rows in the file's order, as (contig, POS, REF, ALT, AK, RK, PK), after the fraction test."""
        F = self.kw["min_fraction"] if min_fraction is None else min_fraction
        out = []
        for ev in self.events:
            x = self.measure(ev)
            if not float(x["ak"]) >= F * float(x["ak"] + x["rk"]):
                continue
            out.append(((ev["ci"], ev["POS"], ev["p"], x["c"]),
                        (self.contigs[ev["ci"]][0], ev["POS"], ev["REF"], ev["ALT"], x["ak"], x["rk"], x["pk"])))
        return [r for _, r in sorted(out)]

    def unique(self):
        """Whether the truth contigs' windows are distinct canonical keys (no accidental repeat)."""
        ws = [canon(w) for _, _, s, circ in self.contigs for w in windows(s, self.k, circ)]
        return len(set(ws)) == len(ws)


def clear(s, p, before=None, at=None):
    """s with base p - 1 set to differ from the bases in `before` and base p from those in `at` (cyclic; None: left alone)."""
    s = list(s)
    for i, b in ((p - 1, before), (p, at)):
        if b is not None and s[i % len(s)] in b:
            s[i % len(s)] = next(x for x in BASES if x not in b)
    return "".join(s)


def plain_del(s, p, d):
    """s with the deletion of d bases at p made rightmost (base p + d differs from base p) and not shiftable (base p - 1 differs from
    base p + d - 1)."""
    s = clear(s, p + d, at=s[p])
    return clear(s, p, before=s[(p + d - 1) % len(s)])


# ---- A. every kind with exact counts ------------------------------------------------------------------------------------------------
C1, C2, C3 = 1, 1, 2


def kinds(k, L, seed=0x7A01, step=150):
    """A circular chromosome at C1 copies and one copy at C2 carrying, `step` bases apart: the three substitutions, insertions and
    deletions of 1 .. L bases (the base before an indel differs from its last base, so nothing shifts) and a homopolymer run of 4 one
    base longer and one of 5 one base shorter.  Tag "plain": AK = C2 m, RK = C1 m, PK = 0; "hins" / "hdel": PK = 4 / 4 (the run's
    windows slide onto the assembly's own).  Beside them:
      held_sub / held_del: a linear contig holds a copy of the edited sequence from p - 3 to p + k - 1 (a two-copy repeat shorter than k
        on each side of the event), so exactly 4 (substitution, its last window included) or 3 (a deletion, whose last window, the
        truth's own at p + d, is left out) checked windows are held;
      ref_beyond, ref_beyond_del: a third copy at C3 carries a substitution k bases after the event's last base, so the truth window
        just after the range a .. p + d is the least near it (RK = (C1 + C3) m; a range one window too long gives (C1 + C2) m);
      ref_last: a third copy carries one k - 1 bases after p, so the range's last window p is its only least one (RK = C1 m; one window
        short gives (C1 + C3) m).
    The third copy's substitutions give rows of their own ("third")."""
    for attempt in range(50):
        case = Case(k, L)
        x, plan = 200, []
        for j in range(3):
            plan.append(("sub", x, j))
            x += step
        for d in range(1, L + 1):
            plan += [("ins", x, d), ("del", x + step, d)]
            x += 2 * step
        if L:
            plan += [("hins", x, 4), ("hdel", x + step, 5), ("held_del", x + 2 * step, 3), ("ref_beyond_del", x + 3 * step, min(L, 2))]
            x += 4 * step
        plan += [("held_sub", x, 3), ("ref_beyond", x + step, 0), ("ref_last", x + 2 * step, 0)]
        s = genome(seed + attempt, x + 3 * step + 200)
        edits, third, events, held = [], [], [], []

        def sub(p, e, tag):
            edits.append((p, e, 1))
            events.append((p, e, 1, p + 1, s[p], e, tag))
        for kind, p, arg in plan:
            if kind == "sub":
                sub(p, other(s[p], arg + 1), "plain")
            elif kind == "ins":
                ins = "GATTACA"[:arg]
                s = clear(s, p, before=ins[-1], at=ins[0])
                edits.append((p, ins, 0))
                events.append((p, ins, 0, p, s[p - 1], s[p - 1] + ins, "plain"))
            elif kind in ("del", "ref_beyond_del", "held_del"):
                d = 1 if kind == "held_del" else arg
                s = plain_del(s, p, d)
                edits.append((p, "", d))
                events.append((p, "", d, p, s[p - 1:p + d], s[p - 1], "plain" if kind == "del" else kind))
                if kind == "held_del":
                    held.append((s[p - arg - 1], s[p - arg:p] + s[p + 1:p + k], s[p + k]))   # E's windows p - 3 .. p - 1
                elif kind == "ref_beyond_del":
                    q = p + d + k
                    third.append((q, other(s[q]), 1))
                    events.append((q, other(s[q]), 1, q + 1, s[q], other(s[q]), "third"))
            elif kind in ("hins", "hdel"):                  # a run of `arg` bases at p .. p + arg - 1
                b = s[p]
                s = s[:p] + b * arg + s[p + arg:]
                s = clear(clear(s, p, before=b), p + arg, at=b)
                if kind == "hins":
                    edits.append((p + arg, b, 0))
                    events.append((p + arg, b, 0, p, s[p - 1], s[p - 1] + b, kind))
                else:
                    edits.append((p + arg - 1, "", 1))
                    events.append((p + arg - 1, "", 1, p, s[p - 1] + b, s[p - 1], kind))
            elif kind == "held_sub":
                sub(p, other(s[p]), kind)
                held.append((s[p - arg - 1], s[p - arg:p] + other(s[p]) + s[p + 1:p + k], s[p + k]))
            else:                                            # ref_beyond: the third copy's change at p + k; ref_last: at p + k - 1
                sub(p, other(s[p]), kind)
                q = p + k if kind == "ref_beyond" else p + k - 1
                third.append((q, other(s[q], 2), 1))
                events.append((q, other(s[q], 2), 1, q + 1, s[q], other(s[q], 2), "third"))
        flank = genome(seed + 1000 + attempt, 60 * (len(held) + 1))
        par = flank[:60]
        for i, (before, h, after) in enumerate(held):      # flanks that differ from E's bases on either side of the copy
            par = clear(par, len(par), before=before) + h + clear(flank[60 * i + 60:60 * i + 120], 0, at=after)
        ci = case.contig("chrom", s, True, C1)
        case.contig("paralog", par, False, C1)
        if not case.unique():
            continue
        case.copy(ci, edits, C2)
        case.copy(ci, third, C3)
        if L == 0:
            events = [e for e in events if (len(e[1]), e[2]) == (1, 1)]
        for ev in events:
            case.expect(ci, *ev)
        case.shape = dict(m=case.R - k + 1)
        return case
    raise AssertionError("no repeat-free construction")


# ---- B. word offsets and layouts ------------------------------------------------------------------------------------------------------
def layout(k, contigs):
    """The first packed word of each contig: woff += bytes / 32 + 1, bytes = len + k - 1 on a circular contig of at least k bases."""
    woff = [0]
    for _, _, s, circ in contigs:
        woff.append(woff[-1] + (len(s) + (k - 1 if circ and len(s) >= k else 0)) // 32 + 1)
    return woff


def word_of(case, ev):
    """(packed word, offset, in the junction bytes) of the byte that the window ending at the event's p ends at: n + p for p < k - 1
    on a circular contig."""
    _, _, s, circ = case.contigs[ev["ci"]]
    p = ev["p"]
    idx = len(s) + p if circ and p < case.k - 1 else p
    return layout(case.k, case.contigs)[ev["ci"]] + idx // 32, idx % 32, idx >= len(s)


def offsets(k, L, seed=0x7B01):
    """Many contigs in one FASTA: a linear one first with a substitution in packed word 0 (no word before it); linear ones of k, k + 1,
    31, 32, 33, 63, 64 and 65 bases with a substitution at p = k - 1 (a row only where p + k fits); circular ones of 2k + 2L - 1 bases (no
    tried position) and 2k + 2L (every position tried) with one at p = 3; and a circular contig with substitutions 97 = 3 x 32 + 1 bases
    apart, one at every offset 0 .. 31 of a packed word, and one in its last word.  Every contig at C1, one copy of each at C2."""
    for attempt in range(50):
        case = Case(k, L)
        g = genome(seed + attempt, 6_000)
        at = 0
        small = 2 * k + 2 * L
        words = 32 * 97 + 3 * k
        plan = [("w0", 80, False, [k - 1])]
        plan += [(f"lin{n}", n, False, [k - 1] if n >= k else []) for n in sorted({k, k + 1, 31, 32, 33, 63, 64, 65})]
        plan += [("short", small - 1, True, [3]), ("tried", small, True, [3])]
        plan += [("words", words, True, [97 * j + 40 for j in range(32)] + [words - 2])]
        for name, n, circ, subs in plan:
            seq = g[at:at + n]
            at += n
            ci = case.contig(name, seq, circ, C1)
            if subs:
                case.copy(ci, [(p, other(seq[p]), 1) for p in subs], C2)
            for p in subs:
                if (circ and n >= small) or (not circ and p + k <= n):
                    case.expect(ci, p, other(seq[p]), 1, p + 1, seq[p], other(seq[p]), name)
        if case.unique():
            return case
    raise AssertionError("no repeat-free construction")


# ---- C. the circular junction and linear ends -------------------------------------------------------------------------------------------
def junction(k, L=3, seed=0x7C01):
    """Contigs of n = 4k + 2L + 16 bases, one per event, each at C1 with its copy at C2 (so no two events share windows).  Circular:
    substitutions at p = 0, 1, k - 2, k - 1 and n - 1; an insertion at p = 0 (the same event as one after the last base: POS 1); the
    deletions of the last d bases (p + d = n, d = 1 .. L: POS n - d); a deletion of 2 across the junction (p = n - 1, p + d > n: no row);
    the deletion of a last C before a first C, which is the first C's (evaluated at p = 0: POS 1, CT -> T); a homopolymer run of A across
    the junction one base longer (evaluated at p = 2, one row at POS 1).  Linear: substitutions at p = k - 2 (not tried) and n - k + 1
    (windows past the end), none giving a row, and at k - 1 and n - k, the first and last rows; deletions of 2 at n - k - 2 (the last
    row) and n - k - 1 (none)."""
    n = 4 * k + 2 * L + 16
    for attempt in range(50):
        case = Case(k, L)
        g = genome(seed + attempt, 20 * n)
        nothing = []

        def add(name, seq, circ, edit, row):
            ci = case.contig(name, seq, circ, C1)
            p, mid, skip = edit
            if p + skip <= n:
                case.copy(ci, [edit], C2)
            else:
                case.tile(f"{name}_v", apply(seq, p, mid, skip), C2)
            if row:
                case.expect(ci, p, mid, skip, *row, tag=name)
            else:
                nothing.append(name)
        piece = iter(g[i:i + n] for i in range(0, 20 * n, n))
        for p in (0, 1, k - 2, k - 1, n - 1):
            s = next(piece)
            add(f"sub{p}", s, True, (p, other(s[p]), 1), (p + 1, s[p], other(s[p])))
        s = clear(next(piece), 0, before="G", at="G")
        add("ins0", s, True, (0, "G", 0), (1, s[0], "G" + s[0]))
        for d in range(1, L + 1):
            s = plain_del(next(piece), n - d, d)
            add(f"del_end{d}", s, True, (n - d, "", d), (n - d, s[n - d - 1:], s[n - d - 1]))
        s = clear(next(piece), 1, at=next(piece)[0])
        s = clear(s, 1, at=s[n - 1])
        add("del_wrap", s, True, (n - 1, "", 2), None)
        s = next(piece)
        s = "CT" + s[2:n - 2] + "GC"                          # ...GC|CT...: the last C's deletion is the first C's
        add("del_cc", s, True, (0, "", 1), (1, "CT", "T"))
        s = next(piece)
        s = clear(clear("AA" + s[2:n - 2] + "AA", 2, at="A"), n - 2, before="A")   # A at n - 2, n - 1, 0, 1
        add("homo", s, True, (2, "A", 0), (1, "A", "AA"))
        for name, p, d, row in (("lin_first", k - 1, 0, True), ("lin_early", k - 2, 0, False), ("lin_last", n - k, 0, True),
                                ("lin_late", n - k + 1, 0, False), ("lin_del_last", n - k - 2, 2, True),
                                ("lin_del_late", n - k - 1, 2, False)):
            s = next(piece)
            if d:
                s = plain_del(s, p, d)
                add(name, s, False, (p, "", d), (p, s[p - 1:p + d], s[p - 1]) if row else None)
            else:
                add(name, s, False, (p, other(s[p]), 1), (p + 1, s[p], other(s[p])) if row else None)
        if case.unique():
            case.shape = dict(nothing=nothing, n=n)
            return case
    raise AssertionError("no repeat-free construction")


# ---- D. multi-allelic sites -------------------------------------------------------------------------------------------------------------
def multi(k=21, L=3, seed=0x7D01, sites=24, step=120):
    """A circular chromosome at 4 copies and three copies at 1, 2 and 3.  At each of `sites` positions two or three of the copies carry
    different substitutions (rows at one POS and p, in candidate order, each with its own AK and one RK); at every fourth site one copy
    carries a substitution and another a deletion (or an insertion) at the same p, whose first base differs from the substitution's."""
    for attempt in range(50):
        case = Case(k, L)
        s = genome(seed + attempt, sites * step + 300)
        copies, events = [[], [], []], []
        for i in range(sites):
            p = 150 + i * step
            if i % 4 == 3:
                e = other(s[p])
                if i % 8 == 3:
                    s = clear(s, p + 1, at=s[p] + e)
                    s = clear(s, p, before=s[p])
                    indel = (p, "", 1, p, s[p - 1:p + 1], s[p - 1])
                else:
                    ins = other(s[p], 2) + "T"
                    s = clear(s, p, before="T")
                    indel = (p, ins, 0, p, s[p - 1], s[p - 1] + ins)
                copies[0].append((p, e, 1))
                copies[1].append(indel[:3])
                events += [(p, e, 1, p + 1, s[p], e), indel]
            else:
                for j in range(2 + i % 2):
                    e = other(s[p], j + 1)
                    copies[j].append((p, e, 1))
                    events.append((p, e, 1, p + 1, s[p], e))
        ci = case.contig("chrom", s, True, 4)
        if not case.unique():
            continue
        for j, c in enumerate(copies):
            case.copy(ci, c, j + 1)
        for ev in events:
            case.expect(ci, *ev)
        return case
    raise AssertionError("no repeat-free construction")


# ---- E. high counts -----------------------------------------------------------------------------------------------------------------
HIGH = {16_383: (127, 129), 16_384: (16, 1024), 65_536: (64, 1024), 70_000: (70, 1000)}    # count: (copies, R - k + 1)


def high(k=21, seed=0x7E01, n=60):
    """Circular contigs of n bases, each with one substitution at p = 30 whose truth and alternative windows are read exactly RK and AK
    times: (AK, RK) = (16,383, 16,384), (65,536, 70,000) and (70,000, 65,536).  A count c is `copies` reads of R bases at every start,
    copies x (R - k + 1) = c."""
    pairs = [(16_383, 16_384), (65_536, 70_000), (70_000, 65_536)]
    for attempt in range(50):
        case = Case(k, 1)
        g = genome(seed + attempt, n * len(pairs))
        for i, (ak, rk) in enumerate(pairs):
            s = g[i * n:(i + 1) * n]
            ci = case.contig(f"high{i}", s, True, HIGH[rk][0], R=HIGH[rk][1] + k - 1)
            e = other(s[30])
            case.copy(ci, [(30, e, 1)], HIGH[ak][0], R=HIGH[ak][1] + k - 1)
            case.expect(ci, 30, e, 1, 31, s[30], e)
        if case.unique():
            case.shape = dict(pairs=pairs)
            return case
    raise AssertionError("no repeat-free construction")


def candidate_windows(k, L):
    """The checked windows of every candidate at one position; a batch of B positions takes a candidate table of 2 B times this."""
    return 3 * k + L * k + sum(4 ** s * (k + s) for s in range(1, L + 1))
