"""The adjacency stage's extension filter (pipeline.cu: one 64-bit word per (k-1)-mer node, which of its ten extensions some distinct
k-mer makes) on the host-emulation build, on the inputs whose paths the filter makes rare: (k-1)-mers that are their own reverse
complement, the dot extensions at unrepaired sequence ends, and a filter shrunk to a single word (AC_EXT_FILTER_WORDS), where every
test passes by chance and every candidate neighbour goes to the table.  Every case must give the oracle's bytes."""
import os
import random
import subprocess
import sys

import pytest

import cases
import oracle_lib as o
from parity_common import check_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")
# W = 1, 2, 3 and 4 words, and the k whose keys fill exactly 2 bits of their top word (33, 65)
KS = [5, 11, 31, 33, 51, 63, 65, 91, 127]
UNITS = ["AC", "GT", "AT", "GC", "ACGT", "TGCA", "AATT", "GAATTC"]     # tandem repeats: (AT)n, (ACGT)n ... hold (k-1)-mers equal to their own rc


def palindrome_case(seed, k):
    """Tandem repeats of short units, their reverse complements and random flanks, in several files; some contigs share the runs with
    other flanks.  Every contig also holds one (k-1)-mer P = h + rc(h) between two random bases, on either strand: the k-mer that
    enters P from one contig has the k-mers that leave it in the others as neighbours the insert never saw next to it, and the filter
    may hold them from either side of P."""
    rng = random.Random(seed)
    files = []
    shared = cases.rand_seq(rng, rng.randint(k, 2 * k))
    half = cases.rand_seq(rng, (k - 1) // 2)
    pal = half + cases.rc(half)
    for f in range(rng.randint(2, 4)):
        recs = []
        for c in range(rng.randint(1, 2)):
            unit = rng.choice(UNITS)
            run = unit * rng.randint(2, (3 * k) // len(unit) + 2)
            s = cases.rand_seq(rng, rng.randint(0, k)) + run + (shared if rng.random() < 0.5 else cases.rand_seq(rng, rng.randint(1, k)))
            s += cases.rand_seq(rng, rng.randint(1, k)) + pal + cases.rand_seq(rng, rng.randint(1, k))
            if rng.random() < 0.5:
                s += cases.rc(run) + cases.rand_seq(rng, rng.randint(0, k))
            if rng.random() < 0.5:
                s = cases.rc(s)
            if len(s) < k:
                s += cases.rand_seq(rng, k - len(s))
            recs.append((f"c{c + 1}", s))
        files.append((f"asm_{f:02d}.fasta", recs))
    return files


def unrepaired_case(seed, k):
    """A genome in several files, next to contigs of their own and fragments whose ends are random: end repair finds nothing for those
    ends, so their dots stay, and the k-mer before each dot run has the dotted k-mer ("X." or ".X") as a neighbour in the table."""
    rng = random.Random(seed)
    genome = cases.rand_seq(rng, rng.randint(2 * k, 6 * k))
    files = []
    for f in range(rng.randint(2, 4)):
        recs = [("g", genome if rng.random() < 0.5 else cases.rc(genome))]
        if rng.random() < 0.7:
            a = rng.randrange(len(genome) - k)
            frag = genome[a:a + rng.randint(k, len(genome) - a)]
            recs.append(("frag", cases.rand_seq(rng, rng.randint(1, k)) + frag + cases.rand_seq(rng, rng.randint(0, k))))
        if rng.random() < 0.5:
            recs.append(("own", cases.rand_seq(rng, rng.randint(k, 3 * k))))
        if rng.random() < 0.3:
            recs.append(("run", rng.choice(UNITS) * (k // 2 + 3)))
        files.append((f"asm_{f:02d}.fasta", recs))
    return files


def _oracle_sequences(files, k):
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        try:
            return [t[4] for t in o.load_sequences(d, k)[1]]
        except o.OracleError:
            return []


def _has_palindromic_node(seqs, k):
    for s in seqs:
        for i in range(len(s) - (k - 1) + 1):
            w = s[i:i + k - 1]
            if "." not in w and w == cases.rc(w):
                return True
    return False


def _has_dots(seqs, k):
    return any(s.startswith(".") or s.endswith(".") for s in seqs)


def test_the_cases_hold_what_they_are_for():
    """Most palindrome cases hold a (k-1)-mer equal to its reverse complement; most unrepaired cases keep dots after end repair (at
    k = 5 the two-base end literals occur everywhere and every end is repaired)."""
    for k in KS:
        pal = sum(_has_palindromic_node(_oracle_sequences(palindrome_case(seed, k), k), k) for seed in range(10))
        dots = sum(_has_dots(_oracle_sequences(unrepaired_case(seed, k), k), k) for seed in range(10))
        assert pal >= 5 and (dots >= 5 or k < 11), (k, pal, dots)


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    from autocycler_b200 import api
    return api.load_library(EMU)


@pytest.mark.parametrize("k", KS)
def test_palindromic_nodes(emu, k):
    for seed in range(20):
        check_case(emu, palindrome_case(100 * k + seed, k), k)


@pytest.mark.parametrize("k", KS)
def test_dot_extensions_at_unrepaired_ends(emu, k):
    for seed in range(20):
        check_case(emu, unrepaired_case(200 * k + seed, k), k)


SHRUNK = """
import sys
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
import cases, test_ext_filter_emu as t
from autocycler_b200 import api
from parity_common import check_case
lib = api.load_library(%(lib)r)
for k in t.KS:
    for seed in range(12):
        check_case(lib, cases.random_case(300 * k + seed, k), k)
        check_case(lib, t.palindrome_case(400 * k + seed, k), k)
        check_case(lib, t.unrepaired_case(500 * k + seed, k), k)
print("SAME AS THE ORACLE")
"""


@pytest.mark.parametrize("words", [1, 3])
def test_a_filter_of_a_few_words(emu, words):
    """The filter shrunk to one or three words: almost every extension of every node tests present, so every candidate neighbour that
    the insert did not see is looked up in the table.  The switch is read once per process, so the cases run in a child."""
    code = SHRUNK % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": EMU}
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, "AC_EXT_FILTER_WORDS": str(words)}, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "SAME AS THE ORACLE" in r.stdout, r.stderr[-3000:]
