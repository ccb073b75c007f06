"""The compress tail (pipeline.cu) at shapes the other suites leave out: the GFA text's sequence bytes and path-line wrappers are
copied by a warp per piece, and the H, S and L lines go to the host on a stream of their own while the P lines render.  The cases:
S lines whose sequences end anywhere in a 32-byte sector and a 64-base piece, a repeat expansion with a single level, a graph with
no candidates at all, and, from tests/expand_shapes.py, a full looping simplify grid and a cascade whose later passes step over
levels.  Each case runs on the emulation build and, marked gpu, on the CUDA build, against the oracle; a census from the emulation
build's AC_HOST_PROFILE lines shows that the small cases plant what they say."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import cases
import expand_shapes as E
from autocycler_b200 import api
from parity_common import check_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_LIB = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(EMU_LIB)


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def _rand(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def _no_candidates():
    """Three copies of one random contig: one unitig, no repeat-expansion candidate."""
    s = _rand(np.random.default_rng(41), 5000)
    return 51, [(f"asm_{a}.fasta", [("contig_1", s)]) for a in range(3)]


def _single_level():
    """Forks that never meet again: in each contig a shared head runs into one of two unrelated tails, so every candidate (a head and
    its two tails) is alone on its unitigs, and every candidate sits on level 1."""
    rng = np.random.default_rng(42)
    heads = [_rand(rng, 3000) for _ in range(3)]
    tails = [[_rand(rng, 2000) for _ in range(2)] for _ in range(3)]
    return 51, [(f"asm_{a}.fasta", [(f"contig_{c + 1}", heads[c] + tails[c][a]) for c in range(3)]) for a in range(2)]


def _ragged_sequences():
    """Unitig lengths of every residue mod 32 and mod 64: contigs of lengths 1000 + i, i < 64, each in two assemblies, so the S lines'
    sequences start and end anywhere in a sector and in a 64-base piece."""
    rng = np.random.default_rng(43)
    contigs = [(f"contig_{i + 1}", _rand(rng, 1000 + i)) for i in range(64)]
    return 51, [(f"asm_{a}.fasta", contigs) for a in range(2)]


SMALL = {"no_candidates": _no_candidates, "single_level": _single_level, "ragged_sequences": _ragged_sequences}
LOOPING_CASE = "snp_k67_looping"      # threads of a full simplify grid loop within a level
EMPTY_LEVELS_CASE = "cascade_k65"     # later passes that step over levels nobody is due on


def _profile(k, files):
    """-> (launch lines, per-level lines) of one fused emulation build under AC_HOST_PROFILE."""
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        code = E.CHILD % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": EMU_LIB}
        env = {**os.environ, "AC_HOST_PROFILE": "1"}
        env.pop("AC_DEVICE_TIGHT_ARENA", None)
        r = subprocess.run([sys.executable, "-c", code, d, str(k), "fused"], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "DONE" in r.stdout, r.stderr[-3000:]
    return E.launches(r.stderr), E.level_lines(r.stderr)


def _named(name):
    _, k, files, _ = E.case(E.NAMES.index(name))
    return k, files


def test_census_small_cases(emu):
    launches, _ = _profile(*_no_candidates())
    assert launches == []                                        # no candidate: the expansion is not launched
    launches, levels = _profile(*_single_level())
    assert launches and launches[0][2] == 1 and launches[0][3] > 1, launches
    k, files = _ragged_sequences()
    lengths = {len(s) for _, recs in files for _, s in recs}
    assert {n % 32 for n in lengths} == set(range(32))


@pytest.mark.parametrize("name", sorted(SMALL) + [LOOPING_CASE, EMPTY_LEVELS_CASE])
def test_tail_schedule_emu(emu, name):
    k, files = SMALL[name]() if name in SMALL else _named(name)
    check_case(emu, files, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SMALL) + [LOOPING_CASE, EMPTY_LEVELS_CASE])
def test_tail_schedule_gpu(gpu, name):
    k, files = SMALL[name]() if name in SMALL else _named(name)
    check_case(gpu, files, k)
