"""The device repeat expansion of the fused build (pipeline.cu: LevelsCoopBody, SimplifyCoopBody, ApplyLevelBody and its warp byte
loops) at the shapes only the CUDA build runs: a full simplify grid whose threads loop within a level, more than one CTA relaxing the
levels, compares whose first mismatch lies past the first 32-byte chunk or whose second mismatch lies a chunk further on, destinations
that move on the first pass, multi-pass cascades that step over levels nobody is due on, sources holding both strands of one unitig,
and a closing renumbering full of ties.  The emulation build runs the same bodies on one thread with plain byte loops, so every case
runs there (which checks the generators and the oracle) and, marked gpu, on the CUDA build, through check_case against the oracle.
A census, which needs no GPU, shows from the graph before simplify and from the profile lines that each case plants what it says
(the generators are in tests/expand_shapes.py)."""
import os
import subprocess
import sys
import tempfile

import pytest

import cases
import expand_shapes as E
import oracle_lib as o
from autocycler_b200 import api
from parity_common import check_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_LIB = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")
INDEX = {name: x for x, name in enumerate(E.NAMES)}
FULL_GRID_CASE = "snp_pair_k129"          # large k, a full grid, relocations on the first pass and compares across two chunks
REPEAT_CASE = "cascade_k129"              # relocations on several passes: the arena bump order is a race on the GPU


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(EMU_LIB)


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


_cases, _oracle, _census = {}, {}, {}


def _case(name):
    if name not in _cases:
        _cases[name] = E.case(INDEX[name])
    return _cases[name]


def _oracle_gfa(name):
    if name not in _oracle:
        _, k, files, _ = _case(name)
        with tempfile.TemporaryDirectory() as d:
            cases.write_case(files, d)
            _oracle[name] = o.compress_dir(d, k)[0]
    return _oracle[name]


def _child(lib_path, name, mode, env_add=None):
    """The case's builds in a child process (AC_HOST_PROFILE and AC_DEVICE_TIGHT_ARENA are read by the library) -> (stderr, {file: text})."""
    _, k, files, _ = _case(name)
    env = {**os.environ, "AC_HOST_PROFILE": "1", **(env_add or {})}
    if "AC_DEVICE_TIGHT_ARENA" not in (env_add or {}):
        env.pop("AC_DEVICE_TIGHT_ARENA", None)
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        code = E.CHILD % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": lib_path}
        r = subprocess.run([sys.executable, "-c", code, d, str(k), mode], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0 and "DONE" in r.stdout, r.stderr[-3000:]
        out = {f: open(os.path.join(d, f)).read() for f in os.listdir(d) if f.endswith(".gfa")}
    return r.stderr, out


def _census_of(name):
    """-> (candidates of the graph before simplify, launch lines, per-level lines, final GFA) from the emulation build, once per process."""
    if name not in _census:
        err, out = _child(EMU_LIB, name, "census")
        _census[name] = (E.candidates(out["before.gfa"]), E.launches(err), E.level_lines(err), out["fused.gfa"], out["before.gfa"])
    return _census[name]


# ---- the device ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_sm_count_gpu(gpu):
    """The grid sizes below assume an H100's 132 SMs: a device with another count fails here rather than moving the boundaries."""
    assert E.device_sm_count() == E.H100_SMS


# ---- the census ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", E.NAMES)
def test_census(emu, name):
    """What each case plants, from the plain build's graph before simplify (the oracle's exclusive sets and common sequences) and from
    the fused build's AC_HOST_PROFILE lines."""
    _, k, _, planted = _case(name)
    cands, launch, levels, _, before = _census_of(name)
    h = k // 2
    assert len(launch) == 1, launch                                   # the arena held every pass: one launch
    passes, _, n_levels, n_cands = launch[0]
    assert n_cands == len(cands)                                      # the census sees the device's candidates (no fixed end took one away)
    for c in cands[:: max(1, len(cands) // 6)]:                       # the Python common length is the oracle's
        assert len(o.gfa_common_seq(before, c["spec"], c["side"] == 0)) == c["common"], c
    first_c = [E.first_pass_c(c) for c in cands]
    assert max(c["gn"] for c in cands) <= 4                           # a strand has at most four successors: gn never reaches 5 or 6
    if k >= E.LARGE_K:
        assert n_cands > E.full_grid(E.H100_SMS), n_cands
    if "snp" in planted and len(planted) <= 2 and "inv" not in planted and not name.startswith("contig"):
        # an SNP's alleles are k bases that agree on h = k // 2 at both ends: the first candidate of a site takes h from the pristine
        # alleles, its partner then compares h + 1 bases in the arena and stops at index h
        snp = [c for c in cands if c["gn"] == 2 and c["min_len"] == k and len(c["mism"][0]) == 1]
        assert len(snp) == 2 * planted["snp"], (len(snp), planted)
        assert all(c["common"] == h and c["mism"][0] == [h] for c in snp)
        assert (max(first_c) > E.SEQ_SLACK) == (h > E.SEQ_SLACK) and max(first_c) == h
    if "pair" in planted:
        # two substitutions 33-40 apart: the partner's compare (h + 1 + d bases once the first took h) meets both, in different chunks
        pair = [c for c in cands if c["gn"] == 2 and len(c["mism"][0]) == 2 and c["mism"][0][0] == h]
        assert len(pair) == 2 * planted["pair"], (len(pair), planted)
        for c in pair:
            first, second = c["mism"][0]
            assert 33 <= second - first <= 40 and first // E.CHUNK != second // E.CHUNK and second < c["min_len"] - h
    if name in E.MULTI_PASS:
        assert passes >= 3, launch
        assert {3, 4} <= {c["gn"] for c in cands}
        assert sum(c["common"] > c["zero_cap"] > 0 for c in cands) > 100   # avoid_zero_len_unitigs caps, then the pass after goes on
        # a later pass steps over a level nobody is due on and works on another
        assert any(len(levels[p]) < n_levels and any(due for lv, due in levels[p].items() if lv < n_levels) for p in range(1, passes))
    if "inv" in planted:
        dup = [c for c in cands if c["dup"] and c["common"] > 0]
        assert len(dup) == planted["inv"] and all(c["zero_cap"] == (c["min_len"] - 1) // 2 for c in dup)
    if name.startswith("contig"):
        # avoid_start_of_path: every occurrence of a destination follows one of its sources, so its bound (first position - 1) is never
        # below the zero-length cap (shortest source - 1); sites 1, 2, ... bases from the contig ends bring the two together
        margins = [c["start_cap"] - min(c["common"], c["zero_cap"]) for c in cands if c["start_cap"] is not None and c["common"] > 0]
        assert min(margins) == 0 and sum(m <= 2 for m in margins) >= 4, sorted(margins)[:10]
    assert all(levels[0].values()) and len(levels[0]) == n_levels     # the first pass visits every level


def test_census_grid_shapes(emu):
    """Across the cases: the levels relaxed by more than one CTA, a full simplify grid at every large k, and one case whose threads
    take more than one candidate per level."""
    counts = {name: _census_of(name)[1][0][3] for name in E.NAMES}
    assert max(counts.values()) > E.LEVELS_PER_BLOCK
    assert max(counts.values()) > E.looping_grid(E.H100_SMS), counts
    assert all(counts[n] > E.full_grid(E.H100_SMS) for n, c in zip(E.NAMES, E.CASES) if c[1] >= E.LARGE_K), counts
    assert sum(len(s) for n in E.NAMES for _, recs in _case(n)[2] for _, s in recs) < 40_000_000


def test_census_renumber_ties(emu):
    """The closing device renumbering: fully expanded sites leave runs of equal 1-base unitigs and the copy-number alleles equal
    sequences longer than 8 bases, so NumberLess goes past the 8-base prefix to the arena, then to depth and position.  The tied
    groups span more than one sort tile."""
    _, _, _, final, _ = _census_of(REPEAT_CASE)
    ties = E.tie_groups(final)
    assert any(first // E.SORT_TILE != last // E.SORT_TILE for _, first, last in ties)
    assert sum(1 for length, _, _ in ties if length > 8) > 50


# ---- every case against the oracle -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", E.NAMES)
def test_expand_emu(emu, name):
    _, k, files, _ = _case(name)
    check_case(emu, files, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", E.NAMES)
def test_expand_gpu(gpu, name):
    _, k, files, _ = _case(name)
    check_case(gpu, files, k)


# ---- the arena regrown before every pass, and repeated builds ----------------------------------------------------------------------

def _check_tight(lib_path):
    err, out = _child(lib_path, FULL_GRID_CASE, "fused", {"AC_DEVICE_TIGHT_ARENA": "1"})
    launch = E.launches(err)
    assert len(launch) >= 2 and all(p == 1 for p, _, _, _ in launch) and launch[-1][1] == len(launch), launch
    assert launch[0][3] > E.full_grid(E.H100_SMS)
    assert out["fused.gfa"] == _oracle_gfa(FULL_GRID_CASE)


def test_tight_arena_emu(emu):
    _check_tight(EMU_LIB)


@pytest.mark.gpu
def test_tight_arena_gpu(gpu):
    """One pass per launch, the arena regrown and the work resumed from next_set / next_due before every pass."""
    _check_tight(api.DEFAULT_LIB)


def _check_repeat(lib_path):
    _, out = _child(lib_path, REPEAT_CASE, "repeat")
    assert out["fused_0.gfa"] == out["fused_1.gfa"] == out["fused_2.gfa"] == _oracle_gfa(REPEAT_CASE)


def test_repeat_builds_emu(emu):
    _check_repeat(EMU_LIB)


@pytest.mark.gpu
def test_repeat_builds_gpu(gpu):
    """Two fused builds on one handle and one on a fresh handle: the same bytes, whatever order the relocations took arena space in."""
    _check_repeat(api.DEFAULT_LIB)
