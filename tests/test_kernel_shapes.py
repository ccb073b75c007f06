"""The CUDA-only kernel code at the shapes where its multi-round, multi-tile and racing branches run: the trim overlap sweep with
diagonals of several 1024-thread rounds and windows on both sides of the last shared-memory size; the bridge distance sweep at row
counts around multiples of 256 and around the last shared-memory size, with and without u32 wraparound; the UPGMA CTA past one block
of rows with ties everywhere, +inf and signed zeros; and the k-mer table build under contention (whole warps inserting one k-mer, a
high table load, 32-bit side counts) with unitig sorts of several tiles and merge passes.  Every case runs on the host-emulation
build (which checks the generators and the oracles) and, marked gpu, on the CUDA build; each is compared with the CPU oracles
(the generators are in tests/kernel_shapes.py)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import cases
import kernel_shapes as S
import oracle_lib as o
import resolve_oracle as R
import table_routes
import table_sizing
import trim_oracle as T
from autocycler_b200 import api
from parity_common import check_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_LIB = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")
ORACLE_FN = {"start_end": T.trim_path_start_end, "hairpin_end": T.trim_path_hairpin_end, "hairpin_start": T.trim_path_hairpin_start}
PRODUCT_FN = {"start_end": api.trim_path_start_end, "hairpin_end": api.trim_path_hairpin_end, "hairpin_start": api.trim_path_hairpin_start}


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(EMU_LIB)


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


@pytest.fixture(scope="session")
def optin_emu():
    return S.H100_SHARED_OPTIN


@pytest.fixture(scope="session")
def optin_gpu(gpu):
    return S.device_shared_optin()


# ---- the shared-memory boundaries ----------------------------------------------------------------------------------------------------

def test_boundaries_emu(optin_emu):
    assert S.overlap_shared_k_max(optin_emu) == 9681 and S.bridge_shared_n_max(optin_emu) == 19369


@pytest.mark.gpu
def test_boundaries_gpu(optin_gpu):
    """On an H100 the largest shared-memory trim window is 9,681 and the largest shared-memory bridge row count 19,369: a change to
    either formula fails here rather than moving the boundary away from the cases below."""
    assert optin_gpu == S.H100_SHARED_OPTIN
    assert S.overlap_shared_k_max(optin_gpu) == 9681 and S.bridge_shared_n_max(optin_gpu) == 19369


# ---- A. the trim overlap kernel --------------------------------------------------------------------------------------------------------

def _reference_panics(p, w, mi, mu):
    """With weights near 2^32 the u32 sums of find_midpoint (trim.rs:482-507) wrap; when no matched piece then comes within 1.0 of the
    middle, the midpoint stays at piece 0, and if that is a gap the reference slices the path at usize::MAX and panics (the product
    reports an error).  Such a path has no answer to compare with."""
    al = T.overlap_alignment(p, p, w, mi, mu, True)
    return bool(al) and min(al[T.find_midpoint(al, w)][1::2]) < 0


def _check_trim(lib, optin, mode, kind):
    k_shared = S.overlap_shared_k_max(optin)
    paths, w, mi, mu = S.trim_call(mode, kind, k_shared, seed=len(mode) * 10 + S.TRIM_WEIGHTS.index(kind))
    if mode == "start_end" and kind == "big":
        paths = [p for p in paths if not _reference_panics(p, w, mi, mu)]
        assert len(paths) >= len(S.TRIM_WINDOWS) - 2
    assert {k_shared, k_shared + 1} <= {len(p) for p in paths}          # both sides of the shared-memory boundary in one call
    got = PRODUCT_FN[mode](paths, w, mi, mu, lib=lib)
    for x, p in enumerate(paths):
        assert got[x] == ORACLE_FN[mode](p, w, mi, mu), (mode, kind, len(p))
    return got


@pytest.mark.parametrize("kind", S.TRIM_WEIGHTS)
@pytest.mark.parametrize("mode", sorted(ORACLE_FN))
def test_trim_windows_emu(emu, optin_emu, mode, kind):
    _check_trim(emu, optin_emu, mode, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", S.TRIM_WEIGHTS)
@pytest.mark.parametrize("mode", sorted(ORACLE_FN))
def test_trim_windows_gpu(gpu, optin_gpu, mode, kind):
    _check_trim(gpu, optin_gpu, mode, kind)


def test_trim_cases_plant_what_they_say():
    """The oracle's view of the smaller windows: the planted overlaps are found, and with equal weights the identity of a planted
    start-end overlap is 3/4 exactly (kept at min_identity 0.75, dropped just above it)."""
    trimmed = exact = 0
    for mode in ORACLE_FN:
        for kind in S.TRIM_WEIGHTS:
            paths, w, mi, mu = S.trim_call(mode, kind, 40, seed=len(mode) * 10 + S.TRIM_WEIGHTS.index(kind))
            for p in paths:
                if len(p) > 2049:
                    continue
                t = ORACLE_FN[mode](p, w, mi, mu)
                trimmed += t is not None
                if kind == "equal" and mode == "start_end" and t is not None:
                    exact += ORACLE_FN[mode](p, w, mi + 1e-12, mu) is None
    assert trimmed >= 20 and exact >= 3, (trimmed, exact)


# ---- B. the bridge distance kernel -----------------------------------------------------------------------------------------------------

def _check_bridges(lib, big):
    n_units = 1200
    groups = S.bridge_groups(7 if big else 3, n_units)
    w = S.bridge_weights(big, n_units, 11 if big else 5)
    h = api._Handle(lib, 51)
    got = api.bridge_best_paths(groups, w, lib=lib, handle=h)
    info = api.AcResolveInfo()
    h.check(lib.ac_resolve_stats(h.ptr, info))
    assert (info.shared_jobs, info.hbm_jobs) == S.expected_jobs(groups, 10 ** 9)
    flag = "WRAP_DP" if big else "FAST_DP"
    setattr(R, flag, True)
    try:
        want_t, want_b = [], []
        for g in groups:
            b = R.Bridge(1, 2, [[1] + p + [2] for p in g], w)
            want_t.append(b.totals)
            want_b.append(b.best_path)
    finally:
        setattr(R, flag, False)
    assert got == (want_t, want_b)
    return want_t


def test_bridge_diagonal_dp_equals_cells():
    """The anti-diagonal form of the u32 DP against the literal cell loop, with wrapping weights, both ways round."""
    import random
    for s in range(120):
        rng = random.Random(s)
        w = S.bridge_weights(s % 2 == 0, 30, s)
        a = [rng.choice([1, -1]) * rng.randint(1, 30) for _ in range(rng.randint(0, 25))]
        b = [rng.choice([1, -1]) * rng.randint(1, 30) for _ in range(rng.randint(0, 25))]
        want = R.global_alignment_distance_cells(a, b, w)
        assert R.global_alignment_distance_diagonals(a, b, w) == want == R.global_alignment_distance_cells(b, a, w)
        assert R.global_alignment_distance_diagonals(b, a, w) == want


def test_bridge_big_weights_wrap():
    """The wrapping set makes the DP's u32 sums wrap at these sizes (the oracle's view)."""
    groups = S.bridge_groups(7, 1200)
    w = S.bridge_weights(True, 1200, 11)
    assert any(sum(w[abs(u)] for u in p) >= 2 ** 32 for g in groups for p in g)


@pytest.mark.parametrize("big", [False, True], ids=["small_weights", "wrapping_weights"])
def test_bridge_rows_emu(emu, big):
    _check_bridges(emu, big)


@pytest.mark.gpu
@pytest.mark.parametrize("big", [False, True], ids=["small_weights", "wrapping_weights"])
def test_bridge_rows_gpu(gpu, big):
    _check_bridges(gpu, big)


def _check_bridge_boundary(lib, optin):
    n_shared = S.bridge_shared_n_max(optin)
    paths, w = S.bridge_boundary_group(n_shared, 19)
    h = api._Handle(lib, 51)
    got = api.bridge_best_paths([paths], w, lib=lib, handle=h)
    info = api.AcResolveInfo()
    h.check(lib.ac_resolve_stats(h.ptr, info))
    assert (info.shared_jobs, info.hbm_jobs) == S.expected_jobs([paths], n_shared) == (5, 1)
    R.FAST_DP = True
    try:
        b = R.Bridge(1, 2, [[1] + p + [2] for p in paths], w)
    finally:
        R.FAST_DP = False
    assert got == ([b.totals], [b.best_path])


def test_bridge_boundary_emu(emu, optin_emu):
    _check_bridge_boundary(emu, optin_emu)


@pytest.mark.gpu
def test_bridge_boundary_gpu(gpu, optin_gpu):
    _check_bridge_boundary(gpu, optin_gpu)


# ---- C. the UPGMA kernel ---------------------------------------------------------------------------------------------------------------

UPGMA_CASES = [(kind, n) for kind in S.UPGMA_KINDS for n in S.UPGMA_N]


def _check_upgma(lib, kind, n):
    m, ids = S.upgma_matrix(kind, n, seed=n + S.UPGMA_KINDS.index(kind))
    got, _ = api.upgma(m, ids, lib=lib)
    assert S.merge_bits(got) == S.merge_bits(S.upgma_expected(m, ids))


@pytest.mark.parametrize("kind,n", UPGMA_CASES)
def test_upgma_emu(emu, kind, n):
    _check_upgma(emu, kind, n)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n", UPGMA_CASES)
def test_upgma_gpu(gpu, kind, n):
    _check_upgma(gpu, kind, n)


RESCAN = [(300, 100), (1100, 600)]


def _check_rescan(lib, n, rows):
    m, ids = S.upgma_rescan_matrix(n, rows, seed=n)
    got, _ = api.upgma(m, ids, lib=lib)
    assert S.merge_bits(got) == S.merge_bits(S.upgma_expected(m, ids))


def test_upgma_rescan_matrix_does_what_it_says():
    for n, rows in RESCAN:
        m, ids = S.upgma_rescan_matrix(n, rows, seed=n)
        first = S.upgma_expected(m, ids)[0]
        assert first[1:] == (n // 2 + 1, n, 0.25)
        assert all(np.argmin(np.where(np.arange(n) > i, m[i], np.inf)) == n - 1 for i in range(rows))


@pytest.mark.parametrize("n,rows", RESCAN)
def test_upgma_rescan_emu(emu, n, rows):
    _check_rescan(emu, n, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("n,rows", RESCAN)
def test_upgma_rescan_gpu(gpu, n, rows):
    _check_rescan(gpu, n, rows)


def test_upgma_inf_cases_reach_inf():
    """Each +inf matrix has a merge at +inf, after which the tie order alone decides."""
    for n in S.UPGMA_N[1:]:
        m, ids = S.upgma_matrix("inf", n, seed=n + S.UPGMA_KINDS.index("inf"))
        if np.isinf(m).any():
            assert S.upgma_expected(m, ids)[-1][3] == np.inf


# ---- D. the k-mer build under contention ------------------------------------------------------------------------------------------------

KMER_IDS = [c[0] for c in S.KMER_CASES]
_oracle = {}


def _kmer_oracle(index):
    """-> (name, k, files, oracle GFA, oracle stats, padded strands), computed once per process."""
    if index not in _oracle:
        name, k, files = S.kmer_case(index)
        with tempfile.TemporaryDirectory() as d:
            cases.write_case(files, d)
            gfa, _, st = o.compress_dir(d, k)
            _, oseqs = o.load_sequences(d, k)
        _oracle[index] = (name, k, files, gfa, st, [s[4] for s in oseqs])
    return _oracle[index]


def test_kmer_cases_cover_the_sort_shapes():
    """From the oracle's counts: the unitig sorts of the set take several 2,048-record tiles and up to two merge passes, and the input
    stays at a size the oracle checks in a few minutes."""
    shapes = [S.sort_shape(_kmer_oracle(x)[4].unitigs_before) for x in range(len(S.KMER_CASES))]
    assert max(t for t, _ in shapes) >= 2 and max(p for _, p in shapes) >= 2, shapes
    assert sum(1 for _, p in shapes if p >= 1) >= 2, shapes
    total = sum(len(s) for x in range(len(S.KMER_CASES)) for _, recs in _kmer_oracle(x)[2] for _, s in recs)
    assert total < 20_000_000, total


@pytest.mark.parametrize("index", range(len(S.KMER_CASES)), ids=KMER_IDS)
def test_kmer_build_emu(emu, index):
    _, k, files, _, _, _ = _kmer_oracle(index)
    check_case(emu, files, k)


@pytest.mark.gpu
@pytest.mark.parametrize("index", range(len(S.KMER_CASES)), ids=KMER_IDS)
def test_kmer_build_gpu(gpu, index):
    _, k, files, _, _, _ = _kmer_oracle(index)
    check_case(gpu, files, k)


LOADS = (0.9, 0.85, 0.8, 0.75, 0.7)


def _route(index, switch):
    """-> (environment, predicted sizing, expected attempts): AC_TABLE_LOAD at the highest of LOADS whose predicted route is the
    estimated table with no retry, or AC_BIG_COUNTS=1 at the default load."""
    _, k, _, _, st, padded = _kmer_oracle(index)
    if switch == "big_counts":
        pred = table_sizing.predict(padded, k, st.n_kmers // 2)
        att = [(pred["estimate_cap"], 1), (pred["safe"], 1)] if pred["retry"] else [(pred["capacity"], 1)]
        return {"AC_BIG_COUNTS": "1"}, pred, att
    for load in LOADS:
        try:
            pred = table_sizing.predict(padded, k, st.n_kmers // 2, load=load)
        except ValueError:
            continue
        if pred["estimate_cap"] is not None and not pred["retry"] and pred["capacity"] < pred["safe"]:
            return {"AC_TABLE_LOAD": repr(load)}, pred, [(pred["capacity"], 0)]
    raise AssertionError(f"no load in {LOADS} keeps case {index} on the estimated route")


def _check_child(lib_path, index, switch):
    """The case's build in a child process with the switch set (they are read once per process): three builds on one handle, each
    the oracle's GFA, each on the predicted route."""
    _, k, files, gfa, _, _ = _kmer_oracle(index)
    env_add, pred, want = _route(index, switch)
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        with open(os.path.join(d, "want.gfa"), "w") as f:
            f.write(gfa)
        code = S.CHILD % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": lib_path}
        env = {**os.environ, "AC_HOST_PROFILE": "1", **env_add}
        for v in ("AC_COUNT_ALARM", "AC_TABLE_LOAD", "AC_BIG_COUNTS"):
            if v not in env_add:
                env.pop(v, None)
        r = subprocess.run([sys.executable, "-c", code, d, str(k), os.path.join(d, "want.gfa")], env=env, capture_output=True, text=True,
                           timeout=1200)
    assert r.returncode == 0 and "CHECKED" in r.stdout, r.stderr[-3000:]
    caps = [tuple(map(int, ln.split()[1:])) for ln in r.stdout.splitlines() if ln.startswith("CAPACITY")]
    assert caps == [(pred["capacity"], pred["distinct"])] * 3, (caps, pred)
    blocks = r.stderr.split("BUILD\n")[1:]
    assert len(blocks) == 3
    for block in blocks:
        att = [(int(c), int(b)) for _, c, b in table_routes.ATTEMPT.findall(block)]
        assert att == want, (att, want, pred)


SWITCHES = ["high_load", "big_counts"]


@pytest.mark.parametrize("switch", SWITCHES)
@pytest.mark.parametrize("index", range(len(S.KMER_CASES)), ids=KMER_IDS)
def test_kmer_build_switches_emu(emu, index, switch):
    _check_child(EMU_LIB, index, switch)


@pytest.mark.gpu
@pytest.mark.parametrize("switch", SWITCHES)
@pytest.mark.parametrize("index", range(len(S.KMER_CASES)), ids=KMER_IDS)
def test_kmer_build_switches_gpu(gpu, index, switch):
    _check_child(api.DEFAULT_LIB, index, switch)
