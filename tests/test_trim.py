"""`autocycler trim` (trim.rs): the reference's unit-test data (tests/golden/trim_kats.json, extracted from trim.rs:516-823), seeded
random paths and whole-cluster runs, each checked against the CPU oracle (tests/trim_oracle.py).  The CPU tests run the product's
code through the host-emulation library (the alignment kernel's per-cell recurrence, right-edge maximum and traceback, serially);
the tests marked gpu run the CUDA build on the H100."""
import hashlib
import json
import os
import random
import subprocess

import pytest

import oracle_lib
import trim_oracle as T
from autocycler_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "trim_kats.json")))["cases"]
ORACLE_FN = {"start_end": T.trim_path_start_end, "hairpin_end": T.trim_path_hairpin_end, "hairpin_start": T.trim_path_hairpin_start}
PRODUCT_FN = {"start_end": api.trim_path_start_end, "hairpin_end": api.trim_path_hairpin_end, "hairpin_start": api.trim_path_hairpin_start}


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def _weights(case):
    return {int(u): w for u, w in case["weights"].items()}


# ---- the reference's KATs ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", KATS, ids=[f"{c['test']}-{i}" for i, c in enumerate(KATS)])
def test_kats_oracle(case):
    w = _weights(case)
    if case["kind"] == "overlap_alignment":
        for cells in (False, True):
            got = T.overlap_alignment(case["path"], case["path"], w, case["min_identity"], case["max_unitigs"], case["skip_diagonal"], cells=cells)
            assert [list(p) for p in got] == (case["expected"] or [])
        return
    steps = case["kind"].split("_then_")
    path = case["path"]
    for s in steps:
        path = ORACLE_FN[s](path, w, case["min_identity"], case["max_unitigs"])
    assert path == case["expected"]


def _product_kats(lib):
    for case in KATS:
        w = _weights(case)
        if case["kind"] == "overlap_alignment":
            # the product exposes the alignment through trim_path_start_end: the oracle's alignment above is the reference's, and the
            # product's start-end trim must equal the oracle's on the same path
            want = T.trim_path_start_end(case["path"], w, case["min_identity"], case["max_unitigs"])
            assert api.trim_path_start_end([case["path"]], w, case["min_identity"], case["max_unitigs"], lib=lib) == [want], case["test"]
            continue
        path = case["path"]
        for s in case["kind"].split("_then_"):
            path = PRODUCT_FN[s]([path], w, case["min_identity"], case["max_unitigs"], lib=lib)[0]
        assert path == case["expected"], case["test"]


def test_kats_emu(emu):
    _product_kats(emu)


@pytest.mark.gpu
def test_kats_gpu(gpu):
    _product_kats(gpu)


# ---- seeded random paths ----------------------------------------------------------------------------------------------------------

def _random_case(seed):
    """A path with a planted start-end or hairpin overlap (substitutions, indels), tied weights, and a trim setting."""
    rng = random.Random(seed)
    n_units = rng.randint(3, 40)
    weights = {u: rng.choice([1, 5, 10, 10, 10, 50, 100, 1000, rng.randint(1, 5000)]) for u in range(1, n_units + 1)}
    core = [rng.choice([1, -1]) * rng.randint(1, n_units) for _ in range(rng.randint(1, 40))]
    ov = max(1, min(len(core), rng.randint(1, 12)))

    def mutate(p):
        p = list(p)
        for _ in range(rng.choice([0, 0, 1, 2, 3])):
            r = rng.random()
            x = rng.randrange(len(p) + 1)
            if r < 0.4 and p:
                p[min(x, len(p) - 1)] = rng.choice([1, -1]) * rng.randint(1, n_units)
            elif r < 0.7:
                p.insert(x, rng.choice([1, -1]) * rng.randint(1, n_units))
            elif p:
                del p[min(x, len(p) - 1)]
        return p
    kind = rng.choice(["start_end", "hairpin_end", "hairpin_start", "none", "both"])
    if kind == "start_end":
        path = core + mutate(core[:ov])
    elif kind == "hairpin_end":
        path = core + mutate(T.reverse_path(core[-ov:]))
    elif kind == "hairpin_start":
        path = mutate(T.reverse_path(core[:ov])) + core
    elif kind == "both":
        path = mutate(T.reverse_path(core[:ov])) + core + mutate(T.reverse_path(core[-ov:]))
    else:
        path = core
    n = len(path)
    max_unitigs = rng.choice([0, 1, 2, 3, 5, n // 2, n, n + 7, 1000])
    min_identity = rng.choice([0.0, 1.0, 0.5, 0.75, 0.9, 0.95, 2 / 3, 0.8])
    return path, weights, min_identity, max_unitigs


def _check_random(lib, seeds):
    for mode in ("start_end", "hairpin_end", "hairpin_start"):
        cases = [_random_case(s * 3 + len(mode)) for s in seeds]
        # one batch per setting: the product runs a batch as one round
        by_setting = {}
        for path, w, mi, mu in cases:
            by_setting.setdefault((mi, mu, tuple(sorted(w.items()))), []).append(path)
        for (mi, mu, wi), paths in by_setting.items():
            w = dict(wi)
            want = [ORACLE_FN[mode](p, w, mi, mu) for p in paths]
            assert PRODUCT_FN[mode](paths, w, mi, mu, lib=lib) == want, (mode, mi, mu)


def test_random_paths_emu(emu):
    _check_random(emu, range(300))


@pytest.mark.gpu
def test_random_paths_gpu(gpu):
    _check_random(gpu, range(300))


def test_exact_identity_threshold(emu):
    """identity = total_matches / mean_length compared with `<` in f64: a trim whose identity equals min_identity is kept."""
    w = {1: 10, 2: 10, 3: 10, 4: 10, 5: 10, 6: 10, 7: 10}
    path = [1, 2, 3, 4, 5, 6, 1, 7, 3]            # overlap 1,2,3 against 1,7,3: identity 2/3 exactly
    for mi in (2 / 3, 0.6666, 0.6667, 1.0, 0.0):
        assert api.trim_path_start_end([path], w, mi, 100, lib=emu) == [T.trim_path_start_end(path, w, mi, 100)]


def test_ties_and_windows(emu):
    """Equal weights everywhere make the up/left comparison (>=) and the right-edge maximum (strict >) decide; windows cover the
    last k entries of path_b against the first k of path_a."""
    w = {u: 1 for u in range(1, 9)}
    for path in ([1, 2, 1, 2, 1, 2], [1, 2, 3, 1, 3, 2, 1, 2], [5, 5, 5, 5], [1, -1, 1, -1, 1], [3, 4, -4, -3, 3, 4]):
        for mu in range(0, len(path) + 2):
            for mi in (0.0, 0.5, 1.0):
                for mode in ORACLE_FN:
                    assert PRODUCT_FN[mode]([path], w, mi, mu, lib=emu) == [ORACLE_FN[mode](path, w, mi, mu)], (path, mu, mi, mode)


def test_oracle_rows_equal_cells():
    for seed in range(200):
        path, w, mi, mu = _random_case(seed)
        for a, b, skip in ((path, path, True), (T.reverse_path(path), path, False)):
            assert T.overlap_alignment(a, b, w, mi, max(mu, 1), skip) == T.overlap_alignment(a, b, w, mi, max(mu, 1), skip, cells=True)


# ---- whole clusters ---------------------------------------------------------------------------------------------------------------

def _rc(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def _cluster_gfa(tmp_path, contigs):
    """1_untrimmed.gfa of a one-cluster genome: compress (CPU oracle) + merge_linear_paths (cluster.rs:794-806)."""
    d = tmp_path / "asm"
    d.mkdir()
    for i, seq in enumerate(contigs):
        (d / f"a{i}.fasta").write_text(f">c{i} len={len(seq)}\n{seq}\n")
    gfa, _, _ = oracle_lib.compress_dir(str(d), 51)
    return oracle_lib.gfa_merge_linear_paths(gfa, use_paths=True, renumber=False)


def _genome(seed, n):
    rng = random.Random(seed)
    return "".join(rng.choice("ACGT") for _ in range(n))


def _mutate(seq, seed, n):
    rng = random.Random(seed)
    s = list(seq)
    for _ in range(n):
        x = rng.randrange(len(s))
        s[x] = rng.choice("ACGT".replace(s[x], ""))
    return "".join(s)


def _clusters():
    g = _genome(1, 6000)
    return {
        "circular_overlaps": [g + g[:700], _mutate(g, 2, 3) + g[:400], g[1500:] + g[:1500] + g[1500:2300], g],
        "hairpin": [g + _rc(g[-600:]), _mutate(g, 3, 2) + _rc(g[-500:]), _rc(g[:450]) + g, g],
        "length_outlier": [g, _mutate(g, 4, 2), _mutate(g, 5, 2), g[:3000], g + g[:200]],
        "nothing_trims": [g, _mutate(g, 6, 4), _mutate(g, 7, 1)],
    }


CLUSTER_SETTINGS = [(0.75, 5000, 5.0), (0.75, 5000, 0.0), (0.75, 0, 5.0), (0.95, 3, 1.0)]


def _check_cluster(lib, tmp_path, name, settings):
    untrimmed = _cluster_gfa(tmp_path, _clusters()[name])
    mi, mu, mad = settings
    want_gfa, want_yaml = T.trim_gfa(untrimmed, mi, mu, mad)
    g, _ = api.UnitigGraph.from_gfa_lines(untrimmed.encode(), lib=lib)
    g.trim(mi, mu, mad)
    assert bytes(g.gfa_bytes()).decode() == want_gfa
    assert g.trimmed_yaml() == want_yaml
    return untrimmed, want_gfa, want_yaml


@pytest.mark.parametrize("settings", CLUSTER_SETTINGS)
@pytest.mark.parametrize("name", sorted(_clusters()))
def test_cluster_emu(emu, tmp_path, name, settings):
    _check_cluster(emu, tmp_path, name, settings)


def test_cluster_cases_trim(tmp_path):
    """The synthetic clusters exercise what they are named for (the oracle's own view)."""
    c = _clusters()
    for name in c:
        u = _cluster_gfa(tmp_path / name, c[name]) if (tmp_path / name).mkdir() is None else None
        gfa, yaml = T.trim_gfa(u, 0.75, 5000, 5.0)
        lengths = [int(x[2:]) for x in yaml.splitlines() if x.startswith("- ")]
        if name == "nothing_trims":
            assert sorted(lengths) == sorted(len(s) for s in c[name])
        elif name == "length_outlier":
            assert len(lengths) < len(c[name])
        else:
            assert lengths.count(6000) >= 3, (name, lengths)


def test_trim_dir_emu(emu, tmp_path):
    untrimmed = _cluster_gfa(tmp_path, _clusters()["circular_overlaps"])
    d = tmp_path / "cluster_001"
    d.mkdir()
    (d / "1_untrimmed.gfa").write_text(untrimmed)
    api.trim(str(d), lib=emu)
    want_gfa, want_yaml = T.trim_gfa(untrimmed)
    assert (d / "2_trimmed.gfa").read_text() == want_gfa
    assert (d / "2_trimmed.yaml").read_text() == want_yaml


@pytest.mark.parametrize("kw,message", [
    (dict(min_identity=1.5), "--min_identity must be between 0.0 and 1 (inclusive)"),
    (dict(min_identity=-0.1), "--min_identity must be between 0.0 and 1 (inclusive)"),
    (dict(threads=0), "--threads cannot be less than 1"),
    (dict(threads=101), "--threads cannot be greater than 100"),
    (dict(mad=-1.0), "--mad cannot be less than 0"),
])
def test_trim_dir_settings(emu, tmp_path, kw, message):
    (tmp_path / "1_untrimmed.gfa").write_text("H\tVN:Z:1.0\tKM:i:51\n")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.trim(str(tmp_path), lib=emu, **kw)
    assert e.value.code == -6 and e.value.message == message


def test_trim_dir_missing_input(emu, tmp_path):
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.trim(str(tmp_path / "nope"), lib=emu)
    assert e.value.code == -6 and e.value.message == f"directory does not exist: {tmp_path / 'nope'}"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.trim(str(tmp_path), lib=emu)
    assert e.value.code == -6 and e.value.message == f"file does not exist: {tmp_path / '1_untrimmed.gfa'}"


def test_empty_cluster_yaml():
    assert T.metrics_yaml([]) == "trimmed_cluster_size: 0\ntrimmed_cluster_lengths: []\ntrimmed_cluster_median: 0\ntrimmed_cluster_mad: 0\n"


def test_trimmed_depths_are_counts(emu, tmp_path):
    untrimmed = _cluster_gfa(tmp_path, _clusters()["circular_overlaps"])
    g, _ = api.UnitigGraph.from_gfa_lines(untrimmed.encode(), lib=emu)
    g.trim()
    for u in g.unitigs():
        assert u["depth"] == int(u["depth"]) and u["depth"] >= 1


# ---- on the H100 ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("settings", CLUSTER_SETTINGS)
@pytest.mark.parametrize("name", sorted(_clusters()))
def test_cluster_gpu(gpu, tmp_path, name, settings):
    _check_cluster(gpu, tmp_path, name, settings)


@pytest.mark.gpu
def test_window_beyond_shared_memory_gpu(gpu):
    """A window of more than the ~9,650 unitigs whose three diagonals fit a CTA's shared memory keeps them in HBM."""
    rng = random.Random(7)
    n_units = 12000
    w = {u: rng.randint(1, 3) * 10 for u in range(1, n_units + 1)}
    core = list(range(1, n_units + 1))
    rng.shuffle(core)
    path = core + core[:50]
    mu = len(path)
    got = api.trim_path_start_end([path, path[:200] + path[:20]], w, 0.75, mu, lib=gpu)
    assert got[0] == T.trim_path_start_end(path, w, 0.75, mu)
    assert got[1] == T.trim_path_start_end(path[:200] + path[:20], w, 0.75, mu)


@pytest.mark.gpu
def test_cli_trim_gpu(tmp_path):
    untrimmed = _cluster_gfa(tmp_path, _clusters()["hairpin"])
    d = tmp_path / "cluster_001"
    d.mkdir()
    (d / "1_untrimmed.gfa").write_text(untrimmed)
    r = subprocess.run([os.path.join(ROOT, "autocycler_b200", "bin", "autocycler"), "trim", "-c", str(d)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    want_gfa, want_yaml = T.trim_gfa(untrimmed)
    assert (d / "2_trimmed.gfa").read_text() == want_gfa
    assert (d / "2_trimmed.yaml").read_text() == want_yaml
    r = subprocess.run([os.path.join(ROOT, "autocycler_b200", "bin", "autocycler"), "trim", "-c", str(d), "--mad", "-1"], capture_output=True, text=True)
    assert r.returncode == 1 and "Error: --mad cannot be less than 0" in r.stderr


@pytest.mark.gpu
def test_determinism_gpu(gpu, tmp_path):
    untrimmed = _cluster_gfa(tmp_path, _clusters()["circular_overlaps"])
    g, _ = api.UnitigGraph.from_gfa_lines(untrimmed.encode(), lib=gpu)
    g.trim()
    first = bytes(g.gfa_bytes())
    g._h.check(g._h.lib.ac_load_gfa(g._h.ptr, untrimmed.encode(), len(untrimmed)))
    g.trim()
    assert bytes(g.gfa_bytes()) == first


@pytest.mark.gpu
def test_cfg2_trim_gpu():
    """cfg2's compress GFA through merge_linear_paths (what cluster writes for a one-cluster genome), trimmed on the GPU, against
    the SHA-256 of the oracle's 2_trimmed.gfa (tests/golden/trim_goldens.json, made by make_trim_goldens.py)."""
    import tempfile
    from autocycler_b200 import synth
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "trim_goldens.json")))["cfg2_k51_trim_mu5000"]["sha256"]
    with tempfile.TemporaryDirectory() as d:
        synth.write_assemblies(synth.make_assemblies("cfg2"), d)
        kg, _, _ = api.load_sequences(d, 51)
        kg.upload()
        g = api.UnitigGraph.compress(kg)
        api.merge_linear_paths(g, seqs=[1])
        untrimmed = bytes(g.gfa_bytes())
    g2, _ = api.UnitigGraph.from_gfa_lines(untrimmed)
    g2.trim()
    assert hashlib.sha256(bytes(g2.gfa_bytes())).hexdigest() == want
