"""`autocycler trim -c DIR...` and `autocycler resolve -c DIR...`: several clusters in one call, every device round shared by all of
them.  Every directory's files equal a single-directory call's byte for byte, the reports equal the single calls' except for the
kernel time and one closing line, errors write nothing, and the launches do not grow with the number of clusters."""
import os
import random
import re
import shutil
import subprocess

import pytest

from autocycler_b200 import api, synth
import resolve_oracle as R
import trim_oracle as T
from test_resolve import _cluster_text, _synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
TRIM_OUT = ("2_trimmed.gfa", "2_trimmed.yaml")
RESOLVE_OUT = ("3_bridged.gfa", "4_merged.gfa", "5_final.gfa")
BANNER = api.VERBOSE_REPORT | api.VERBOSE_BANNER


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


# ---- cluster directories ------------------------------------------------------------------------------------------------------------

def _seq(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def _pass_clusters(lib, tmp, config, lengths=None, n_assemblies=None):
    """compress -> cluster of a seeded synthetic config; -> the qc_pass cluster directories, in order."""
    asm = synth.make_assemblies(config, replicon_lengths=lengths, n_assemblies=n_assemblies)
    synth.write_assemblies(asm, str(tmp / "asm"))
    api.compress(str(tmp / "asm"), str(tmp / "ac"), lib=lib)
    api.cluster(str(tmp / "ac"), lib=lib)
    dirs = sorted((tmp / "ac" / "clustering" / "qc_pass").iterdir())
    assert len(dirs) > 1
    return dirs


def _write_dirs(root, name, texts):
    """One directory per text under root, holding it as `name`; -> the directories."""
    dirs = []
    for i, t in enumerate(texts):
        d = root / f"cluster_{i + 1:03d}"
        d.mkdir(parents=True)
        (d / name).write_text(t)
        dirs.append(d)
    return dirs


def _copy(dirs, root):
    root.mkdir(parents=True)
    out = []
    for d in dirs:
        shutil.copytree(d, root / d.name)
        out.append(root / d.name)
    return out


def _files(dirs, names):
    return [tuple((d / n).read_bytes() for n in names) for d in dirs]


def _snapshot(dirs):
    return [sorted((p.name, p.stat().st_mtime_ns, p.stat().st_size) for p in d.iterdir()) for d in dirs]


_MS = re.compile(r", (alignment|distance) kernels [0-9.]+ ms")


def _batched_equals_singles(lib, dirs, tmp, capfd, command, **kw):
    """Runs every directory alone (in a copy) and all of them in one batched call; the files and the reports must agree.  -> batch info."""
    single, batch = _copy(dirs, tmp / "single"), _copy(dirs, tmp / "batch")
    fn, names = (api.trim_dirs, TRIM_OUT) if command == "trim" else (api.resolve_dirs, RESOLVE_OUT)
    capfd.readouterr()
    for d in single:
        fn([str(d)], verbose=BANNER, lib=lib, **kw)
    want_err = capfd.readouterr().err
    info = fn([str(d) for d in batch], verbose=BANNER, lib=lib, **kw)
    got_err = capfd.readouterr().err
    assert _files(batch, names) == _files(single, names)
    body, last = got_err.rstrip("\n").rsplit("\n", 1)
    verb = "Trimmed" if command == "trim" else "Resolved"
    assert re.fullmatch(rf"{verb} {len(dirs)} clusters: {info['launches']} kernel launches, {info['jobs']} (alignments|distance jobs), "
                        rf"{info['cells']} DP cells, (alignment|distance) kernels [0-9.]+ ms", last), last
    assert body + "\n" == _MS.sub("", want_err).replace(str(tmp / "single"), str(tmp / "batch"))
    assert info["clusters"] == len(dirs)
    assert info["launches"] <= (4 if command == "trim" else 2)
    return info


# ---- batched equals single, on the emulation build ----------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cfg3_small(emu, tmp_path_factory):
    """cfg3's six replicons and twelve assemblies, each replicon shortened so that the emulation build compresses it in seconds."""
    return _pass_clusters(emu, tmp_path_factory.mktemp("cfg3"), "cfg3", lengths=[40_000, 16_000, 9_000, 7_000, 5_000, 3_000])


def test_cfg3_pass_clusters_emu(emu, cfg3_small, tmp_path, capfd):
    t = _batched_equals_singles(emu, cfg3_small, tmp_path / "t", capfd, "trim")
    assert t["jobs"] > 0 and t["cells"] > 0
    trimmed = [tmp_path / "t" / "batch" / d.name for d in cfg3_small]
    for d in trimmed:
        assert tuple((d / n).read_text() for n in TRIM_OUT) == T.trim_gfa((d / "1_untrimmed.gfa").read_text())
    r = _batched_equals_singles(emu, trimmed, tmp_path / "r", capfd, "resolve")
    assert r["clusters"] == len(cfg3_small)
    for d in cfg3_small:
        got = tmp_path / "r" / "batch" / d.name
        assert tuple((got / n).read_text() for n in RESOLVE_OUT) == R.resolve_gfa((got / "2_trimmed.gfa").read_text())
    # combine over the batched finals equals combine over the single calls' finals
    outs = []
    for arm in ("single", "batch"):
        a = tmp_path / f"combine_{arm}"
        api.combine(str(a), [str(tmp_path / "r" / arm / d.name / "5_final.gfa") for d in cfg3_small], lib=emu)
        outs.append(tuple((a / f"consensus_assembly.{e}").read_bytes() for e in ("gfa", "fasta", "yaml")))
    assert outs[0] == outs[1]


def test_synthetic_resolve_clusters_emu(emu, tmp_path, capfd):
    dirs = _write_dirs(tmp_path / "in", "2_trimmed.gfa", list(_synthetic().values()))
    _batched_equals_singles(emu, dirs, tmp_path, capfd, "resolve")
    for d in _copy(dirs, tmp_path / "oracle"):
        api.resolve(str(d), lib=emu)
        assert tuple((d / n).read_text() for n in RESOLVE_OUT) == R.resolve_gfa((d / "2_trimmed.gfa").read_text())


def test_synthetic_trim_clusters_emu(emu, tmp_path, capfd):
    """Resolve's synthetic clusters as untrimmed graphs: hairpins, circular paths and untrimmable ones together, under four settings."""
    texts = list(_synthetic().values())
    dirs = _write_dirs(tmp_path / "in", "1_untrimmed.gfa", texts)
    for kw in ({}, {"max_unitigs": 3}, {"max_unitigs": 0}, {"mad": 0.0, "min_identity": 0.5}):
        _batched_equals_singles(emu, dirs, tmp_path / str(len(os.listdir(tmp_path))), capfd, "trim", **kw)


def test_single_dir_equals_ac_dir_emu(emu, cfg3_small, tmp_path):
    a, b = _copy(cfg3_small[:1], tmp_path / "a"), _copy(cfg3_small[:1], tmp_path / "b")
    api.trim(str(a[0]), lib=emu)
    info = api.trim_dirs([str(b[0])], lib=emu)
    assert _files(a, TRIM_OUT) == _files(b, TRIM_OUT) and info["clusters"] == 1
    api.resolve(str(a[0]), lib=emu)
    info = api.resolve_dirs([str(b[0])], lib=emu)
    assert _files(a, RESOLVE_OUT) == _files(b, RESOLVE_OUT) and info["clusters"] == 1


# ---- the weight tables are the clusters' own ----------------------------------------------------------------------------------------

def _planted_trim(heavy_overlap):
    """Two sequences whose paths end in (1, 9) and start with (1, 2): the start-end overlap matches unitig 1 and mismatches 9 against 2.
    With unitig 1 long the overlap passes the identity test and the sequences are trimmed; with 2 and 9 long it fails."""
    rng = random.Random(3)
    long_, short = (3000, 40) if heavy_overlap else (40, 3000)
    lens = {1: long_, 2: short, 9: short, **{u: 500 for u in range(3, 9)}}
    segs = {u: _seq(rng, lens[u]) for u in range(1, 10)}
    return _cluster_text(segs, [[1, 2, 3, 4, 5, 6, 7, 8, 1, 9], [1, 2, 3, 4, 5, 6, 7, 8, 1, 9]])


def _planted_resolve(x_short):
    """Anchors 1 and 2, three bridge paths (3), (4, 5) and (6).  Whichever of 3 and 6 is short is closer to (4, 5) and is the best path."""
    rng = random.Random(4)
    lens = {1: 300, 2: 300, 3: 10 if x_short else 1000, 4: 500, 5: 500, 6: 1000 if x_short else 10}
    segs = {u: _seq(rng, lens[u]) for u in range(1, 7)}
    return _cluster_text(segs, [[1, 3, 2], [1, 4, 5, 2], [1, 6, 2]])


def test_planted_weights_emu(emu, tmp_path, capfd):
    trim_texts = [_planted_trim(True), _planted_trim(False)]
    singles = []
    for i, t in enumerate(trim_texts):
        d = _write_dirs(tmp_path / f"t{i}", "1_untrimmed.gfa", [t])
        api.trim(str(d[0]), lib=emu)
        singles.append((d[0] / "2_trimmed.yaml").read_text())
        assert singles[-1] + (d[0] / "2_trimmed.gfa").read_text() == "".join(reversed(T.trim_gfa(t)))
    # only the first one trims: 9,080 bp untrimmed, 6,040 bp without the repeated (1, 9)
    assert "trimmed_cluster_lengths:\n- 6040\n- 6040\n" in singles[0] and "trimmed_cluster_lengths:\n- 9080\n- 9080\n" in singles[1]
    res_texts = [_planted_resolve(True), _planted_resolve(False)]
    bests = [R.resolve_gfa(t)[2] for t in res_texts]
    assert "\n".join(l for l in bests[0].splitlines() if l.startswith("S")) != "\n".join(l for l in bests[1].splitlines() if l.startswith("S"))
    for order in ((0, 1), (1, 0)):
        root = tmp_path / f"order{order[0]}{order[1]}"
        dirs = _write_dirs(root / "trim", "1_untrimmed.gfa", [trim_texts[i] for i in order])
        _batched_equals_singles(emu, dirs, root / "t", capfd, "trim")
        dirs = _write_dirs(root / "resolve", "2_trimmed.gfa", [res_texts[i] for i in order])
        _batched_equals_singles(emu, dirs, root / "r", capfd, "resolve")
        api.resolve_dirs([str(d) for d in dirs], lib=emu)
        assert [(d / "5_final.gfa").read_text() for d in dirs] == [bests[i] for i in order]


# ---- errors: the single call's, and nothing written -----------------------------------------------------------------------------------

def _error(fn):
    with pytest.raises(api.AutocyclerGpuError) as e:
        fn()
    return e.value.code, e.value.message


def _four(tmp, name, text):
    return _write_dirs(tmp, name, [text] * 4)


@pytest.mark.parametrize("command", ["trim", "resolve"])
def test_errors_write_nothing_emu(emu, tmp_path, command):
    name = "1_untrimmed.gfa" if command == "trim" else "2_trimmed.gfa"
    fn = (lambda ds, **kw: api.trim_dirs([str(d) for d in ds], lib=emu, **kw)) if command == "trim" else \
         (lambda ds, **kw: api.resolve_dirs([str(d) for d in ds], lib=emu, **kw))
    one = (lambda d, **kw: api.trim(str(d), lib=emu, **kw)) if command == "trim" else (lambda d, **kw: api.resolve(str(d), lib=emu, **kw))
    text = list(_synthetic().values())[0]
    cases = []
    # a missing input in the third of four directories
    dirs = _four(tmp_path / "missing", name, text)
    (dirs[2] / name).unlink()
    cases.append((dirs, dirs, dirs[2], {}))
    # a malformed GFA in the last directory
    dirs = _four(tmp_path / "malformed", name, text)
    (dirs[3] / name).write_text("S\t1\tACGT\nP\tbroken\n")
    cases.append((dirs, dirs, dirs[3], {}))
    # the same directory twice, by the same path and by another path to it
    dirs = _four(tmp_path / "twice", name, text)
    cases.append((dirs, dirs + [dirs[1]], dirs[1], "twice"))
    other = dirs[0].parent / ".." / dirs[0].parent.name / dirs[0].name
    cases.append((dirs, dirs[:2] + [other] + dirs[2:], other, "twice"))
    if command == "trim":   # a bad setting: the first directory's error
        dirs = _four(tmp_path / "setting", name, text)
        cases.append((dirs, dirs, dirs[0], {"min_identity": 1.5}))
    for dirs, args, failing, kw in cases:
        before = _snapshot(dirs)
        got = _error(lambda: fn(args, **(kw if kw != "twice" else {})))
        assert _snapshot(dirs) == before
        if kw == "twice":
            assert got == (-6, f"cluster directory given twice: {failing}")
        else:
            assert got == _error(lambda: one(failing, **kw))
            assert _snapshot(dirs) == before


# ---- the command line -----------------------------------------------------------------------------------------------------------------

def test_cli_cluster_dir_values(tmp_path):
    """-c takes every value up to the next flag; with no value its message is unchanged.  Runs before any device work."""
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc")], check=True)
    for d in ("a", "b", "c"):
        (tmp_path / d).mkdir()
    a, b, c = (str(tmp_path / d) for d in "abc")
    r = subprocess.run([AUTOCYCLER, "trim", "-c", a, b, c], capture_output=True, text=True)
    assert r.returncode == 1 and r.stderr.endswith(f"\nError: file does not exist: {a}/1_untrimmed.gfa\n"), r.stderr
    r = subprocess.run([AUTOCYCLER, "trim", "-c", a, b, "--mad", "2", "--max_unitigs", "7"], capture_output=True, text=True)
    assert r.returncode == 1 and "  --max_unitigs 7\n  --mad 2\n" in r.stderr and r.stderr.count("Starting autocycler trim") == 1, r.stderr
    r = subprocess.run([AUTOCYCLER, "resolve", "-c", a, b, "--verbose"], capture_output=True, text=True)
    assert r.returncode == 1 and r.stderr.endswith(f"\nError: file does not exist: {a}/2_trimmed.gfa\n"), r.stderr
    for command in ("trim", "resolve"):
        r = subprocess.run([AUTOCYCLER, command, "-c"], capture_output=True, text=True)
        assert r.returncode == 2 and r.stderr == "error: a value is required for '-c'\n"
        r = subprocess.run([AUTOCYCLER, command, "-c", a, "-x"], capture_output=True, text=True)
        assert r.returncode == 2 and r.stderr.startswith("error: unexpected argument '-x'\n")


def test_launches_do_not_grow_emu(emu, tmp_path):
    texts = list(_synthetic().values())
    for n in (1, 2, 8, 24):
        dirs = _write_dirs(tmp_path / f"t{n}", "1_untrimmed.gfa", [texts[i % len(texts)] for i in range(n)])
        t = api.trim_dirs([str(d) for d in dirs], lib=emu)
        assert t["clusters"] == n and 0 < t["launches"] <= 4
        for d in dirs:
            (d / "2_trimmed.gfa").write_text((d / "1_untrimmed.gfa").read_text())
        r = api.resolve_dirs([str(d) for d in dirs], lib=emu)
        assert r["clusters"] == n and 0 < r["launches"] <= 2 and r["buffer_bytes"] > 0


# ---- on the H100 ----------------------------------------------------------------------------------------------------------------------

def _gpu_batch_equals_singles(gpu, dirs, tmp, command, **kw):
    single, batch = _copy(dirs, tmp / "single"), _copy(dirs, tmp / "batch")
    fn, one, names = (api.trim_dirs, api.trim, TRIM_OUT) if command == "trim" else (api.resolve_dirs, api.resolve, RESOLVE_OUT)
    for d in single:
        one(str(d), lib=gpu, **kw)
    info = fn([str(d) for d in batch], lib=gpu, **kw)
    assert _files(batch, names) == _files(single, names)
    assert info["launches"] <= (4 if command == "trim" else 2)
    return batch, info


@pytest.mark.gpu
def test_cfg3_pass_clusters_gpu(gpu, tmp_path):
    """cfg3 at full size: the batch against the single-directory GPU calls, the CLI batch against the shell loop, and combine."""
    dirs = _pass_clusters(gpu, tmp_path / "chain", "cfg3")
    trimmed, _ = _gpu_batch_equals_singles(gpu, dirs, tmp_path / "t", "trim")
    _gpu_batch_equals_singles(gpu, trimmed, tmp_path / "r", "resolve")
    loop, cli = _copy(dirs, tmp_path / "loop"), _copy(dirs, tmp_path / "cli")
    for d in loop:
        for command in ("trim", "resolve"):
            assert subprocess.run([AUTOCYCLER, command, "-c", str(d)], capture_output=True).returncode == 0
    for command in ("trim", "resolve"):
        r = subprocess.run([AUTOCYCLER, command, "-c", *map(str, cli)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    assert _files(cli, TRIM_OUT + RESOLVE_OUT) == _files(loop, TRIM_OUT + RESOLVE_OUT)
    outs = []
    for arm in (loop, cli):
        a = arm[0].parent / "combined"
        assert subprocess.run([AUTOCYCLER, "combine", "-a", str(a), "-i", *[str(d / "5_final.gfa") for d in arm]], capture_output=True).returncode == 0
        outs.append(tuple((a / f"consensus_assembly.{e}").read_bytes() for e in ("gfa", "fasta", "yaml")))
    assert outs[0] == outs[1]


@pytest.mark.gpu
def test_small_chain_against_oracles_gpu(gpu, tmp_path):
    dirs = _pass_clusters(gpu, tmp_path / "chain", "cfg3", lengths=[40_000, 16_000, 9_000, 7_000, 5_000, 3_000])
    trimmed, _ = _gpu_batch_equals_singles(gpu, dirs, tmp_path / "t", "trim")
    for d in trimmed:
        assert tuple((d / n).read_text() for n in TRIM_OUT) == T.trim_gfa((d / "1_untrimmed.gfa").read_text())
    resolved, _ = _gpu_batch_equals_singles(gpu, trimmed, tmp_path / "r", "resolve")
    for d in resolved:
        assert tuple((d / n).read_text() for n in RESOLVE_OUT) == R.resolve_gfa((d / "2_trimmed.gfa").read_text())


@pytest.mark.gpu
def test_window_beyond_shared_memory_batch_gpu(gpu, tmp_path):
    """A start-end window of 12,050 unitigs (beyond the ~9,681 whose diagonals fit shared memory) next to small clusters: both launch
    forms in each round, and every cluster's files as its own call writes them."""
    rng = random.Random(7)
    n_units = 12000
    segs = {u: _seq(rng, rng.randint(1, 3) * 10) for u in range(1, n_units + 1)}
    core = list(range(1, n_units + 1))
    rng.shuffle(core)
    big = _cluster_text(segs, [core + core[:50], core + core[:50]])
    texts = [big] + list(_synthetic().values())[:4]
    dirs = _write_dirs(tmp_path / "in", "1_untrimmed.gfa", texts)
    _, info = _gpu_batch_equals_singles(gpu, dirs, tmp_path / "a", "trim", max_unitigs=12100)
    assert info["launches"] == 4


@pytest.mark.gpu
def test_long_bridge_batch_gpu(gpu, tmp_path):
    """A bridge whose paths have 20,500 unitigs (diagonals in HBM scratch) next to dense small bridges, in one resolve batch."""
    rng = random.Random(11)
    n = 20_500
    segs = {u: _seq(rng, rng.randint(5, 40)) for u in range(1, 2 * n + 3)}
    p, q = list(range(3, n + 3)), list(range(n + 3, 2 * n + 3))
    long_ = _cluster_text(segs, [[1] + p + [2], [1] + q + [2], [1] + p[:n // 2] + q[n // 2:] + [2]])
    texts = [long_] + list(_synthetic().values())
    dirs = _write_dirs(tmp_path / "in", "2_trimmed.gfa", texts)
    _, info = _gpu_batch_equals_singles(gpu, dirs, tmp_path / "a", "resolve")
    assert info["launches"] == 2 and info["jobs"] > 3


@pytest.mark.gpu
def test_determinism_gpu(gpu, tmp_path):
    texts = list(_synthetic().values())
    outs = []
    for run in range(2):
        dirs = _write_dirs(tmp_path / f"run{run}", "1_untrimmed.gfa", texts)
        api.trim_dirs([str(d) for d in dirs], lib=gpu)
        api.resolve_dirs([str(d) for d in dirs], lib=gpu)
        outs.append(_files(dirs, TRIM_OUT + RESOLVE_OUT))
    assert outs[0] == outs[1]
