"""`autocycler resolve` (resolve.rs) and `autocycler combine` (combine.rs): the reference's unit-test data (tests/golden/resolve_kats.json,
extracted from resolve.rs:517-702), seeded random bridges, the reference's GFA fixtures, synthetic clusters and the whole chain, each
checked against the CPU oracle (tests/resolve_oracle.py).  The CPU tests run the product's code through the host-emulation library (the
distance kernel's diagonal sweep and per-cell body, serially); the tests marked gpu run the CUDA build on the H100."""
import glob
import hashlib
import json
import os
import random
import subprocess

import pytest

import cluster_oracle
import resolve_oracle as R
import trim_oracle
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "resolve_kats.json")))["cases"]
FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "ref_test_gfa_*.gfa")))
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def _w(case):
    return {int(u): w for u, w in case["weights"].items()}


# ---- the reference's KATs ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", KATS, ids=[f"{c['test']}-{i}" for i, c in enumerate(KATS)])
def test_kats_oracle(case):
    k = case["kind"]
    if k == "distance":
        assert R.global_alignment_distance(case["a"], case["b"], _w(case)) == case["expected"]
    elif k == "best_path":
        assert R.Bridge(case["start"], case["end"], case["paths"], _w(case)).best_path == case["expected"]
    elif k.startswith("bridge_"):
        b = R.Bridge(case["start"], case["end"], case["paths"], _w(case))
        assert {"bridge_rev_start": b.rev_start(), "bridge_rev_end": b.rev_end(), "bridge_depth": b.depth()}[k] == case["expected"]
    elif k == "ambiguity":
        bridges = [R.Bridge(b["start"], b["end"], b["paths"], _w(case)) for b in case["bridges"]]
        R.determine_ambiguity(bridges)
        assert [b.conflicting for b in bridges] == case["expected"]
    elif k == "anchor_to_anchor":
        assert R.get_anchor_to_anchor_paths(case["sequence_paths"], set(case["anchor_set"])) == case["expected"]
    elif k == "group":
        assert R.group_paths_by_start_end(case["paths"]) == {tuple(a): b for a, b in case["expected"]}
    else:
        raise AssertionError(k)


def _product_kats(lib):
    n = 0
    for case in KATS:
        if case["kind"] == "distance":           # a group of the two paths: both totals are D(a, b)
            totals, _ = api.bridge_best_paths([[case["a"], case["b"]]], _w(case), lib=lib)
            assert totals[0] == [case["expected"]] * 2, case["test"]
            n += 1
        elif case["kind"] == "best_path":
            _, best = api.bridge_best_paths([[p[1:-1] for p in case["paths"]]], _w(case), lib=lib)
            assert best == [case["expected"]], case["test"]
            n += 1
    assert n == 15


def test_kats_emu(emu):
    _product_kats(emu)


@pytest.mark.gpu
def test_kats_gpu(gpu):
    _product_kats(gpu)


# ---- seeded random bridges --------------------------------------------------------------------------------------------------------

def _random_groups(seed, big_weights=False, long_paths=0):
    """Groups of 1..40 paths with planted duplicates, ties (equal weights) and empty paths; big_weights: lengths up to 2^31, which wrap
    the u32 DP and the totals."""
    rng = random.Random(seed)
    n_units = rng.randint(2, 30) if not long_paths else long_paths + 50
    if big_weights:
        w = {u: rng.choice([2 ** 31, 2 ** 31 - 1, rng.randint(2 ** 30, 2 ** 31), rng.randint(1, 100)]) for u in range(1, n_units + 1)}
    else:
        w = {u: rng.choice([1, 10, 10, 10, rng.randint(1, 5000)]) for u in range(1, n_units + 1)}
    groups = []
    for _ in range(rng.randint(1, 4)):
        P = rng.randint(1, 40)
        base = [rng.choice([1, -1]) * rng.randint(1, n_units) for _ in range(long_paths or rng.randint(0, 12))]
        paths = []
        for _ in range(P):
            r = rng.random()
            if r < 0.3 and paths:
                paths.append(list(rng.choice(paths)))            # a duplicate
            elif r < 0.4:
                paths.append([])
            else:
                p = list(base)
                for _ in range(rng.choice([0, 1, 2, 3])):
                    x = rng.randrange(len(p) + 1)
                    if rng.random() < 0.5 and p:
                        del p[min(x, len(p) - 1)]
                    else:
                        p.insert(x, rng.choice([1, -1]) * rng.randint(1, n_units))
                paths.append(p)
        groups.append(paths)
    return groups, w


def _oracle_groups(groups, w):
    out_t, out_b = [], []
    for g in groups:
        b = R.Bridge(1, 2, [[1] + p + [2] for p in g], w)
        out_t.append(b.totals)
        out_b.append(b.best_path)
    return out_t, out_b


def _check_random(lib, seeds, **kw):
    for s in seeds:
        groups, w = _random_groups(s, **kw)
        assert api.bridge_best_paths(groups, w, lib=lib) == _oracle_groups(groups, w), s


def test_random_bridges_emu(emu):
    _check_random(emu, range(60))


def test_random_bridges_wraparound_emu(emu):
    _check_random(emu, range(100, 140), big_weights=True)


def test_row_dp_equals_cells():
    """The vectorised DP (golden generation only) against the literal one, where no sum can wrap."""
    for s in range(200):
        groups, w = _random_groups(s)
        for g in groups:
            for a in g[:4]:
                for b in g[:4]:
                    assert R.global_alignment_distance_rows(a, b, w) == R.global_alignment_distance_cells(a, b, w)


@pytest.mark.gpu
def test_random_bridges_gpu(gpu):
    _check_random(gpu, range(60))
    _check_random(gpu, range(100, 140), big_weights=True)


@pytest.mark.gpu
def test_paths_beyond_shared_memory_gpu(gpu):
    """Rows of more than the ~19,000 unitigs whose three diagonals fit a CTA's shared memory keep them in HBM scratch; a shorter
    group in the same call runs in shared memory.  The long group's weights keep every sum below 2^32, so the oracle's row form of the
    DP (checked against the cell form in test_row_dp_equals_cells) computes it."""
    rng = random.Random(11)
    n = 20_500
    w = {u: rng.randint(1, 1000) for u in range(1, n + 60)}
    base = [rng.choice([1, -1]) * u for u in range(1, n + 1)]
    paths = []
    for k in range(3):
        p = list(base)
        for _ in range(5):
            p[rng.randrange(n)] = rng.randint(n + 1, n + 59)
        paths.append(p)
    small = [p[:300] + [n + 1 + k] for k, p in enumerate(paths)]
    h = api._Handle(gpu, 51)
    got = api.bridge_best_paths([paths + [paths[0]], small], w, lib=gpu, handle=h)
    info = api.AcResolveInfo()
    h.check(gpu.ac_resolve_stats(h.ptr, info))
    assert info.hbm_jobs == 3 and info.shared_jobs == 3
    R.FAST_DP = True
    try:
        want = _oracle_groups([paths + [paths[0]], small], w)
    finally:
        R.FAST_DP = False
    assert got == want


# ---- whole resolves ---------------------------------------------------------------------------------------------------------------

def _seq(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def _cluster_text(segs, paths, extra_links=(), headers=None, ids=None):
    """A 2_trimmed.gfa: segments {number: sequence}, paths of signed numbers (one sequence each), links from the paths' steps (and
    extra_links) with their mirrors, depths = path steps through each unitig."""
    depth = {n: 0 for n in segs}
    links = []

    def add(a, b):
        for x in ((a, b), (-b, -a)):
            if x not in links:
                links.append(x)
    for p in paths:
        for s in p:
            depth[abs(s)] += 1
        for a, b in zip(p, p[1:]):
            add(a, b)
    for a, b in extra_links:
        add(a, b)
    out = ["H\tVN:Z:1.0\tKM:i:51"]
    for n, s in segs.items():
        out.append(f"S\t{n}\t{s}\tDP:f:{depth[n] or 1}.00")
    for a, b in links:
        out.append(f"L\t{abs(a)}\t{'+' if a > 0 else '-'}\t{abs(b)}\t{'+' if b > 0 else '-'}\t0M")
    for i, p in enumerate(paths):
        hd = (headers or {}).get(i, f"c{i}")
        sid = (ids or {}).get(i, i + 1)
        out.append(f"P\t{sid}\t{','.join(f'{abs(s)}{chr(43) if s > 0 else chr(45)}' for s in p)}\t*\tLN:i:{sum(len(segs[abs(s)]) for s in p)}"
                   f"\tFN:Z:a{i}.fasta\tHD:Z:{hd}")
    return "\n".join(out) + "\n"


def _synthetic():
    rng = random.Random(5)
    segs = {n: _seq(rng, rng.choice([30, 60, 120, 400])) for n in range(1, 31)}
    cases = {}
    # A, B, C anchors; the bridges carry alternative middles, consensus weights 0, 1 and 3
    cases["weights"] = _cluster_text(segs, [[1, 4, 5, 2, 6, 3], [1, 7, 2, 6, 3], [1, 4, 5, 2, 8, 3], [1, 7, 2, 8, 3]],
                                     headers={0: "c0 autocycler_consensus_weight=3", 1: "c1 Autocycler_consensus_weight=0", 3: "c3 x"})
    # the anchors come in different orders: conflicting bridges, culling and the second pass
    cases["conflicts"] = _cluster_text(segs, [[1, 4, 2, 5, 3, 6], [1, 4, 2, 5, 3, 6], [1, 7, 3, 8, 2, 9]])
    # a component nobody's path touches is deleted; a second one without an anchor too
    cases["anchor_free"] = _cluster_text(segs, [[1, 4, 2, -3], [1, 5, 2, -3]], extra_links=[(20, 21), (21, 22)])
    cases["zero_anchors"] = _cluster_text(segs, [[1, 2, 3, 1], [4, 5, 6], [7, 1, 8]])
    cases["single_anchor"] = _cluster_text(segs, [[1, 2, 3], [4, 2, 5], [2, 6]])
    # two sequences share an id: unitig 1 occurs twice in one of them, once per strand, and is an anchor; its bridge runs 1 -> -1
    cases["hairpin"] = _cluster_text(segs, [[1, 2, 3, -2, -1], [4, 5]], ids={1: 1})
    cases["circular"] = _cluster_text(segs, [[1, 4, 2, 5, 3, 6, 1], [2, 5, 3, 7, 1, 4, 2]])
    cases["reverse"] = _cluster_text(segs, [[1, 4, 2, 5, 3], [-3, -5, -2, -9, -1], [1, 4, 2, 10, 3]])
    return cases


def _fixture_texts():
    return {os.path.basename(f): open(f).read() for f in FIXTURES}


def _check_resolve(lib, text):
    want = R.resolve_gfa(text)
    g, _ = api.UnitigGraph.from_gfa_lines(text.encode(), lib=lib)
    before = bytes(g.gfa_bytes())
    g.resolve()
    got = (g.resolve_text("bridged"), g.resolve_text("merged"), g.resolve_text("final"))
    assert got == want
    assert bytes(g.gfa_bytes()) == before
    return want


@pytest.mark.parametrize("name", sorted(_fixture_texts()))
def test_fixtures_emu(emu, name):
    _check_resolve(emu, _fixture_texts()[name])


@pytest.mark.parametrize("name", sorted(_synthetic()))
def test_synthetic_emu(emu, tmp_path, name):
    text = _synthetic()[name]
    _check_resolve(emu, text)
    (tmp_path / "2_trimmed.gfa").write_text(text)
    api.resolve(str(tmp_path), lib=emu)
    want = R.resolve_gfa(text)
    assert tuple((tmp_path / f).read_text() for f in ("3_bridged.gfa", "4_merged.gfa", "5_final.gfa")) == want


def test_synthetic_cases_do_what_they_say():
    """The oracle's own view of the synthetic clusters."""
    c = _synthetic()
    info = {}
    for name in c:
        info[name] = {}
        R.resolve_gfa(c[name], info[name])
    assert info["conflicts"]["culled"] > 0
    assert info["zero_anchors"]["anchors"] == 0 and info["single_anchor"]["anchors"] == 1
    assert info["weights"]["bridges"] == 2 and info["hairpin"]["bridges"] >= 1
    g = R.Graph(c["hairpin"])
    anchors = R.find_anchors(g)
    assert 1 in anchors and any(b.start == -b.end for b in R.create_bridges(g, anchors))
    _, merged, _ = R.resolve_gfa(c["anchor_free"])
    assert "\t20\t" not in merged and all(len(ln.split("\t")[2]) != len(_synthetic_segs()[20]) for ln in merged.splitlines() if ln.startswith("S"))


def _synthetic_segs():
    rng = random.Random(5)
    return {n: _seq(rng, rng.choice([30, 60, 120, 400])) for n in range(1, 31)}


def test_hairpin_bridge_conflicts_with_itself():
    """determine_ambiguity counts start and rev_start in one map: start == -end conflicts with itself."""
    b = R.Bridge(3, -3, [[3, 5, -3]], {3: 10, 5: 10})
    assert R.determine_ambiguity([b]) == 1 and b.conflicting


# ---- combine ----------------------------------------------------------------------------------------------------------------------

def test_combine_emu(emu, tmp_path):
    texts = [R.resolve_gfa(t)[2] for t in list(_synthetic().values())[:4]] + [_fixture_texts()["ref_test_gfa_9.gfa"], "H\tVN:Z:1.0\n"]
    names = []
    for i, t in enumerate(texts):
        p = tmp_path / f"c{i}.gfa"
        p.write_text(t)
        names.append(str(p))
    out = tmp_path / "out" / "nested"
    api.combine(str(out), names, lib=emu)
    want = R.combine_gfas(texts)
    got = tuple((out / f"consensus_assembly.{e}").read_text() for e in ("gfa", "fasta", "yaml"))
    assert got == want
    assert "topology: empty" in want[2] and "fully_resolved: false" in want[2]


def test_combine_one_circular_emu(emu, tmp_path):
    (tmp_path / "a.gfa").write_text("H\tVN:Z:1.0\tKM:i:51\nS\t1\tACGTACGT\tDP:f:3.25\tCL:Z:steelblue\nL\t1\t+\t1\t+\t0M\nL\t1\t-\t1\t-\t0M\n")
    (tmp_path / "b.gfa").write_text("H\tVN:Z:1.0\tKM:i:51\nS\t2\tAAAT\tDP:f:1\n")
    api.combine(str(tmp_path), [str(tmp_path / "a.gfa"), str(tmp_path / "b.gfa")], lib=emu)
    want = R.combine_gfas([(tmp_path / "a.gfa").read_text(), (tmp_path / "b.gfa").read_text()])
    assert (tmp_path / "consensus_assembly.yaml").read_text() == want[2]
    assert want[2] == ("consensus_assembly_bases: 12\nconsensus_assembly_unitigs: 2\nconsensus_assembly_fully_resolved: true\n"
                       "consensus_assembly_clusters:\n- length: 8\n  unitigs: 1\n  topology: circular\n- length: 4\n  unitigs: 1\n"
                       "  topology: linear-open-open\n")
    assert (tmp_path / "consensus_assembly.fasta").read_text() == want[1] == \
        ">1 length=8 circular=true topology=circular\nACGTACGT\n>3 length=4 circular=false topology=linear\nAAAT\n"
    assert (tmp_path / "consensus_assembly.gfa").read_text() == want[0]


# ---- errors -----------------------------------------------------------------------------------------------------------------------

def test_errors_emu(emu, tmp_path):
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.resolve(str(tmp_path / "nope"), lib=emu)
    assert e.value.code == -6 and e.value.message == f"directory does not exist: {tmp_path / 'nope'}"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.resolve(str(tmp_path), lib=emu)
    assert e.value.code == -6 and e.value.message == f"file does not exist: {tmp_path / '2_trimmed.gfa'}"
    (tmp_path / "file").write_text("x")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.resolve(str(tmp_path / "file"), lib=emu)
    assert e.value.code == -6 and e.value.message == f"{tmp_path / 'file'} is not a directory"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.combine(str(tmp_path / "out"), [str(tmp_path / "file"), str(tmp_path / "missing.gfa")], lib=emu)
    assert e.value.code == -6 and e.value.message == f"file does not exist: {tmp_path / 'missing.gfa'}"
    assert not (tmp_path / "out").exists()


# ---- the chain ----------------------------------------------------------------------------------------------------------------------

def _chain_dir(tmp_path, config="cfg1", n_assemblies=5, lengths=(30_000, 6_000), seed=3):
    asm = synth.make_assemblies(config, n_assemblies=n_assemblies, replicon_lengths=list(lengths), seed=seed)
    asm = [(fn, list(recs)) for fn, recs in asm]
    asm[1][1][0] = (asm[1][1][0][0] + " Autocycler_consensus_weight=2", asm[1][1][0][1])
    d = tmp_path / "asm"
    synth.write_assemblies(asm, str(d))
    return d


def _chain(lib, tmp_path, **kw):
    """compress -> cluster -> trim -> resolve of every qc_pass cluster -> combine, by the product; every file against the oracle chain."""
    d = _chain_dir(tmp_path, **kw)
    a = tmp_path / "ac"
    api.compress(str(d), str(a), lib=lib)
    gfa = (a / "input_assemblies.gfa").read_text()
    want = cluster_oracle.cluster(gfa)
    api.cluster(str(a), lib=lib)
    finals, want_finals = [], []
    for k in sorted(want):
        if k.startswith("qc_pass") and k.endswith(".gfa"):
            cd = a / "clustering" / os.path.dirname(k)
            api.trim(str(cd), lib=lib)
            tg, _ = trim_oracle.trim_gfa(want[k])
            assert (cd / "2_trimmed.gfa").read_text() == tg
            api.resolve(str(cd), lib=lib)
            rw = R.resolve_gfa(tg)
            assert tuple((cd / f).read_text() for f in ("3_bridged.gfa", "4_merged.gfa", "5_final.gfa")) == rw, k
            finals.append(str(cd / "5_final.gfa"))
            want_finals.append(rw[2])
    assert finals
    api.combine(str(a), finals, lib=lib)
    cw = R.combine_gfas(want_finals)
    assert tuple((a / f"consensus_assembly.{e}").read_text() for e in ("gfa", "fasta", "yaml")) == cw
    return a


def test_chain_emu(emu, tmp_path):
    _chain(emu, tmp_path)


# ---- on the H100 ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_synthetic()))
def test_synthetic_gpu(gpu, name):
    _check_resolve(gpu, _synthetic()[name])


@pytest.mark.gpu
def test_fixtures_gpu(gpu):
    for text in _fixture_texts().values():
        _check_resolve(gpu, text)


@pytest.mark.gpu
def test_chain_gpu(gpu, tmp_path):
    _chain(gpu, tmp_path)


@pytest.mark.gpu
def test_cli_gpu(tmp_path):
    text = _synthetic()["conflicts"]
    (tmp_path / "2_trimmed.gfa").write_text(text)
    outs = []
    for _ in range(2):                                   # deterministic across runs
        r = subprocess.run([AUTOCYCLER, "resolve", "-c", str(tmp_path), "--verbose"], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        outs.append(tuple((tmp_path / f).read_text() for f in ("3_bridged.gfa", "4_merged.gfa", "5_final.gfa")))
    assert outs[0] == outs[1] == R.resolve_gfa(text)
    r = subprocess.run([AUTOCYCLER, "combine", "-a", str(tmp_path / "c"), "-i", str(tmp_path / "5_final.gfa"), str(tmp_path / "4_merged.gfa")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    want = R.combine_gfas([outs[0][2], outs[0][1]])
    assert (tmp_path / "c" / "consensus_assembly.yaml").read_text() == want[2]
    r = subprocess.run([AUTOCYCLER, "resolve", "-c", str(tmp_path / "nope")], capture_output=True, text=True)
    assert r.returncode == 1 and f"Error: directory does not exist: {tmp_path / 'nope'}" in r.stderr
    r = subprocess.run([AUTOCYCLER, "combine", "-a", str(tmp_path / "c"), "-i", str(tmp_path / "missing.gfa")], capture_output=True, text=True)
    assert r.returncode == 1 and f"Error: file does not exist: {tmp_path / 'missing.gfa'}" in r.stderr


@pytest.mark.gpu
def test_goldens_gpu(tmp_path):
    """The benchmark workloads' resolves against the SHA-256 of the oracle's outputs (tests/golden/resolve_goldens.json, made by
    make_resolve_goldens.py)."""
    import bench_resolve
    goldens = json.load(open(os.path.join(ROOT, "tests", "golden", "resolve_goldens.json")))
    for name, trimmed in bench_resolve.workloads(str(tmp_path)).items():
        g, _ = api.UnitigGraph.from_gfa_lines(trimmed.encode())
        g.resolve()
        got = {w: hashlib.sha256(g.resolve_text(w).encode()).hexdigest() for w in ("bridged", "merged", "final")}
        assert got == goldens[name]["sha256"], name
