"""`autocycler cluster` (cluster.rs): UPGMA on seeded random matrices and the reference's unit-test data (tests/golden/cluster_kats.json),
and whole-command runs on synthetic genomes, each checked against the CPU oracle (tests/cluster_oracle.py).  The CPU tests run the
product's code through the host-emulation library (the UPGMA kernel's row scan, merge-row update and pair order, serially); the tests
marked gpu run the CUDA build on the H100."""
import hashlib
import json
import os
import random
import subprocess

import numpy as np
import pytest

import cluster_oracle as O
import oracle_lib
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "cluster_kats.json")))


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


# ---- number formats ---------------------------------------------------------------------------------------------------------------

RUST = [(11.0, "11"), (0.05, "0.05"), (1e-7, "0.0000001"), (0.0, "0"), (-0.0, "-0"), (2.5, "2.5"), (1e21, "1000000000000000000000"),
        (0.1 + 0.2, "0.30000000000000004"), (123456.0, "123456")]
YAML = [(0.0, "0.0"), (1.0, "1.0"), (0.5, "0.5"), (1e-5, "0.00001"), (1.5e-5, "0.000015"), (1e-6, "1e-6"), (1.5e-6, "1.5e-6"),
        (1e15, "1000000000000000.0"), (1e16, "1e16"), (1.25e16, "1.25e16"), (9999999999999998.0, "9999999999999998.0"), (0.1 + 0.2, "0.30000000000000004")]


@pytest.mark.parametrize("v,text", RUST)
def test_rust_display(v, text):
    assert O.rust_display(v) == text


@pytest.mark.parametrize("v,text", YAML)
def test_yaml_float(v, text):
    assert O.yaml_float(v) == text


# ---- UPGMA ------------------------------------------------------------------------------------------------------------------------

def _random_matrix(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 301)) if seed % 5 else int(rng.integers(2, 12))
    m = rng.random((n, n))
    m = np.maximum(m, m.T)
    k = int(rng.integers(0, n))                     # planted exact ties at 0 and 1
    for _ in range(k):
        i, j = rng.integers(0, n, 2)
        m[i, j] = m[j, i] = float(rng.integers(0, 2))
    np.fill_diagonal(m, 0.0)
    ids = sorted(rng.choice(np.arange(1, 3 * n + 1), n, replace=False).tolist()) if seed % 3 == 0 else list(range(1, n + 1))
    return m, ids


def _check_upgma(lib, seeds):
    for seed in seeds:
        m, ids = _random_matrix(seed)
        got, _ = api.upgma(m, ids, lib=lib)
        assert got == O.upgma(m, ids), seed


def test_oracle_upgma_equals_reference_port():
    for seed in range(60):
        m, ids = _random_matrix(seed)
        if len(ids) > 40:
            continue
        _same_as_reference_port(m, ids)
    for m, ids in _kat_matrices():
        _same_as_reference_port(m, ids)


def _same_as_reference_port(m, ids):
    a, b = O.upgma(m, ids), O.upgma_reference(m, ids)
    assert [x[:3] for x in a] == [x[:3] for x in b]
    assert all(abs(x[3] - y[3]) <= 1e-12 for x, y in zip(a, b))


def test_upgma_random_emu(emu):
    _check_upgma(emu, range(80))


# ---- the reference's unit tests (tests/golden/cluster_kats.json, extract_cluster_kats.py) -------------------------------------------

def _kat_matrices():
    out = [(np.array(c["matrix"]), c["ids"]) for c in KATS["cases"] if "matrix" in c]
    return out + [(np.array(t["matrix"]), t["ids"]) for t in KATS["trees"].values()]


def _tree(name):
    nodes = KATS["trees"][name]["nodes"]
    return O.Tree(KATS["trees"][name]["ids"], sorted(nodes))


def _run_case(case, lib=None):
    """Replays one reference test on the oracle (lib=None) or, for the UPGMA steps, on the product's ac_upgma."""
    seqs = [O.Seq(i, [], ln, fn, hd) for i, fn, hd, ln in case.get("sequences", [])]
    tree = root = None
    for op in case["ops"]:
        kind, args = op[0], op[1:]
        if kind == "sequences":
            seqs = [O.Seq(i, [], ln, fn, hd) for i, fn, hd, ln in args[0]]
        elif kind == "tree":
            tree = _tree(args[0])
        elif kind == "upgma":
            m, ids = np.array(case["matrix"]), case["ids"]
            merges = api.upgma(m, ids, lib=lib)[0] if lib else O.upgma(m, ids)
            root = O.Tree(ids, merges)
        elif kind == "normalise":
            root.normalise()
        elif kind == "root_distance":
            assert abs(root.dist[root.root] - args[0]) < 1e-8
        elif kind == "newick":
            assert root.newick(root.root, {s.id: s for s in seqs}) == args[0]
        elif lib:
            continue                                 # the rest are host steps: the oracle's, checked below
        elif kind == "automatic":
            out = []
            tree.collect(tree.root, args[0] / 2.0, [], out)
            assert sorted(out) == args[1]
        elif kind == "manual":
            tree.check_consistency(tree.root, args[1])
            out = []
            tree.collect(tree.root, args[0] / 2.0, args[1], out)
            assert sorted(out) == args[2]
        elif kind == "has_manual_child":
            assert tree.has_manual(tree.root, args[0]) == args[1]
        elif kind in ("consistency", "coverage"):
            fn = (lambda c: tree.check_consistency(tree.root, c)) if kind == "consistency" else tree.check_complete_coverage
            if args[1]:
                fn(args[0])
            else:
                with pytest.raises(ValueError):
                    fn(args[0])
        elif kind == "max_pairwise_distance":
            assert abs(tree.max_pairwise_distance(args[0]) - args[1]) < 1e-8
        elif kind == "get_tips":
            assert (tree.tips(args[0]) if tree.find(args[0]) else []) == args[1]
        elif kind == "split":
            tree.check_complete_coverage(args[0])
            assert tree.splits(args[0]) == args[1]
        elif kind == "find_node":
            assert tree.find(args[0]) == args[1]
        elif kind == "parse_manual":
            if args[1] is None:
                with pytest.raises(ValueError):
                    O.parse_manual_clusters(args[0])
            else:
                assert O.parse_manual_clusters(args[0]) == args[1]
        elif kind == "set_cluster":
            seqs[args[0]].cluster = args[1]
        elif kind == "cluster_assembly_count":
            assert O.cluster_assembly_count(seqs, args[0]) == args[1]
        elif kind == "set_min_assemblies":
            assert O.set_min_assemblies(args[0], seqs) == args[1]
        elif kind == "pop":
            seqs.pop()
        elif kind == "truncate":
            del seqs[args[0]:]
        elif kind == "reorder":
            O.reorder_clusters(seqs)
        elif kind == "cluster_of":
            assert seqs[args[0]].cluster == args[1]
        elif kind == "assembly_count":
            assert len({s.filename for s in seqs}) == args[0]
        elif kind == "max_cluster":
            assert max(s.cluster for s in seqs) == args[0]
        else:
            raise AssertionError(f"unknown step {kind}")


@pytest.mark.parametrize("case", KATS["cases"], ids=lambda c: c["test"])
def test_reference_cases(case):
    _run_case(case)


@pytest.mark.parametrize("name", sorted(KATS["trees"]))
def test_reference_trees_are_upgma_trees(emu, name):
    """test_tree_1 / test_tree_2 as ultrametric matrices: their UPGMA tree (oracle and ac_upgma) is that tree; test_tree_2 has exact ties."""
    t = KATS["trees"][name]
    for merges in (O.upgma(np.array(t["matrix"]), t["ids"]), api.upgma(np.array(t["matrix"]), t["ids"], lib=emu)[0]):
        assert [list(m[:3]) for m in merges] == [n[:3] for n in t["nodes"]]
        assert all(abs(m[3] - n[3]) <= 1e-12 for m, n in zip(merges, t["nodes"]))


def test_reference_upgma_cases_emu(emu):
    for case in KATS["cases"]:
        if "matrix" in case:
            _run_case(case, lib=emu)


# ---- whole command ----------------------------------------------------------------------------------------------------------------

def _autocycler_dir(tmp_path, name):
    """input_assemblies.gfa of a synthetic genome (compressed by the CPU oracle) with what `name` asks for injected."""
    asm = synth.make_assemblies(name, n_assemblies=6, replicon_lengths=[30_000, 8_000, 3_000], seed=sum(map(ord, name)))
    asm = [(fn, list(recs)) for fn, recs in asm]
    rng = random.Random(7)
    if name in ("contaminant", "mixed"):
        junk = np.frombuffer(bytes(rng.choice(b"ACGT") for _ in range(4000)), dtype=np.uint8).copy()
        asm[2][1].append(("contaminant_1", junk))
    if name in ("fragment", "mixed"):
        asm[4][1].append(("fragment_1", asm[4][1][0][1][5000:17000].copy()))
    if name in ("headers", "mixed"):
        asm[0][1][0] = (asm[0][1][0][0] + " Autocycler_trusted", asm[0][1][0][1])
        asm[1][1][-1] = (asm[1][1][-1][0] + " autocycler_cluster_weight=3", asm[1][1][-1][1])
        asm[3][1][1] = (asm[3][1][1][0] + " Autocycler_consensus_weight=2", asm[3][1][1][1])
    d = tmp_path / "asm"
    synth.write_assemblies(asm, str(d))
    gfa, _, _ = oracle_lib.compress_dir(str(d), 51)
    a = tmp_path / "ac"
    a.mkdir()
    (a / "input_assemblies.gfa").write_text(gfa)
    return a, gfa


def _tree_files(d):
    out = {}
    for root, _, files in os.walk(d):
        for f in files:
            p = os.path.join(root, f)
            out[os.path.relpath(p, d)] = open(p).read()
    return out


CASES = [("contaminant", 0.2, None, None), ("fragment", 0.2, None, None), ("headers", 0.2, None, None), ("mixed", 0.05, None, None),
         ("mixed", 0.2, None, None), ("mixed", 0.5, None, None), ("mixed", 0.2, 4, None), ("mixed", 0.2, None, "manual")]


def _manual_from_newick(gfa):
    """the two children of the oracle tree's root: node numbers a user would read off clustering.newick"""
    lengths, seqs = O.parse_gfa(gfa)
    order = sorted(range(len(seqs)), key=lambda i: seqs[i].id)
    merges = O.upgma(O.symmetric(O.distances(lengths, seqs))[np.ix_(order, order)], [seqs[i].id for i in order])
    return sorted(merges[-1][1:3])


def _check_command(lib, tmp_path, name, cutoff, min_asm, manual):
    a, gfa = _autocycler_dir(tmp_path, name)
    man = _manual_from_newick(gfa) if manual else None
    want = O.cluster(gfa, cutoff, min_asm, man)
    api.cluster(str(a), cutoff=cutoff, min_assemblies=min_asm, manual=",".join(map(str, man)) if man else None, lib=lib)
    got = _tree_files(a / "clustering")
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k] == want[k], k
    g, seqs = api.UnitigGraph.from_gfa_lines(gfa.encode(), lib=lib)
    before = bytes(g.gfa_bytes())
    g.cluster(cutoff, min_asm, man)
    assert bytes(g.gfa_bytes()) == before                      # the handle's graph and sequences are left as they were
    assert _handle_texts(g, want) == want
    lengths, oseqs = O.parse_gfa(gfa)                          # the sum-based UPGMA equals the reference's loop on real distances
    _same_as_reference_port(O.symmetric(O.distances(lengths, oseqs)), [s.id for s in oseqs])
    return want


def _handle_texts(g, like):
    got = {"pairwise_distances.phylip": g.cluster_text("phylip"), "clustering.newick": g.cluster_text("newick"),
           "clustering.tsv": g.cluster_text("tsv"), "clustering.yaml": g.cluster_text("yaml")}
    for k in like:
        if "/" in k:
            got[k] = g.cluster_text("gfa" if k.endswith(".gfa") else "untrimmed_yaml", int(k.split("/")[1][8:]))
    return got


@pytest.mark.parametrize("name,cutoff,min_asm,manual", CASES)
def test_command_emu(emu, tmp_path, name, cutoff, min_asm, manual):
    _check_command(emu, tmp_path, name, cutoff, min_asm, manual)


def test_cases_do_what_they_say(tmp_path):
    """The oracle's own view: the contaminant (one assembly) and the chromosome fragment (contained) end up in failed clusters."""
    for name, contig in (("contaminant", "contaminant_1"), ("fragment", "fragment_1")):
        (tmp_path / name).mkdir()
        _, gfa = _autocycler_dir(tmp_path / name, name)
        tsv = O.cluster(gfa)["clustering.tsv"]
        assert any(ln.split("\t")[1] == "none" and ln.split("\t")[5] == contig for ln in tsv.splitlines()), (name, tsv)


def test_chain_emu(emu, tmp_path):
    """compress -> cluster -> trim of every qc_pass cluster, against the oracle chain."""
    import trim_oracle
    a, gfa = _autocycler_dir(tmp_path, "mixed")
    want = O.cluster(gfa)
    api.cluster(str(a), lib=emu)
    for k in want:
        if k.startswith("qc_pass") and k.endswith(".gfa"):
            d = a / "clustering" / os.path.dirname(k)
            api.trim(str(d), lib=emu)
            tg, ty = trim_oracle.trim_gfa(want[k])
            assert (d / "2_trimmed.gfa").read_text() == tg and (d / "2_trimmed.yaml").read_text() == ty


@pytest.mark.parametrize("kw,message", [
    (dict(cutoff=0.0), "--cutoff must be between 0 and 1 (exclusive)"),
    (dict(cutoff=1.0), "--cutoff must be between 0 and 1 (exclusive)"),
    (dict(min_assemblies=0), "--min_assemblies must be 1 or greater"),
    (dict(manual="1,x"), "failed to parse 'x' as a node number"),
    (dict(max_contigs=1), "the mean number of contigs per input assembly (3.0) exceeds the allowed threshold (1). Are your input assemblies fragmented or contaminated?"),
])
def test_errors(emu, tmp_path, kw, message):
    a, _ = _autocycler_dir(tmp_path, "headers")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(a), lib=emu, **kw)
    assert e.value.code == -6 and e.value.message == message


def _tiny_distance_gfa():
    """Two contigs that share a 1,999,999 bp unitig and differ in one 1 bp unitig each: distance 5e-7, so the Newick lengths and the YAML
    distance take the formats' small-number branches (decimal digits far right of the point, ryu's exponent form)."""
    big = "".join(random.Random(3).choice("ACGT") for _ in range(1_999_999))
    return ("H\tVN:Z:1.0\tKM:i:51\n"
            f"S\t1\t{big}\tDP:f:2.00\nS\t2\tA\tDP:f:1.00\nS\t3\tC\tDP:f:1.00\n"
            "L\t1\t+\t2\t+\t0M\nL\t1\t+\t3\t+\t0M\nL\t2\t-\t1\t-\t0M\nL\t3\t-\t1\t-\t0M\n"
            "P\t1\t1+,2+\t*\tLN:i:2000000\tFN:Z:a.fasta\tHD:Z:c1\n"
            "P\t2\t1+,3+\t*\tLN:i:2000000\tFN:Z:b.fasta\tHD:Z:c1\n")


def test_small_number_formats_emu(emu, tmp_path):
    """The product's own Rust `{}` and serde_yaml f64 writers on values below 1e-5, against the oracle's (pinned by the tests above)."""
    gfa = _tiny_distance_gfa()
    want = O.cluster(gfa, 0.2)
    (tmp_path / "input_assemblies.gfa").write_text(gfa)
    api.cluster(str(tmp_path), lib=emu)
    got = _tree_files(tmp_path / "clustering")
    assert got == want
    y = got["qc_pass/cluster_001/1_untrimmed.yaml"]
    assert "untrimmed_cluster_distance: " in y and "e-7\n" in y, y
    assert ":0.00000025" in got["clustering.newick"] or ":0.0000002" in got["clustering.newick"], got["clustering.newick"]


def _empty_paths_gfa():
    return ("H\tVN:Z:1.0\tKM:i:51\nS\t1\tACGTACGT\tDP:f:1.00\n"
            "P\t1\t1+\t*\tLN:i:8\tFN:Z:a.fasta\tHD:Z:c1\nP\t2\t\t*\tLN:i:0\tFN:Z:b.fasta\tHD:Z:c1\n"
            "P\t3\t\t*\tLN:i:0\tFN:Z:c.fasta\tHD:Z:c1\n")


def test_nan_distances_are_refused_emu(emu, tmp_path):
    """Two paths without length have a 0 / 0 distance; a NaN leaves UPGMA without a pair to merge.  Both entry points refuse it."""
    m = np.array([[0.0, 0.3, np.nan], [0.3, 0.0, 0.5], [np.nan, 0.5, 0.0]])
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.upgma(m, [1, 2, 3], lib=emu)
    assert e.value.code == -6 and "NaN" in e.value.message
    (tmp_path / "input_assemblies.gfa").write_text(_empty_paths_gfa())
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(tmp_path), lib=emu)
    assert e.value.code == -6 and e.value.message == "the distance between sequences 2 and 3 is not a number (their paths have no length)"


def test_clustering_path_that_is_a_file(emu, tmp_path):
    """Only a directory called clustering is replaced; a file of that name is left alone and the command fails."""
    a, _ = _autocycler_dir(tmp_path, "headers")
    (a / "clustering").write_text("keep me")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(a), lib=emu)
    assert e.value.code == -6 and e.value.message.startswith(f"failed to create directory {a / 'clustering'}")
    assert (a / "clustering").read_text() == "keep me"


def test_errors_inputs(emu, tmp_path):
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(tmp_path / "nope"), lib=emu)
    assert e.value.code == -6 and e.value.message == f"directory does not exist: {tmp_path / 'nope'}"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(tmp_path), lib=emu)
    assert e.value.code == -6 and e.value.message == f"file does not exist: {tmp_path / 'input_assemblies.gfa'}"
    (tmp_path / "input_assemblies.gfa").write_text("H\tVN:Z:1.0\tKM:i:51\n")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(tmp_path), lib=emu)
    assert e.value.code == -6 and e.value.message == "no sequences found in input_assemblies.gfa"


def test_nested_manual(emu, tmp_path):
    a, gfa = _autocycler_dir(tmp_path, "headers")
    lengths, seqs = O.parse_gfa(gfa)
    merges = O.upgma(O.symmetric(O.distances(lengths, seqs)), [s.id for s in seqs])
    root = merges[-1][0]
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.cluster(str(a), manual=f"{root},{merges[-1][1]}", lib=emu)
    assert e.value.code == -6 and e.value.message == "manual clusters cannot be nested"


# ---- on the H100 ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_upgma_random_gpu(gpu):
    _check_upgma(gpu, range(80))


@pytest.mark.gpu
def test_reference_upgma_cases_gpu(gpu):
    for case in KATS["cases"]:
        if "matrix" in case:
            _run_case(case, lib=gpu)
    for t in KATS["trees"].values():
        merges = api.upgma(np.array(t["matrix"]), t["ids"], lib=gpu)[0]
        assert merges == O.upgma(np.array(t["matrix"]), t["ids"])


@pytest.mark.gpu
def test_upgma_3000_gpu(gpu):
    rng = np.random.default_rng(3000)
    m = rng.random((3000, 3000))
    m = np.maximum(m, m.T)
    np.fill_diagonal(m, 0.0)
    ids = list(range(1, 3001))
    got, _ = api.upgma(m, ids, lib=gpu)
    assert got == O.upgma(m, ids)


@pytest.mark.gpu
@pytest.mark.parametrize("name,cutoff,min_asm,manual", CASES)
def test_command_gpu(gpu, tmp_path, name, cutoff, min_asm, manual):
    _check_command(gpu, tmp_path, name, cutoff, min_asm, manual)


@pytest.mark.gpu
def test_cli_and_determinism_gpu(tmp_path):
    a, gfa = _autocycler_dir(tmp_path, "mixed")
    want = O.cluster(gfa)
    exe = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
    r = subprocess.run([exe, "cluster", "-a", str(a)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    first = _tree_files(a / "clustering")
    assert first == want
    r = subprocess.run([exe, "cluster", "-a", str(a)], capture_output=True, text=True)
    assert r.returncode == 0 and _tree_files(a / "clustering") == first
    r = subprocess.run([exe, "cluster", "-a", str(a), "--cutoff", "1.5"], capture_output=True, text=True)
    assert r.returncode == 1 and "Error: --cutoff must be between 0 and 1 (exclusive)" in r.stderr


@pytest.mark.gpu
def test_cfg3_gpu(tmp_path):
    """cfg3 (12 assemblies x 6 replicons) compressed on the GPU and clustered, against the SHA-256 of every file the oracle wrote
    (tests/golden/cluster_goldens.json, made by make_cluster_goldens.py)."""
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "cluster_goldens.json")))["cfg3_k51_cutoff0.2"]
    synth.write_assemblies(synth.make_assemblies("cfg3"), str(tmp_path / "asm"))
    api.compress(str(tmp_path / "asm"), str(tmp_path / "ac"))
    api.cluster(str(tmp_path / "ac"))
    got = {k: hashlib.sha256(v.encode()).hexdigest() for k, v in _tree_files(tmp_path / "ac" / "clustering").items()}
    assert got == want
