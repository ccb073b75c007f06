"""Parity tests proper: the CUDA path, through the C ABI, against the oracle (bit-exact: integer/byte work).
Run on an H100 with `pytest -m gpu`."""
import hashlib
import json
import os

import pytest

import cases
import oracle_lib as o
from autocycler_b200 import api, synth
from parity_common import check_case, run_library

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    lib = api.load_library()   # the in-tree sm_90a build; raises if it is missing
    assert b"sm_90a" in lib.ac_version()
    return lib


@pytest.mark.parametrize("k", [3, 5, 9, 11, 31, 33, 51, 63, 65, 91, 127, 129, 255, 321, 501])
def test_random_adversarial_cases(lib, k):
    for seed in range(10):
        check_case(lib, cases.random_case(1000 * k + seed, k), k)


@pytest.mark.parametrize("seed,k", [(339, 3), (717, 9), (780, 33), (802, 65), (865, 91), (871, 51), (944, 31)])
def test_regressions_found_by_the_stress_harness(lib, seed, k):
    check_case(lib, cases.random_case(seed * 100 + k, k), k)


def test_reference_fixed_seqs(lib):   # tests.rs:131-148 inputs
    from test_oracle_kats import FIXED
    files = [(f"{n}.fasta", [(n, s.split("\n")[1])]) for n, s in zip("abcde", FIXED)]
    for k in (5, 9, 13, 51):
        check_case(lib, files, k)


@pytest.mark.parametrize("k", [31, 51, 91])
def test_config1(lib, tmp_path, k):   # BASELINE.json configs[0] at the k sweep of configs[3]
    d = str(tmp_path / "cfg1")
    synth.write_assemblies(synth.make_assemblies("cfg1"), d)
    expected, yaml, st = o.compress_dir(d, k)
    got = run_library(lib, d, k)
    assert got["gfa"] == expected
    assert got["before"].n_kmers == st.n_kmers


def test_medium_with_plasmids_and_repeats(lib, tmp_path):   # a scaled-down configs[2]: chromosome + plasmids, 6 assemblies
    d = str(tmp_path / "m")
    synth.write_assemblies(synth.make_assemblies("m", n_assemblies=6, replicon_lengths=[400_000, 22_000, 8_000, 3_000], seed=99), d)
    expected, yaml, st = o.compress_dir(d, 51)
    got = run_library(lib, d, 51)
    assert got["gfa"] == expected


def test_identical_assemblies_long_unitigs(lib, tmp_path):   # zero divergence: one unitig spans the whole replicon
    d = str(tmp_path / "i")
    synth.write_assemblies(synth.make_assemblies("i", n_assemblies=4, replicon_lengths=[300_000], seed=5, sub=0, ins=0, dele=0), d)
    expected, yaml, st = o.compress_dir(d, 51)
    got = run_library(lib, d, 51)
    assert got["gfa"] == expected


def test_config2_full_size_golden_and_round_trip(lib, tmp_path):
    """BASELINE.json configs[1]: 8 x 4.64 Mbp, k=51.  Byte identity through the committed SHA-256 of the oracle's
    GFA (tests/golden/config_goldens.json), plus the reference's size-independent invariants (tests.rs:108-127):
    save -> load -> save is the identity and decompress reproduces every input file."""
    goldens = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))
    g = goldens["cfg2_k51"]
    d = str(tmp_path / "cfg2")
    assemblies = synth.make_assemblies("cfg2")
    synth.write_assemblies(assemblies, d)
    got = run_library(lib, d, 51)
    assert got["before"].n_kmers == g["n_kmers"]
    assert (got["after"].n_unitigs, got["after"].n_links) == (g["unitigs_after"], g["links_after"])
    assert len(got["gfa"]) == g["gfa_bytes"]
    assert hashlib.sha256(got["gfa"].encode()).hexdigest() == g["sha256"]
    assert o.gfa_roundtrip(got["gfa"]) == got["gfa"]
    rec = tmp_path / "rec"; rec.mkdir()
    o.decompress(got["gfa"], str(rec))
    for fn, recs in assemblies:
        assert open(os.path.join(rec, fn), "rb").read() == open(os.path.join(d, fn), "rb").read()
    # the same invariants through the library itself, and the step every downstream command takes next
    graph, originals = got["graph"], [bytes(s).decode() for _, recs in assemblies for _, s in recs]
    assert [graph.reconstruct_original_sequence(i) for i in range(len(originals))] == originals
    api.simplify_structure(graph)                                  # idempotent: nothing left to expand, same numbering
    assert graph.gfa_bytes().decode() == got["gfa"]
    api.merge_linear_paths(graph, got["seqs"])
    merged = graph.gfa_bytes().decode()
    assert merged == o.gfa_merge_linear_paths(got["gfa"])
    assert [graph.reconstruct_original_sequence(i) for i in range(len(originals))] == originals


@pytest.mark.parametrize("name,k", [("cfg3", 51), ("cfg4", 51), ("cfg4", 31), ("cfg4", 91)])
def test_larger_configs_against_committed_oracle_hashes(lib, tmp_path, name, k):
    """BASELINE.json configs[2] and configs[3] (k sweep): SHA-256 of the oracle's GFA, generated in the build container by
    tests/golden/make_config_goldens.py (the oracle needs 3-15 minutes per entry, so only the hash travels)."""
    goldens = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))
    key = f"{name}_k{k}"
    if key not in goldens:
        pytest.skip(f"no committed oracle hash for {key}")
    g = goldens[key]
    d = str(tmp_path / name)
    synth.write_assemblies(synth.make_assemblies(name), d)
    got = run_library(lib, d, k)
    assert got["before"].n_kmers == g["n_kmers"]
    assert (got["after"].n_unitigs, got["after"].n_links, len(got["gfa"])) == (g["unitigs_after"], g["links_after"], g["gfa_bytes"])
    assert hashlib.sha256(got["gfa"].encode()).hexdigest() == g["sha256"]


def test_handle_reuse_and_determinism(lib, tmp_path):
    """Two builds on one handle and a build on a fresh handle give the same bytes (atomics race for slots, the
    output must not depend on who wins)."""
    d = str(tmp_path / "r")
    synth.write_assemblies(synth.make_assemblies("r", n_assemblies=5, replicon_lengths=[150_000], seed=11), d)
    kg, seqs, count = api.load_sequences(d, 51, lib=lib)
    outs = []
    for _ in range(3):
        kg.upload()
        g = api.UnitigGraph.from_kmer_graph(kg)
        api.simplify_structure(g)
        outs.append(g.gfa_bytes())
    assert outs[0] == outs[1] == outs[2]
    assert outs[0].decode() == o.compress_dir(d, 51)[0]


def test_cli_binary(lib, tmp_path):
    import subprocess
    d = str(tmp_path / "c"); out = str(tmp_path / "out")
    synth.write_assemblies(synth.make_assemblies("c", n_assemblies=3, replicon_lengths=[30_000], seed=3), d)
    exe = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
    r = subprocess.run([exe, "compress", "-i", d, "-a", out, "--kmer", "51", "-t", "4"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    expected, yaml, st = o.compress_dir(d, 51)
    assert open(os.path.join(out, "input_assemblies.gfa")).read() == expected
    assert open(os.path.join(out, "input_assemblies.yaml")).read() == yaml
    r = subprocess.run([exe, "compress", "-i", d, "-a", out, "--kmer", "50"], capture_output=True, text=True)
    assert r.returncode == 1 and "Error: --kmer must be odd" in r.stderr      # compress.rs:58, misc.rs:130-136


def test_loaded_graphs_and_reference_kats(lib, golden_dir, tmp_path):
    """The host-side rows after compress, in the CUDA build: the reference's simplify / merge KATs on its own GFA fixtures
    (graph_simplification.rs:627-671, 742-801) through ac_load_gfa, and decompress of a graph this GPU just built."""
    text = lambda n: open(os.path.join(golden_dir, f"ref_test_gfa_{n}.gfa")).read()
    g, seqs = api.UnitigGraph.from_gfa_lines(text(1), lib=lib)
    api.simplify_structure(g)
    assert [u["seq"] for u in g.unitigs()] == ["GCATTCGCTGCGCTCGCTTCGCTTT", "TGCCGTCGTCGCTGT", "CTGAATCGCCTA", "GCTCGGCTCGA", "CGAACCAT", "TACTTGT", "GCCT", "TCT", "GC", "T"]
    g, seqs = api.UnitigGraph.from_gfa_lines(text(3), lib=lib)
    api.merge_linear_paths(g, seqs)
    assert {u["number"]: u["seq"] for u in g.unitigs()} == {8: "TTCGCTGCGCTCGCTTCGCTTTTGCACAGCGACGACGGCATGCCTGAATCGCCTA", 9: "GCTCGGCTCGATGGTTCG", 10: "TACTTGTAAGGC"}
    for n in range(1, 15):
        g, seqs = api.UnitigGraph.from_gfa_lines(text(n), lib=lib)
        assert g.gfa_bytes().decode() == o.gfa_roundtrip(text(n))
    d = str(tmp_path / "in"); out = str(tmp_path / "out")
    assemblies = synth.make_assemblies("d", n_assemblies=4, replicon_lengths=[60_000, 4_000], seed=21)
    synth.write_assemblies(assemblies, d)
    got = run_library(lib, d, 51)
    gfa_path = str(tmp_path / "g.gfa"); open(gfa_path, "w").write(got["gfa"])
    api.decompress(gfa_path, out_dir=out, lib=lib)
    for fn, recs in assemblies:
        assert open(os.path.join(out, fn), "rb").read() == open(os.path.join(d, fn), "rb").read()


@pytest.mark.parametrize("env", [{}, {"AC_DEVICE_TIGHT_ARENA": "1"}], ids=["fused", "fused_tight_arena"])
def test_device_expansion_switches_match_the_oracle(lib, tmp_path, env):
    """The fused build (ac_compress: expand_repeats applied by device kernels, pipeline.cu ApplyLevelBody, then the device GFA writer), as it
    runs and with the arena regrown before every pass: same bytes as the oracle on a medium graph.  The switch is read once per process, so
    the build runs in a child."""
    import subprocess
    import sys
    d = str(tmp_path / "m")
    synth.write_assemblies(synth.make_assemblies("m", n_assemblies=6, replicon_lengths=[400_000, 22_000, 8_000, 3_000], seed=99), d)
    expected, yaml, st = o.compress_dir(d, 51)
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from autocycler_b200 import api\n"
            "kg, seqs, count = api.load_sequences(%r, 51)\nkg.upload()\n"
            "open(%r, 'wb').write(bytes(api.UnitigGraph.compress(kg).gfa_view()))\n") % (os.path.join(ROOT, "tests"), ROOT, d, str(tmp_path / "out.gfa"))
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, **env}, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-2000:]
    assert open(tmp_path / "out.gfa").read() == expected
