"""CPU tests of the product's host logic and of the device function bodies, the latter through the
host-emulation build (tests/emu/libautocycler_emu.so: the same kernel bodies run serially).  The CUDA
build itself is exercised by test_parity_gpu.py on the H100."""
import os
import subprocess

import pytest

import cases
import oracle_lib as o
from autocycler_b200 import api, synth
from parity_common import check_case, run_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="session")
def emu():
    path = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(path)


@pytest.mark.parametrize("k", [3, 5, 7, 9, 11, 31, 33, 51, 63, 65, 91, 127, 129, 159, 161, 255, 257, 319, 321, 401, 501, 511])
def test_random_adversarial_cases(emu, k):
    for seed in range(40):
        check_case(emu, cases.random_case(1000 * k + seed, k), k)


@pytest.mark.parametrize("seed,k", [(339, 3), (717, 9), (755, 7), (760, 11), (773, 7), (780, 33), (802, 65), (816, 9), (858, 33),
                                    (865, 91), (871, 51), (876, 7), (903, 51), (927, 51), (928, 31), (944, 31), (950, 65), (991, 31)])
def test_regressions_found_by_the_stress_harness(emu, seed, k):
    """Inputs on which an earlier revision differed from the oracle (dotted successor rule; repeat-expansion work list)."""
    check_case(emu, cases.random_case(seed * 100 + k, k), k)


def test_reference_fixed_seqs(emu):   # tests.rs:131-148 inputs
    from test_oracle_kats import FIXED
    files = [(f"{n}.fasta", [(n, s.split("\n")[1])]) for n, s in zip("abcde", FIXED)]
    for k in (5, 9, 13, 51):
        check_case(emu, files, k)


def test_config1(emu, tmp_path):   # BASELINE.json configs[0]: 3 synthetic 100 kbp assemblies, k=51
    d = str(tmp_path / "cfg1")
    synth.write_assemblies(synth.make_assemblies("cfg1"), d)
    expected, yaml, st = o.compress_dir(d, 51)
    got = run_library(emu, d, 51)
    assert got["gfa"] == expected
    assert got["before"].n_kmers == st.n_kmers


def test_positions_match_oracle_seed_state(emu, tmp_path):
    """forward_positions / reverse_positions (unitig.rs:135-146) as multisets, on the graph after from_kmer_graph."""
    files = cases.random_case(4242, 9)
    d = str(tmp_path / "c"); cases.write_case(files, d)
    count, oseqs = o.load_sequences(d, 9)
    gfa, st, seed_dump = o.compress_seqs(oseqs, count, 9, want_seed_dump=True)
    got = run_library(emu, d, 9, positions=True)
    h = 9 // 2
    want = {}
    for line in seed_dump.splitlines():
        seq, depth, fpos, rpos = line.split("\t")
        want[seq[h:len(seq) - h]] = (float(depth), sorted(fpos.split(",")), sorted(rpos.split(",")))
    have = {u["seq"]: (u["depth"], sorted(u["forward_positions"]), sorted(u["reverse_positions"])) for u in got["seed_state"]}
    # distinct unitigs can share a trimmed sequence; compare only unambiguous ones, but require full coverage by count
    assert len(got["seed_state"]) == len(seed_dump.splitlines())
    for seq, val in have.items():
        if sum(1 for u in got["seed_state"] if u["seq"] == seq) == 1 and seq in want:
            assert want[seq] == val


def test_error_behaviour(emu, tmp_path):
    # even k / tiny k are refused like compress.rs:56-58 (the C ABI accepts 3..511 odd; the CLI the reference's 11..501)
    with pytest.raises(api.AutocyclerGpuError):
        api.KmerGraph(10, lib=emu)
    with pytest.raises(api.AutocyclerGpuError):
        api.KmerGraph(513, lib=emu)
    api.KmerGraph(501, lib=emu)
    # non-ACGT input (sequence.rs:40-42)
    d = tmp_path / "bad"; d.mkdir(); (d / "a.fasta").write_text(">a\nACGTNNACGTACGTACGT\n")
    with pytest.raises(api.AutocyclerGpuError, match="non-ACGT"):
        api.load_sequences(str(d), 5, lib=emu)
    # duplicate names (misc.rs:189-193)
    d2 = tmp_path / "dup"; d2.mkdir(); (d2 / "a.fasta").write_text(">a\nACGTACGT\n>a\nACGTACGA\n")
    with pytest.raises(api.AutocyclerGpuError, match="duplicate name"):
        api.load_sequences(str(d2), 5, lib=emu)
    # no assemblies (misc.rs:79-81)
    d3 = tmp_path / "empty"; d3.mkdir()
    with pytest.raises(api.AutocyclerGpuError, match="no assemblies found"):
        api.load_sequences(str(d3), 5, lib=emu)
    # too many contigs (compress.rs:84-95)
    d4 = tmp_path / "many"; d4.mkdir()
    (d4 / "a.fasta").write_text("".join(f">c{i}\nACGTACGTAC\n" for i in range(5)))
    with pytest.raises(api.AutocyclerGpuError, match="exceeds the allowed"):
        api.load_sequences(str(d4), 5, max_contigs=2, lib=emu)


def test_file_discovery_and_gz(emu, tmp_path):   # misc.rs:64-95 incl. the precedence quirk, misc.rs:233-245 gzip sniffing
    import gzip
    d = tmp_path / "in"; d.mkdir()
    seq = "CTTATGAGCAGTCCTTAACGTAGCGGTGTGTGGCTTTGAGAAGTTAGCGG"
    (d / "a.fasta").write_text(f">a\n{seq}\n")
    (d / "b.fna.gz").write_bytes(gzip.compress(f">b desc\n{seq[:25]}\n{seq[25:]}\n".encode()))
    (d / "c.fa.bak").write_text(f">c\n{seq}\n")          # qualifies through the reference's && / || precedence
    (d / "d.txt").write_text(f">d\n{seq}\n")             # ignored
    (d / "e.fasta").write_text(f">e\r\n{seq.lower()}\r\n\r\n")   # CRLF, lower case, blank line
    count, oseqs = o.load_sequences(str(d), 11)
    kg, seqs, n = api.load_sequences(str(d), 11, lib=emu)
    assert n == count == 4
    assert [(s.id, s.filename, s.contig_header, s.length, s.forward_seq) for s in seqs] == oseqs


def test_cli_yaml_and_gfa_files(emu, tmp_path):
    """ac_compress_dir writes both files; the YAML sidecar matches the oracle's rendering (metrics.rs:65-107)."""
    d = str(tmp_path / "cfg"); out = str(tmp_path / "out")
    synth.write_assemblies(synth.make_assemblies("x", n_assemblies=3, replicon_lengths=[5000], seed=7), d)
    api.compress(d, out, 51, lib=emu)
    expected, yaml, st = o.compress_dir(d, 51)
    assert open(os.path.join(out, "input_assemblies.gfa")).read() == expected
    assert open(os.path.join(out, "input_assemblies.yaml")).read() == yaml


@pytest.mark.parametrize("env", [{"AC_EXPAND_MIN_DUE": "1"}, {"AC_EXPAND_MIN_DUE": "1", "AC_EXPAND_TIGHT_ARENA": "1"}, {"AC_EXPAND_SERIAL": "1"},
                                 {"AC_HOST_POOL": "0", "AC_HOST_THREADS": "3"}, {"AC_CHECK_CANDIDATES": "1"}, {"AC_HOST_CANDIDATES": "1"},
                                 {"AC_DEVICE_TIGHT_ARENA": "1"}])
def test_repeat_expansion_schedules_agree(emu, env):
    """simplify_structure has three schedules (serial sweep; conflict levels on several threads; the same with every
    relocation handed back to the barrier) and two sources of its work list (device kernels; the host listing, which
    AC_CHECK_CANDIDATES compares with the device's field by field).  The switches are read once per process, so each
    runs in a child."""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import cases\nfrom autocycler_b200 import api\nfrom parity_common import check_case\n"
            "lib = api.load_library(%r)\n"
            "for k in (5, 9, 31, 51):\n"
            "    for seed in range(25):\n"
            "        check_case(lib, cases.random_case(7000 * k + seed, k), k)\n"
            "print('AGREE')\n") % (os.path.join(ROOT, "tests"), ROOT, os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))
    r = subprocess.run([os.sys.executable, "-c", code], env={**os.environ, **env}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "AGREE" in r.stdout, r.stderr[-2000:]


def _load(emu, text):
    g, seqs = api.UnitigGraph.from_gfa_lines(text, lib=emu)
    return g, seqs


@pytest.mark.parametrize("n", range(1, 15))
def test_gfa_loader_on_the_reference_fixtures(emu, golden_dir, n):   # test_gfa.rs:15-287 through ac_load_gfa
    text = open(os.path.join(golden_dir, f"ref_test_gfa_{n}.gfa")).read()
    g, seqs = _load(emu, text)
    assert g.gfa_bytes().decode() == o.gfa_roundtrip(text)                            # save(load(x)) as the reference's loader + writer give it
    api.merge_linear_paths(g, seqs)
    assert g.gfa_bytes().decode() == o.gfa_merge_linear_paths(text)


def test_gfa_loader_round_trip_on_compress_output(emu):
    """load(save(graph)) behaves like the graph: same text again, every sequence reconstructed (decompress.rs:83-105),
    simplify_structure idempotent, merge_linear_paths + renumber as the oracle does them on the loaded file."""
    for k, seed in [(5, 1), (9, 2), (31, 3), (51, 4), (91, 5), (51, 6), (9, 7), (31, 8)]:
        files = cases.random_case(8800 * k + seed, k)
        got = check_case(emu, files, k)
        if got is None:
            continue
        gfa = got["gfa"]
        g, seqs = _load(emu, gfa)
        assert g.gfa_bytes().decode() == gfa
        originals = [s.forward_seq[k // 2: len(s.forward_seq) - k // 2] for s in got["seqs"]]
        assert [g.reconstruct_original_sequence(i) for i in range(len(originals))] == originals
        assert [(s.id, s.filename, s.contig_header, s.length) for s in seqs] == [(s.id, s.filename, s.contig_header, s.length) for s in got["seqs"]]
        api.simplify_structure(g)
        assert g.gfa_bytes().decode() == gfa
        api.merge_linear_paths(g, seqs)
        assert g.gfa_bytes().decode() == o.gfa_merge_linear_paths(gfa)
        g.renumber_unitigs()
        assert g.gfa_bytes().decode() == o.gfa_merge_linear_paths(gfa, renumber=True)
        g2, seqs2 = _load(emu, gfa)                        # the `&vec![]` form on a loaded graph (clean.rs:114)
        api.merge_linear_paths(g2, None)
        strip = lambda t: [l for l in t.splitlines() if l[0] != "P"]
        assert strip(g2.gfa_bytes().decode()) == strip(o.gfa_merge_linear_paths(gfa, use_paths=False))


def test_gfa_loader_errors(emu):   # unitig_graph.rs:91-157, unitig.rs:62-77
    base = "H\tVN:Z:1.0\tKM:i:9\nS\t1\tACGT\tDP:f:2.00\nS\t2\tTTGCA\tDP:f:1.00\nL\t1\t+\t2\t+\t0M\nL\t2\t-\t1\t-\t0M\nP\t1\t1+,2+\t*\tLN:i:9\tFN:Z:a.fasta\tHD:Z:c1\n"
    g, seqs = _load(emu, base)
    assert g.gfa_bytes().decode() == base and g.reconstruct_original_sequence(0) == "ACGTTTGCA"
    for bad, msg in [(base.replace("DP:f:2.00", "DP:f:0x10"), "depth tag"), (base.replace("\tDP:f:1.00", ""), "depth tag"),
                     (base.replace("0M\nL", "3M\nL"), "non-zero overlap"), (base.replace("L\t1\t+\t2", "L\t1\t+\t7"), "nonexistent unitig: 7"),
                     (base.replace("\tFN:Z:a.fasta", ""), "missing required tag"), (base.replace("LN:i:9", "LN:i:10"), "Position calculation mismatch"),
                     (base.replace("1+,2+", "1+,3+"), "unitig 3 not found"), (base.replace("1+,2+", "1+,2"), "Invalid path strand")]:
        with pytest.raises(api.AutocyclerGpuError, match=msg):
            _load(emu, bad)


def test_decompress_command(emu, tmp_path):   # decompress.rs:83-137 against the oracle's restatement of save_original_seqs_to_dir
    import gzip
    files = cases.random_case(424242, 31)
    files = [(fn + (".gz" if i == 1 else ""), recs) for i, (fn, recs) in enumerate(files)]      # one gzipped input -> one gzipped output
    d = tmp_path / "in"; cases.write_case(files, str(d))
    gfa, yaml, st = o.compress_dir(str(d), 31)
    gfa_path = tmp_path / "g.gfa"; gfa_path.write_text(gfa)
    want, got = tmp_path / "want", tmp_path / "got"
    want.mkdir()
    o.decompress(gfa, str(want))
    api.decompress(str(gfa_path), out_dir=str(got), out_file=str(tmp_path / "all.fasta"), lib=emu)
    assert sorted(os.listdir(want)) == sorted(os.listdir(got))
    single = ""
    for fn in sorted(os.listdir(want)):
        rd = (lambda p: gzip.open(p, "rb").read()) if fn.endswith(".gz") else (lambda p: open(p, "rb").read())
        assert rd(os.path.join(want, fn)) == rd(os.path.join(got, fn))
        for block in rd(os.path.join(want, fn)).decode().split(">")[1:]:
            single += ">" + fn.replace(" ", "_") + "__" + block
    assert open(tmp_path / "all.fasta").read() == single
    with pytest.raises(api.AutocyclerGpuError, match="either --out_dir or --out_file is required"):
        api.decompress(str(gfa_path), lib=emu)
    with pytest.raises(api.AutocyclerGpuError, match="file does not exist"):
        api.decompress(str(tmp_path / "missing.gfa"), out_dir=str(got), lib=emu)


def test_reference_simplify_kats_through_the_library(emu, golden_dir):
    """graph_simplification.rs:627-671 (test_simplify_structure_1 / _2) run on the product: fixture -> ac_load_gfa ->
    simplify_structure -> unitig sequences in graph order, against the expectations the reference's own tests hold."""
    expect = {1: (["TTCGCTGCGCTCGCTTCGCTTT", "TGCCGTCGTCGCTGTGCA", "TGCCTGAATCGCCTA", "GCTCGGCTCG", "CGAACCAT", "TACTTGT", "GCCTT", "ATCT", "GC", "T"],
                  ["GCATTCGCTGCGCTCGCTTCGCTTT", "TGCCGTCGTCGCTGT", "CTGAATCGCCTA", "GCTCGGCTCGA", "CGAACCAT", "TACTTGT", "GCCT", "TCT", "GC", "T"]),
              2: (["ACCGCTGCGCTCGCTTCGCTCT", "ATGAT", "GCGC"], ["CACCGCTGCGCTCGCTTCGCTCTAT", "CG", "G"])}
    for n, (before, after) in expect.items():
        g, seqs = _load(emu, open(os.path.join(golden_dir, f"ref_test_gfa_{n}.gfa")).read())
        assert [u["seq"] for u in g.unitigs()] == before
        api.simplify_structure(g)
        assert [u["seq"] for u in g.unitigs()] == after


def test_reference_merge_kats_through_the_library(emu, golden_dir):   # graph_simplification.rs:742-801 on the product
    def merged(n):
        g, seqs = _load(emu, open(os.path.join(golden_dir, f"ref_test_gfa_{n}.gfa")).read())
        api.merge_linear_paths(g, seqs)
        return {u["number"]: u["seq"] for u in g.unitigs()}
    assert merged(3) == {8: "TTCGCTGCGCTCGCTTCGCTTTTGCACAGCGACGACGGCATGCCTGAATCGCCTA", 9: "GCTCGGCTCGATGGTTCG", 10: "TACTTGTAAGGC"}
    assert merged(4) == {6: "ACGACTACGAGCACGAGTCGTCGTCGTAACTGACT", 7: "GCTCGGTG"}
    m5 = merged(5)
    assert len(m5) == 5 and m5[7] == "AAATGCGACTGTG"
    assert len(merged(14)) == 11


def test_pairwise_distances_on_loaded_graphs_and_header_flags(emu, golden_dir):   # cluster.rs:132-176, sequence.rs:96-135
    text = open(os.path.join(golden_dir, "ref_test_gfa_14.gfa")).read()
    g, seqs = _load(emu, text)
    assert g.distance_matrix_text() == o.pairwise_distances(text)
    d = g.pairwise_contig_distances()
    assert d[0][0] == 0.0 and abs(d[0][1] - 0.01980198) < 1e-8 and abs(d[2][0] - 0.01052632) < 1e-8      # asymmetric by construction
    flagged = text.replace("HD:Z:a_2", "HD:Z:a_2 Autocycler_Trusted autocycler_cluster_weight=3").replace("HD:Z:b_2", "HD:Z:b_2 autocycler_consensus_weight=2 autocycler_ignore")
    assert flagged != text
    g, seqs = _load(emu, flagged)
    out = g.distance_matrix_text()
    assert out == o.pairwise_distances(flagged)
    assert "[trusted, cluster weight = 3]" in out and "[ignored, consensus weight = 2]" in out


def test_general_graphs_fractional_depths_colours_crlf(emu):
    """What compress never writes but later commands do (unitig.rs:62-91, 167-181): any f64 depth, segment colours, and files with
    CRLF line ends (BufRead::lines, misc.rs:51-61).  save(load(x)), merge_linear_paths (depth = get_merge_path_depth,
    graph_simplification.rs:503-526: position count, else the first anchor's depth, else the length-weighted mean; type
    Consentig when the path holds an anchor or a consentig) and renumbering, all against the oracle."""
    with_paths = ("H\tVN:Z:1.0\tKM:i:9\nS\t1\tACGT\tDP:f:2.345\tCL:Z:forestgreen\nS\t2\tTTGCA\tDP:f:1.005\nS\t3\tGG\tDP:f:7.5\tCL:Z:pink\n"
                  "L\t1\t+\t2\t+\t0M\nL\t2\t-\t1\t-\t0M\nL\t2\t+\t3\t+\t0M\nL\t3\t-\t2\t-\t0M\n"
                  "P\t1\t1+,2+,3+\t*\tLN:i:11\tFN:Z:a.fasta\tHD:Z:c1\nP\t2\t3-,2-,1-\t*\tLN:i:11\tFN:Z:b.fasta\tHD:Z:c2\n")
    no_paths = "".join(l + "\n" for l in with_paths.splitlines() if not l.startswith("P"))
    no_anchor = no_paths.replace("\tCL:Z:forestgreen", "").replace("CL:Z:pink", "CL:Z:steelblue")
    plain = no_paths.replace("\tCL:Z:forestgreen", "").replace("\tCL:Z:pink", "")
    for text in (with_paths, no_paths, no_anchor, plain, with_paths.replace("\n", "\r\n")):
        g, seqs = _load(emu, text)
        assert g.gfa_bytes().decode() == o.gfa_roundtrip(text.replace("\r\n", "\n"))
    # the advisor's case: (len 4, DP 1) + (len 8, DP 3) merged without positions -> 2.33
    two = "H\tVN:Z:1.0\tKM:i:9\nS\t1\tACGT\tDP:f:1.00\nS\t2\tTTGCATTG\tDP:f:3.00\nL\t1\t+\t2\t+\t0M\nL\t2\t-\t1\t-\t0M\n"
    g, seqs = _load(emu, two)
    api.merge_linear_paths(g, None)
    out = g.gfa_bytes().decode()
    assert out == o.gfa_merge_linear_paths(two, use_paths=False) and "DP:f:2.33" in out
    for text in (with_paths, no_paths, no_anchor, plain):
        for use_paths in (True, False):
            g, seqs = _load(emu, text)
            api.merge_linear_paths(g, seqs if use_paths else None)
            strip = (lambda t: t) if use_paths else (lambda t: [l for l in t.splitlines() if l[0] != "P"])      # the `&vec![]` form saves no paths
            assert strip(g.gfa_bytes().decode()) == strip(o.gfa_merge_linear_paths(text, use_paths=use_paths)), (text, use_paths)
            g.renumber_unitigs()
            assert strip(g.gfa_bytes().decode()) == strip(o.gfa_merge_linear_paths(text, use_paths=use_paths, renumber=True))


def test_simplify_with_more_than_six_exclusive_inputs(emu):
    """A loaded graph may give one unitig any number of exclusive inputs (the reference handles any count, graph_simplification.rs:233-255);
    the candidate record holds six inline and reads longer lists from the links."""
    tail = "ACGTTGCA"
    lines = ["H\tVN:Z:1.0\tKM:i:9", "S\t1\tGGATCCGATT\tDP:f:1.00"]
    n_in = 9
    for i in range(n_in):
        lines.append("S\t%d\t%s\tDP:f:1.00" % (i + 2, "ACGT"[i % 4] * (3 + i) + "C" + tail))
    for i in range(n_in):
        lines += ["L\t%d\t+\t1\t+\t0M" % (i + 2), "L\t1\t-\t%d\t-\t0M" % (i + 2)]
    text = "\n".join(lines) + "\n"
    g, seqs = _load(emu, text)
    api.simplify_structure(g)
    want = o.gfa_unitig_seqs(text, simplify=True)
    assert [(str(u["number"]), u["seq"]) for u in g.unitigs()] == [(w[0], w[1]) for w in want]
    assert any(u["seq"].startswith("C" + tail) or u["seq"].startswith(tail) for u in g.unitigs())      # the common end moved onto unitig 1


def test_kmer_depth_beyond_the_slot_count_takes_the_side_counts(tmp_path):
    """A k-mer with more occurrences than the 20-bit slot count may show (2^19; the test lowers the alarm to 1000, AC_COUNT_ALARM) trips
    the count alarm; the build repeats with 32-bit counts in the side array and still matches the oracle.  Runs in a child: the
    threshold is read once per process."""
    import subprocess
    import sys
    code = ("import sys, random; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from autocycler_b200 import api\nfrom parity_common import check_case\n"
            "rnd = random.Random(7); flank = lambda n: ''.join(rnd.choice('ACGT') for _ in range(n))\n"
            "files = [('a.fasta', [('c1', flank(300) + 'A' * 3000 + flank(300))]), ('b.fasta', [('c2', flank(200) + 'T' * 800 + flank(200))])]\n"
            "got = check_case(api.load_library(%r), files, 11)\n"
            "assert max(u['depth'] for u in got['graph'].unitigs()) > 1000\nprint('SIDE COUNTS OK')\n") % (os.path.join(ROOT, "tests"), ROOT, os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))
    for env in ({"AC_COUNT_ALARM": "1000"}, {"AC_BIG_COUNTS": "1"}):
        r = subprocess.run([sys.executable, "-c", code], env={**os.environ, **env}, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "SIDE COUNTS OK" in r.stdout, r.stderr[-2000:]


@pytest.mark.parametrize("n_devices", [2, 3, 5])
def test_several_devices_in_one_process(emu, tmp_path, n_devices):
    """ac_config.n_devices > 1: one process, one pipeline per device, the assemblies sharded by file, the peers' exports read in place
    (peer memory on the GPU box, plain memory under emulation).  Same bytes as the oracle, through the handle API and through
    ac_compress_dir_devices (`autocycler compress --devices`)."""
    for seed, k in [(31, 9), (32, 31), (33, 51), (34, 91)]:
        files = cases.random_case(7000 * k + seed, k)
        d = str(tmp_path / f"in{seed}"); cases.write_case(files, d)
        try:
            expected, yaml, st = o.compress_dir(d, k)
        except o.OracleError:
            continue
        count, oseqs = o.load_sequences(d, k)
        seqs = [api.Sequence(t[0], t[4], t[1], t[2], t[3]) for t in oseqs]
        kg = api.KmerGraph(k, lib=emu, devices=list(range(n_devices)))
        kg.add_sequences(seqs, count)
        g = api.UnitigGraph.compress(kg)
        assert bytes(g.gfa_view()).decode() == expected
        kg.upload()
        g = api.UnitigGraph.from_kmer_graph(kg)                       # the step-by-step form on the same devices
        api.simplify_structure(g)
        assert g.gfa_bytes().decode() == expected
        out = str(tmp_path / f"out{seed}")
        api.compress(d, out, k_size=max(k, 11) if k >= 11 else k, lib=emu, devices=list(range(n_devices))) if k >= 11 else None
        if k >= 11:
            assert open(os.path.join(out, "input_assemblies.gfa")).read() == expected and open(os.path.join(out, "input_assemblies.yaml")).read() == yaml


def test_stream_argument_semantics(emu):
    """ac_config.stream (include/autocycler_gpu.h): NULL = a private stream, otherwise the cudaStream_t to run on.  torch's default stream
    has the handle 0, which must not turn into "private" on the way (the N-rank build orders its collectives by the stream only when the
    library really runs on it: autocycler_b200/dist.py): it is handed over as cudaStreamLegacy."""
    assert api.stream_handle(None) is None and api.stream_handle(0) == 1 and api.stream_handle(0x7F00DEAD0000) == 0x7F00DEAD0000
    private, default, side = (api.KmerGraph(51, lib=emu, stream=s) for s in (None, 0, 0x7F00DEAD0000))
    assert not private._h.runs_on(0) and not private._h.runs_on(0x7F00DEAD0000)
    assert default._h.runs_on(0) and not default._h.runs_on(0x7F00DEAD0000)
    assert side._h.runs_on(0x7F00DEAD0000) and not side._h.runs_on(0)


DIFFERENT_KMERS_CODE = """
import os, random, sys, tempfile
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
import cases, oracle_lib as o
from autocycler_b200 import api
emu = api.load_library(%(lib)r)
n_devices = int(sys.argv[1])
for seed, k in [(1, 21), (2, 31), (3, 51)]:
    rng = random.Random(9000 + seed)
    shared = cases.rand_seq(rng, 700)
    files = []
    for f in range(2 * n_devices):
        own = cases.rand_seq(rng, rng.randint(900, 1600))
        cut = rng.randrange(100, 600)
        body = own[:400] + (shared[cut:] if f %% 3 == 0 else cases.rc(shared[:cut]) if f %% 3 == 1 else "") + own[400:]
        recs = [("c1 len=%%d" %% len(body), body)]
        if f %% 2:
            extra = cases.rand_seq(rng, rng.randint(k + 5, 300))
            recs.append(("c2 len=%%d" %% len(extra), extra))
        files.append(("asm_%%02d.fasta" %% f, recs))
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        expected, yaml, st = o.compress_dir(d, k)
        count, oseqs = o.load_sequences(d, k)
    seqs = [api.Sequence(t[0], t[4], t[1], t[2], t[3]) for t in oseqs]
    kg = api.KmerGraph(k, lib=emu, devices=list(range(n_devices)))
    kg.add_sequences(seqs, count)
    g = api.UnitigGraph.compress(kg)
    assert bytes(g.gfa_view()).decode() == expected, (seed, k)
print("SAME AS THE ORACLE")
"""


@pytest.mark.parametrize("n_devices", [2, 3, 4])
def test_devices_holding_different_kmers(emu, n_devices):
    """Ranks whose assemblies share little: the merged table then holds several times a rank's own k-mers, and the adjacency flags are
    computed for the rank's own ones only (pipeline.cu runs_local_w) — the stretch of the coordinate-ordered k-mer list between the
    words of its first and last coordinate.  Some files share a piece (so that k-mers claimed by one rank occur on another), contigs end
    inside shared pieces.  Same bytes as the oracle, in a child process whose device buffers are poisoned before every build (a flag
    nobody wrote would show) and which reports that the short route was taken."""
    import subprocess
    import sys
    code = DIFFERENT_KMERS_CODE % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")}
    r = subprocess.run([sys.executable, "-c", code, str(n_devices)], env={**os.environ, "AC_EMU_POISON": "1", "AC_HOST_PROFILE": "1"}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SAME AS THE ORACLE" in r.stdout, r.stderr[-2000:]
    assert "adjacency flags for this rank's own k-mers" in r.stderr
