"""`autocycler clean`, `autocycler gfa2fasta` and `autocycler table`: the reference's unit-test data (tests/golden/clean_kats.json, made
by extract_clean_kats.py), seeded random edits on the reference's GFA fixtures and on resolve's synthetic graphs, table over chain
directories, and the CLI, each checked against the CPU oracle (tests/clean_oracle.py).  These commands are host only: the CPU tests run
the product's code through the host-emulation library and the real binary; the test marked gpu runs the whole chain with the CUDA
build."""
import glob
import json
import os
import random
import shutil
import subprocess

import pytest

import clean_oracle as O
import resolve_oracle as R
from autocycler_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "clean_kats.json")))
FIXTURES = {int(os.path.basename(p)[13:-4]): open(p).read() for p in glob.glob(os.path.join(ROOT, "tests", "golden", "ref_test_gfa_*.gfa"))}
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def cli():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc")], check=True)
    return AUTOCYCLER


def _components(text):
    return R.Graph(text).connected_components()


def _counts(text):
    g = R.Graph(text)
    return len(g.order), sum(len(g.u[n]["seq"]) for n in g.order), list(O.link_count(g))


# ---- the reference's KATs ---------------------------------------------------------------------------------------------------------

def _run_graph_kat(steps, edit):
    """Runs a graph test's steps; edit(text, op, arg) -> the new text.  Checks every asserted value."""
    text = None
    for step in steps:
        op = step[0]
        if op == "load":
            text = FIXTURES[step[1]]
        elif op in ("remove", "duplicate", "low_depth", "merge"):
            text = edit(text, op, step[1] if len(step) > 1 else None)
        elif op == "components":
            assert _components(text) == step[1]
        else:
            got = dict(zip(("unitigs", "length", "links"), _counts(text)))[op]
            assert got == step[1], (op, step)


def _oracle_edit(text, op, arg):
    g = O._load(text)
    if op == "remove":
        O.remove_unitigs(g, set(arg))
    elif op == "duplicate":
        O.duplicate_unitig(g, arg)
    elif op == "low_depth":
        O.remove_low_depth_unitigs(g, arg)
    else:
        import oracle_lib
        return oracle_lib.gfa_merge_linear_paths(O.gfa_text(g, exact=True), use_paths=False, renumber=True)
    return O.gfa_text(g, exact=True)


def _product_edit(lib):
    def edit(text, op, arg):
        if op == "merge":
            return api.clean_text(text, merge=True, lib=lib)
        kw = {"remove": arg} if op == "remove" else {"duplicate": [arg]} if op == "duplicate" else {"min_depth": arg}
        return api.clean_text(text, merge=False, lib=lib, **kw)
    return edit


@pytest.mark.parametrize("name", sorted(KATS["graph_edits"]))
def test_graph_kats_oracle(name):
    _run_graph_kat(KATS["graph_edits"][name], _oracle_edit)


@pytest.mark.parametrize("name", sorted(KATS["graph_edits"]))
def test_graph_kats_emu(emu, name):
    _run_graph_kat(KATS["graph_edits"][name], _product_edit(emu))


def test_parse_tig_numbers_kats(emu, tmp_path, cli):
    for text, want in KATS["parse_tig_numbers"]["ok"]:
        assert O.parse_tig_numbers(text) == want
    for text in KATS["parse_tig_numbers"]["error"]:
        with pytest.raises(ValueError):
            O.parse_tig_numbers(text)
    # the product parses the CLI's text: each list on fixture 1 (tigs 1-10) is accepted, or refused with the reference's messages
    (tmp_path / "g.gfa").write_text(FIXTURES[1])
    for text, want in KATS["parse_tig_numbers"]["ok"]:
        if text is None:
            continue
        if max(want) > 10:
            with pytest.raises(api.AutocyclerGpuError, match=f"does not contain tig {[n for n in want if n > 10][0]}"):
                api.clean(str(tmp_path / "g.gfa"), str(tmp_path / "o.gfa"), remove=text, lib=emu)
            continue
        api.clean(str(tmp_path / "g.gfa"), str(tmp_path / "o.gfa"), remove=text, lib=emu)
        assert (tmp_path / "o.gfa").read_text() == O.clean(FIXTURES[1], remove=want)
    for text in KATS["parse_tig_numbers"]["error"]:
        item = next(s for s in text.replace(" ", "").split(",") if not s.isdigit())
        with pytest.raises(api.AutocyclerGpuError, match=f"failed to parse '{item}' as a node number"):
            api.clean(str(tmp_path / "g.gfa"), str(tmp_path / "o.gfa"), remove=text, lib=emu)


@pytest.mark.parametrize("case", KATS["gfa2fasta"], ids=[c["test"] for c in KATS["gfa2fasta"]])
def test_gfa2fasta_kats(emu, case):
    assert O.gfa2fasta(FIXTURES[case["fixture"]])[0] == case["fasta"]
    assert api.gfa_fasta_text(FIXTURES[case["fixture"]], lib=emu) == case["fasta"]


def test_table_selection_kats():
    one = KATS["one_copy"]
    for name, want in one["found"]:
        assert O.get_one_copy_yaml(one["files"], name) == want
    for name in one["error"]:
        with pytest.raises(O.TableError, match=f"Multiple {name} files found"):
            O.get_one_copy_yaml(one["files"], name)
    multi = KATS["multi_copy"]
    for name, want in multi["found"]:
        assert O.get_multi_copy_yaml(multi["files"], name) == want
    for text, want in KATS["parse_fields"]["ok"]:
        assert O.parse_fields(text) == want
    for text in KATS["parse_fields"]["error"]:
        with pytest.raises(O.TableError):
            O.parse_fields(text)
    assert O.FIELD_NAMES == KATS["field_names"]


def _yaml_scalar(v):
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, float):
        return repr(v)
    return str(v)


def _yaml(v, indent=""):
    """A value of consensus_assembly_bases as serde_yaml writes it (lists of scalars and single-level mappings)."""
    if isinstance(v, list):
        return "\n" + "".join(f"{indent}- {_yaml_scalar(x)}\n" for x in v)
    if isinstance(v, tuple):
        return "\n" + "".join(f"{indent}  {_yaml_scalar(k)}: {_yaml_scalar(x)}\n" for k, x in v)
    return " " + _yaml_scalar(v) + "\n"


def _one_value(tmp_path, lib, value_yaml, sigfigs):
    d = tmp_path / "v"
    shutil.rmtree(d, ignore_errors=True)
    d.mkdir()
    (d / "consensus_assembly.yaml").write_text("consensus_assembly_bases:" + value_yaml)
    got = api.table(str(d), name="s", fields="consensus_assembly_bases", sigfigs=sigfigs, lib=lib)
    want = O.table(str(d), name="s", fields="consensus_assembly_bases", sigfigs=sigfigs)
    assert got == want
    return got[2:-1]


def test_format_kats(emu, tmp_path):
    for c in KATS["format_value"]:
        assert _one_value(tmp_path, emu, _yaml(c["value"]), c["sigfigs"]) == c["expected"]
    c = KATS["format_sequence"]
    assert _one_value(tmp_path, emu, _yaml(c["value"]), c["sigfigs"]) == c["expected"]
    c = KATS["format_mapping"]
    assert _one_value(tmp_path, emu, _yaml(tuple(tuple(x) for x in c["value"])), c["sigfigs"]) == c["expected"]


def test_format_float_sigfigs_kats(emu, tmp_path):
    for value, sigfigs, want in KATS["format_float_sigfigs"]:
        assert O.format_float_sigfigs(value, sigfigs) == want
        assert _one_value(tmp_path, emu, _yaml(value), sigfigs) == want


def test_format_float_edges(emu, tmp_path):
    """powi is __powidf2 (12345.6 at 3 sigfigs differs from pow()), non-finite values print NaN, large and tiny magnitudes."""
    assert O.format_float_sigfigs(12345.6, 3) == "12300"
    rng = random.Random(7)
    values = [12345.6, 0.5, 2.5, -2.5, 1e22, 1.5e300, 5e-324, 1e-310, 123456789012.345, 9.999999, 0.095, -0.0005]
    values += [rng.uniform(-1e6, 1e6) * 10 ** rng.randint(-12, 12) for _ in range(60)]
    for v in values:
        for s in range(1, 10):
            assert _one_value(tmp_path, emu, _yaml(v), s) == O.format_float_sigfigs(v, s), (v, s)
    for text in (".nan", ".inf", "-.inf"):
        assert _one_value(tmp_path, emu, " " + text + "\n", 3) == "NaN"


# ---- seeded random edits ----------------------------------------------------------------------------------------------------------

def _random_graphs():
    graphs = {f"fixture_{n}": t for n, t in sorted(FIXTURES.items())}
    from test_resolve import _synthetic
    for name, trimmed in sorted(_synthetic().items()):
        final = R.resolve_gfa(trimmed)
        graphs[f"resolve_{name}_bridged"] = final[0]
        graphs[f"resolve_{name}_final"] = final[2]
    return graphs


def _random_case(text, rng):
    g = R.Graph(text)
    nums = list(g.order)
    remove = rng.sample(nums, rng.randint(0, min(3, len(nums)))) if nums and rng.random() < 0.5 else []
    left = R.Graph(text)
    O.remove_unitigs(left, set(remove))
    ok = O.qualifying_duplicates(left)
    duplicate = rng.sample(ok, rng.randint(0, min(2, len(ok)))) if ok and rng.random() < 0.6 else []
    depths = sorted({left.u[n]["depth"] for n in left.order})
    min_depth = rng.choice(depths) if depths and rng.random() < 0.6 else (None if rng.random() < 0.7 else 0.5)
    return remove, duplicate, min_depth


def test_random_edits_emu(emu):
    rng = random.Random(2024)
    n = 0
    for name, text in _random_graphs().items():
        for _ in range(12):
            remove, duplicate, min_depth = _random_case(text, rng)
            for merge in (False, True):
                try:
                    want = O.clean(text, remove, duplicate, min_depth, merge)
                except ValueError as e:     # a duplicate that a removal made ineligible
                    with pytest.raises(api.AutocyclerGpuError, match=str(e)):
                        api.clean_text(text, remove, duplicate, min_depth, merge, lib=emu)
                    continue
                got = api.clean_text(text, remove, duplicate, min_depth, merge, lib=emu)
                assert got == want, (name, remove, duplicate, min_depth, merge)
                assert api.gfa_fasta_text(got, lib=emu) == O.gfa2fasta(got)[0]
                n += 1
    assert n > 300


def test_depth_ties(emu):
    """min_depth equal to a unitig's depth removes it (the test is depth > min_depth to keep)."""
    text = FIXTURES[1]
    for d in sorted({u["depth"] for u in R.Graph(text).u.values()}):
        for merge in (False, True):
            assert api.clean_text(text, min_depth=d, merge=merge, lib=emu) == O.clean(text, min_depth=d, merge=merge)


def test_refused_inputs_emu(emu):
    text = FIXTURES[4]
    dup = O.qualifying_duplicates(R.Graph(text))[0]
    with pytest.raises(api.AutocyclerGpuError, match=f"tig {dup} cannot be both removed and duplicated"):
        api.clean_text(text, remove=[dup], duplicate=[dup], lib=emu)
    with pytest.raises(api.AutocyclerGpuError, match=f"tig {dup} cannot be duplicated more than once"):
        api.clean_text(text, duplicate=[dup, dup], lib=emu)
    with pytest.raises(api.AutocyclerGpuError, match="the GFA does not contain tig 99"):
        api.clean_text(text, remove=[99], lib=emu)
    bad = next(n for n in R.Graph(FIXTURES[1]).order if n not in O.qualifying_duplicates(R.Graph(FIXTURES[1])))
    with pytest.raises(api.AutocyclerGpuError, match=f"unitig {bad} does not contain exactly two non-self links"):
        api.clean_text(FIXTURES[1], duplicate=[bad], lib=emu)


# ---- table on directories ---------------------------------------------------------------------------------------------------------

def _table_both(lib, d, **kw):
    try:
        want = O.table(d, **kw)
    except O.TableError as e:
        with pytest.raises(api.AutocyclerGpuError, match=str(e)):
            api.table(d, lib=lib, **kw)
        return None
    assert api.table(d, lib=lib, **kw) == want
    return want


def _chain_with_extras(lib, tmp_path):
    from test_resolve import _chain
    a = _chain(lib, tmp_path)
    # qc_fail clusters must be left out of the untrimmed and trimmed lists
    fails = sorted(glob.glob(str(a / "clustering" / "qc_fail" / "*")))
    passes = sorted(glob.glob(str(a / "clustering" / "qc_pass" / "*")))
    assert passes
    if fails:
        shutil.copy(a / passes[0] / "2_trimmed.yaml", os.path.join(fails[0], "2_trimmed.yaml"))
    return a


def _check_tables(lib, a, tmp_path):
    fields = ",".join(f for names in O.FIELD_NAMES.values() for f in names)
    assert _table_both(lib, None) == "name\t" + "\t".join(O.parse_fields(O.DEFAULT_FIELDS)) + "\n"
    row = _table_both(lib, str(a), name="s1")
    assert row.startswith("s1\t") and row.count("\t") == 14
    for s in range(1, 10):
        _table_both(lib, str(a), name="x", fields=fields, sigfigs=s)
    _table_both(lib, str(a) + "/", name="x", fields=fields)
    # a hand-written subsample.yaml as serde_yaml writes it, and quoted and empty contig descriptions
    (a / "subsample.yaml").write_text("input_read_count: 12345\ninput_read_bases: 678901234\ninput_read_n50: 15000\noutput_reads:\n"
                                      "- name: sample_01.fastq\n  count: 1000\n- name: 'it''s'\n  count: 2000\n")
    inp = (a / "input_assemblies.yaml").read_text()
    inp = inp.replace("input_assembly_details:\n", "input_assembly_details:\n- filename: extra.fasta\n  contigs:\n  - name: '1'\n"
                      "    description: ''\n    length: 5\n  - name: \"tab\\there\"\n    description: 'a: b #c'\n    length: 7\n  - name: x\n"
                      "    description: null\n    length: 1\n", 1)
    (a / "input_assemblies.yaml").write_text(inp)
    _table_both(lib, str(a), name="s2", fields=fields)
    for bad in ("--sigfigs", "field", "tab"):
        kw = {"sigfigs": 0} if bad == "--sigfigs" else {"fields": "input_read_count,abc"} if bad == "field" else {"name": "a\tb"}
        _table_both(lib, str(a), **kw)
    # two clustering.yaml files are an error
    (a / "copy").mkdir()
    shutil.copy(a / "clustering" / "clustering.yaml", a / "copy" / "clustering.yaml")
    assert _table_both(lib, str(a), name="s3") is None
    with pytest.raises(api.AutocyclerGpuError, match="directory does not exist"):
        api.table(str(tmp_path / "nope"), lib=lib)


def test_table_chain_emu(emu, tmp_path):
    a = _chain_with_extras(emu, tmp_path)
    _check_tables(emu, a, tmp_path)


def test_table_missing_files_and_parse_errors(emu, tmp_path):
    d = tmp_path / "t"
    (d / "a" / "b").mkdir(parents=True)
    (d / "a" / "b-c").mkdir(parents=True)
    (d / "a" / "qc_fail").mkdir(parents=True)
    (d / "a" / "b" / "1_untrimmed.yaml").write_text("untrimmed_cluster_size: 3\nuntrimmed_cluster_distance: 0.25\n")
    (d / "a" / "b-c" / "1_untrimmed.yaml").write_text("untrimmed_cluster_size: 4\nuntrimmed_cluster_distance: 1e-3\n")
    (d / "a" / "qc_fail" / "1_untrimmed.yaml").write_text("untrimmed_cluster_size: 9\n")
    (d / ".yaml").write_text("garbage: [1, 2\n")           # no extension: never read
    (d / "clustering.yaml").write_text("pass_cluster_count: 007\nfail_cluster_count: 0x1f\noverall_clustering_score: ~\n")
    warnings = []
    want = O.table(str(d), name="n", fields="untrimmed_cluster_size,untrimmed_cluster_distance,pass_cluster_count,fail_cluster_count,"
                   "overall_clustering_score,input_read_count", warnings=warnings)
    assert want == "n\t[3,4]\t[0.250,0.00100]\t007\t31\t\t\n"
    assert api.table(str(d), name="n", fields="untrimmed_cluster_size,untrimmed_cluster_distance,pass_cluster_count,fail_cluster_count,"
                     "overall_clustering_score,input_read_count", lib=emu) == want
    assert "Warning: subsample.yaml not found" in warnings
    (d / "consensus_assembly.yaml").write_text("consensus_assembly_bases: [1, 2]\n")
    with pytest.raises(api.AutocyclerGpuError, match="Failed to parse YAML file"):
        api.table(str(d), lib=emu)


# ---- the CLI ----------------------------------------------------------------------------------------------------------------------

def _run(*args):
    return subprocess.run([AUTOCYCLER, *args], capture_output=True, text=True)


def test_cli(cli, tmp_path):
    text = FIXTURES[4]
    g = tmp_path / "in.gfa"
    g.write_text(text)
    dup = O.qualifying_duplicates(R.Graph(text))[0]
    for args, kw in ((["-r", "1"], {"remove": [1]}), (["-d", str(dup)], {"duplicate": [dup]}), (["-m", "1.0"], {"min_depth": 1.0}),
                     (["--remove", "2, 3", "--min_depth", "2"], {"remove": [2, 3], "min_depth": 2.0}), ([], {})):
        out = tmp_path / "out.gfa"
        r = _run("clean", "-i", str(g), "-o", str(out), *args)
        assert r.returncode == 0 and r.stdout == "", r.stderr
        assert out.read_text() == O.clean(text, **kw)
        fa = tmp_path / "out.fasta"
        r = _run("gfa2fasta", "-i", str(out), "-o", str(fa))
        assert r.returncode == 0 and r.stdout == "", r.stderr
        want, counts = O.gfa2fasta(out.read_text())
        assert fa.read_text() == want
        for n, what in zip(counts, ("circular", "linear", "other")):
            assert f"{n} {what} sequence{'' if n == 1 else 's'}\n" in r.stderr
    errors = [
        (["clean", "-i", str(tmp_path / "no.gfa"), "-o", "x"], f"file does not exist: {tmp_path / 'no.gfa'}"),
        (["clean", "-i", str(g), "-o", "x", "-r", "1,X"], "failed to parse 'X' as a node number"),
        (["clean", "-i", str(g), "-o", "x", "-d", "99"], f"{g} does not contain tig 99"),
        (["clean", "-i", str(g), "-o", "x", "-r", str(dup), "-d", str(dup)], f"tig {dup} cannot be both removed and duplicated"),
        (["clean", "-i", str(g), "-o", "x", "-d", f"{dup},{dup}"], f"tig {dup} cannot be duplicated more than once"),
        (["clean", "-i", str(g), "-o", str(tmp_path / "nodir" / "x.gfa")], f"cannot write {tmp_path / 'nodir' / 'x.gfa'}"),
        (["gfa2fasta", "-i", str(tmp_path / "no.gfa"), "-o", "x"], f"file does not exist: {tmp_path / 'no.gfa'}"),
        (["table", "-a", str(tmp_path / "nope")], f"directory does not exist: {tmp_path / 'nope'}"),
        (["table", "-s", "0"], "--sigfigs must be 1 or greater"),
        (["table", "-f", "abc"], "abc is not a valid field name"),
        (["table", "-a", str(tmp_path), "-n", "a\tb"], "--name cannot contain tab characters"),
    ]
    for args, msg in errors:
        r = _run(*args)
        assert r.returncode == 1 and f"Error: {msg}\n" in r.stderr and r.stdout == "", (args, r.stderr)
    for args in (["clean", "-i", str(g)], ["gfa2fasta", "-o", "x"], ["clean", "-i", str(g), "-o", "x", "--bogus"], ["table", "-s", "x"]):
        assert _run(*args).returncode == 2
    r = _run("table")
    assert r.returncode == 0 and r.stdout == O.table()
    assert r.stdout.startswith("name\tinput_read_count\tinput_read_bases\t")
    (tmp_path / "clustering.yaml").write_text("pass_cluster_count: 2\n")
    r = _run("table", "-a", str(tmp_path), "-n", "s1", "-f", "pass_cluster_count,input_read_count")
    assert r.returncode == 0 and r.stdout == "s1\t2\t\n" and "Warning: subsample.yaml not found" in r.stderr


# ---- on the H100: the whole chain with the CUDA build ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_chain_gpu(tmp_path):
    lib = api.load_library()
    a = _chain_with_extras(lib, tmp_path)
    gfa = (a / "consensus_assembly.gfa").read_text()
    g = R.Graph(gfa)
    depths = sorted({g.u[n]["depth"] for n in g.order})
    min_depth = depths[0] if len(depths) == 1 else (depths[0] + depths[1]) / 2
    api.clean(str(a / "consensus_assembly.gfa"), str(tmp_path / "clean.gfa"), min_depth=min_depth, lib=lib)
    cleaned = (tmp_path / "clean.gfa").read_text()
    assert cleaned == O.clean(gfa, min_depth=min_depth)
    api.gfa2fasta(str(tmp_path / "clean.gfa"), str(tmp_path / "clean.fasta"), lib=lib)
    assert (tmp_path / "clean.fasta").read_text() == O.gfa2fasta(cleaned)[0]
    r = _run("table", "-a", str(a), "-n", "s1")
    assert r.returncode == 0 and r.stdout == O.table(str(a), name="s1")
    _check_tables(lib, a, tmp_path)
