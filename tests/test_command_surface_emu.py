"""The commands' surface around the device work: the CLI's argument parsing (exit codes and messages), the setting and path checks that
run before any device work, unwritable outputs, malformed input graphs, and the two-call text getters of the C ABI.  The CLI links the
CUDA library, but every CLI case here stops before the device is touched; the library calls run through the host-emulation build.  The
successful runs of every command are covered by the command's own test file."""
import ctypes as C
import os
import pathlib
import subprocess

import pytest

from autocycler_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")

EINVAL, ERANGE, EIO, EINPUT = -1, -4, -5, -6

# a two-unitig graph with one path (the loader's test input of test_parity_emu.py), and the same with a link the loader refuses
GFA = "H\tVN:Z:1.0\tKM:i:9\nS\t1\tACGT\tDP:f:2.00\nS\t2\tTTGCA\tDP:f:1.00\nL\t1\t+\t2\t+\t0M\nL\t2\t-\t1\t-\t0M\nP\t1\t1+,2+\t*\tLN:i:9\tFN:Z:a.fasta\tHD:Z:c1\n"
BAD_GFA = GFA.replace("0M\nL", "3M\nL")
BAD_GFA_MESSAGE = "non-zero overlap found on the GFA link line.\nAre you sure this is an Autocycler-generated GFA file?"


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def cli():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc")], check=True)
    return lambda *args: subprocess.run([AUTOCYCLER, *map(str, args)], capture_output=True, text=True)


def _raises(fn):
    with pytest.raises(api.AutocyclerGpuError) as e:
        fn()
    return e.value.code, e.value.message


# ---- argument parsing -------------------------------------------------------------------------------------------------------------

USAGE = {c: f"Usage: autocycler {c} " for c in ("compress", "decompress", "trim", "cluster", "resolve", "combine", "dotplot")}
FIRST_FLAG = {"compress": "-i", "decompress": "-i", "trim": "-c", "cluster": "-a", "resolve": "-c", "combine": "-a", "dotplot": "-i"}


@pytest.mark.parametrize("command", sorted(USAGE))
def test_cli_arguments(cli, command):
    r = cli(command)
    assert r.returncode == 2 and r.stderr.startswith(USAGE[command]), r.stderr
    r = cli(command, "--bogus", "x")
    assert r.returncode == 2 and r.stderr.startswith(f"error: unexpected argument '--bogus'\n{USAGE[command]}"), r.stderr
    r = cli(command, FIRST_FLAG[command])
    assert r.returncode == 2 and r.stderr == f"error: a value is required for '{FIRST_FLAG[command]}'\n", r.stderr
    r = cli(command, "-h")
    if command == "decompress":           # decompress has no -h
        assert r.returncode == 2 and r.stderr.startswith(f"error: unexpected argument '-h'\n{USAGE[command]}"), r.stderr
    else:
        assert r.returncode == 0 and r.stderr.startswith(USAGE[command]), r.stderr
    assert r.stdout == ""


def test_cli_no_command(cli):
    for args in ((), ("frobnicate",)):
        r = cli(*args)
        assert r.returncode == 2 and r.stderr.startswith(USAGE["compress"]), r.stderr


@pytest.mark.parametrize("command,args,flag,value", [
    ("trim", ["-c", "d"], "--min_identity", "abc"),
    ("trim", ["-c", "d"], "--mad", "1.5x"),
    ("trim", ["-c", "d"], "--max_unitigs", "-5"),
    ("trim", ["-c", "d"], "--max_unitigs", "+5"),
    ("trim", ["-c", "d"], "--threads", ""),
    ("cluster", ["-a", "d"], "--cutoff", "x"),
    ("cluster", ["-a", "d"], "--min_assemblies", "-3"),
    ("cluster", ["-a", "d"], "--max_contigs", "2.5"),
])
def test_cli_invalid_number_with_usage(cli, command, args, flag, value):
    r = cli(command, *args, flag, value)
    assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'\n{USAGE[command]}"), r.stderr
    assert r.stderr.count("\n") == 2


@pytest.mark.parametrize("flag,value", [("--res", "abc"), ("--res", "-600"), ("--kmer", "4294967296"), ("--kmer", "")])
def test_cli_invalid_number_dotplot(cli, flag, value):
    r = cli("dotplot", "-i", "x", "-o", "y.png", flag, value)
    assert r.returncode == 2 and r.stderr == f"error: invalid value '{value}' for '{flag}'\n", r.stderr     # no usage line


def test_cli_numbers_that_parse(cli, tmp_path):
    """compress reads its numbers with an unchecked strtoul (text reads as its leading digits, or 0); dotplot's u32 options take a '+'."""
    (tmp_path / "asm").mkdir()
    for flag, value, message in (("--threads", "abc", "--threads cannot be less than 1"), ("--kmer", "9x", "--kmer cannot be less than 11"),
                                 ("--kmer", "50.9", "--kmer must be odd")):
        r = cli("compress", "-i", tmp_path / "asm", "-a", tmp_path / "out", flag, value)
        assert r.returncode == 1 and r.stderr.endswith(f"\nError: {message}\n"), r.stderr
    r = cli("dotplot", "-i", tmp_path / "asm", "-o", tmp_path / "x.png", "--res", "+499")
    assert r.returncode == 1 and r.stderr.endswith("\nError: --res cannot be less than 500\n"), r.stderr


def test_cli_devices_list(cli, tmp_path):
    r = cli("compress", "-i", tmp_path, "-a", tmp_path / "out", "--devices", "0;1")
    assert r.returncode == 2 and r.stderr == "error: --devices wants a comma-separated list of ordinals\n"


# ---- setting and path checks before any device work -------------------------------------------------------------------------------

def _layout(t):
    """t/file: a file; t/empty: an empty directory; t/good: every command's input, well formed; t/dirs: every input name a directory."""
    (t / "file").write_text("x\n")
    for d in ("empty", "good", "dirs"):
        (t / d).mkdir()
    for name in ("in.gfa", "1_untrimmed.gfa", "input_assemblies.gfa", "2_trimmed.gfa"):
        (t / "good" / name).write_text(GFA)
        (t / "dirs" / name).mkdir()


def _setting_cases(t):
    """-> {name: (CLI arguments, library call, message)}; every one is AC_EINPUT."""
    s = str
    good, empty, dirs = t / "good", t / "empty", t / "dirs"
    c = {
        "compress_missing_dir": (["compress", "-i", t / "nope", "-a", t / "out"], lambda lib: api.compress(s(t / "nope"), s(t / "out"), lib=lib),
                                 f"directory does not exist: {t / 'nope'}"),
        "compress_dir_is_file": (["compress", "-i", t / "file", "-a", t / "out"], lambda lib: api.compress(s(t / "file"), s(t / "out"), lib=lib),
                                 f"{t / 'file'} is not a directory"),
        "compress_out_is_file": (["compress", "-i", empty, "-a", t / "file"], lambda lib: api.compress(s(empty), s(t / "file"), lib=lib),
                                 f"{t / 'file'} exists but is not a directory"),
        "decompress_missing_file": (["decompress", "-i", t / "nope", "-f", t / "o.fa"], lambda lib: api.decompress(s(t / "nope"), out_file=s(t / "o.fa"), lib=lib),
                                    f"file does not exist: {t / 'nope'}"),
        "decompress_input_is_dir": (["decompress", "-i", empty, "-f", t / "o.fa"], lambda lib: api.decompress(s(empty), out_file=s(t / "o.fa"), lib=lib),
                                    f"{empty} is not a file"),
        "decompress_no_output": (["decompress", "-i", good / "in.gfa"], lambda lib: api.decompress(s(good / "in.gfa"), lib=lib),
                                 "either --out_dir or --out_file is required"),
        "decompress_out_is_file": (["decompress", "-i", good / "in.gfa", "-o", t / "file"], lambda lib: api.decompress(s(good / "in.gfa"), out_dir=s(t / "file"), lib=lib),
                                   f"{t / 'file'} exists but is not a directory"),
        "combine_missing_input": (["combine", "-a", t / "c", "-i", good / "in.gfa", t / "nope.gfa"],
                                  lambda lib: api.combine(s(t / "c"), [s(good / "in.gfa"), s(t / "nope.gfa")], lib=lib), f"file does not exist: {t / 'nope.gfa'}"),
        "combine_input_is_dir": (["combine", "-a", t / "c", "-i", empty], lambda lib: api.combine(s(t / "c"), [s(empty)], lib=lib), f"{empty} is not a file"),
        "combine_cannot_create": (["combine", "-a", t / "file" / "c", "-i", good / "in.gfa"], lambda lib: api.combine(s(t / "file" / "c"), [s(good / "in.gfa")], lib=lib),
                                  f"failed to create directory {t / 'file' / 'c'}\nNot a directory"),
    }
    for k, kw, message in ((9, {}, "--kmer cannot be less than 11"), (503, {}, "--kmer cannot be greater than 501"), (50, {}, "--kmer must be odd"),
                           (51, {"threads": 0}, "--threads cannot be less than 1"), (51, {"threads": 101}, "--threads cannot be greater than 100")):
        flags = ["--kmer", k] + (["--threads", kw["threads"]] if kw else [])
        c[f"compress_kmer{k}" + "".join(f"_threads{v}" for v in kw.values())] = (["compress", "-i", empty, "-a", t / "out", *flags],
                                    lambda lib, k=k, kw=kw: api.compress(s(empty), s(t / "out"), k, lib=lib, **kw), message)
    commands = {"trim": ("-c", "1_untrimmed.gfa", api.trim), "cluster": ("-a", "input_assemblies.gfa", api.cluster),
                "resolve": ("-c", "2_trimmed.gfa", api.resolve)}
    for command, (flag, name, fn) in commands.items():
        for case, d, message in (("missing_dir", t / "nope", f"directory does not exist: {t / 'nope'}"), ("dir_is_file", t / "file", f"{t / 'file'} is not a directory"),
                                 ("missing_input", empty, f"file does not exist: {empty / name}"), ("input_is_dir", dirs, f"{dirs / name} is not a file")):
            c[f"{command}_{case}"] = ([command, flag, d], lambda lib, fn=fn, d=d: fn(s(d), lib=lib), message)
    for cli_flags, kw, message in ((["--min_identity", "1.5"], {"min_identity": 1.5}, "--min_identity must be between 0.0 and 1 (inclusive)"),
                                   (["--min_identity", "-0.5"], {"min_identity": -0.5}, "--min_identity must be between 0.0 and 1 (inclusive)"),
                                   (["--threads", "0"], {"threads": 0}, "--threads cannot be less than 1"),
                                   (["--threads", "101"], {"threads": 101}, "--threads cannot be greater than 100"),
                                   (["--mad", "-1"], {"mad": -1.0}, "--mad cannot be less than 0")):
        c[f"trim_{cli_flags[0][2:]}_{cli_flags[1]}"] = (["trim", "-c", good, *cli_flags], lambda lib, kw=kw: api.trim(s(good), lib=lib, **kw), message)
    for cli_flags, kw, message in ((["--cutoff", "0"], {"cutoff": 0.0}, "--cutoff must be between 0 and 1 (exclusive)"),
                                   (["--cutoff", "1"], {"cutoff": 1.0}, "--cutoff must be between 0 and 1 (exclusive)"),
                                   (["--min_assemblies", "0"], {"min_assemblies": 0}, "--min_assemblies must be 1 or greater")):
        c[f"cluster_{cli_flags[0][2:]}_{cli_flags[1]}"] = (["cluster", "-a", good, *cli_flags], lambda lib, kw=kw: api.cluster(s(good), lib=lib, **kw), message)
    return c


SETTING_CASES = sorted(_setting_cases(pathlib.Path("/t")))       # the names only; each test builds its own layout


@pytest.mark.parametrize("case", SETTING_CASES)
def test_setting_errors(emu, cli, tmp_path, case):
    _layout(tmp_path)
    args, call, message = _setting_cases(tmp_path)[case]
    assert _raises(lambda: call(emu)) == (EINPUT, message)
    r = cli(*args)
    assert r.returncode == 1 and r.stderr.endswith(f"\nError: {message}\n"), r.stderr
    assert not (tmp_path / "out").exists() and not (tmp_path / "c").exists()


# ---- unwritable outputs -----------------------------------------------------------------------------------------------------------

def test_unwritable_outputs(emu, tmp_path):
    """A directory where an output file should go: the command fails with AC_EIO, and the message names the file (compress, decompress,
    trim) or the directory (resolve, combine)."""
    _layout(tmp_path)
    good = tmp_path / "good"
    asm = tmp_path / "asm"
    asm.mkdir()
    (asm / "a.fasta").write_text(">a\n" + "".join("ACGT"[(i * i + 3 * i) % 7 % 4] for i in range(400)) + "\n")
    (tmp_path / "out" / "input_assemblies.gfa").mkdir(parents=True)
    assert _raises(lambda: api.compress(str(asm), str(tmp_path / "out"), lib=emu)) == (EIO, f"cannot write {tmp_path / 'out' / 'input_assemblies.gfa'}")
    (tmp_path / "o.fa").mkdir()
    assert _raises(lambda: api.decompress(str(good / "in.gfa"), out_file=str(tmp_path / "o.fa"), lib=emu)) == (EIO, f"cannot write {tmp_path / 'o.fa'}")
    (good / "2_trimmed.gfa").unlink()
    (good / "2_trimmed.gfa").mkdir()
    assert _raises(lambda: api.trim(str(good), lib=emu)) == (EIO, f"cannot write {good / '2_trimmed.gfa'}")
    (good / "2_trimmed.gfa").rmdir()
    (good / "2_trimmed.gfa").write_text(GFA)
    (good / "3_bridged.gfa").mkdir()
    assert _raises(lambda: api.resolve(str(good), lib=emu)) == (EIO, f"cannot write the output files under {good}")
    (tmp_path / "c" / "consensus_assembly.gfa").mkdir(parents=True)
    assert _raises(lambda: api.combine(str(tmp_path / "c"), [str(good / "in.gfa")], lib=emu)) == (EIO, f"cannot write the output files under {tmp_path / 'c'}")


@pytest.mark.skipif(not os.path.exists("/dev/full"), reason="needs /dev/full")
def test_failing_close(emu, tmp_path):
    """An output file whose buffered bytes cannot be flushed (a link to /dev/full: opening and a short write succeed, closing fails) is
    AC_EIO as well."""
    _layout(tmp_path)
    good = tmp_path / "good"
    asm = tmp_path / "asm"
    asm.mkdir()
    (asm / "a.fasta").write_text(">a\n" + "".join("ACGT"[(i * i + 3 * i) % 7 % 4] for i in range(400)) + "\n")
    (tmp_path / "out").mkdir()
    for path in (tmp_path / "out" / "input_assemblies.gfa", tmp_path / "o.fa", good / "2_trimmed.gfa", good / "3_bridged.gfa"):
        if path.exists():
            path.unlink()
        path.symlink_to("/dev/full")
    # compress, decompress and trim ignored the result of fclose before the commands shared one file writer
    assert _raises(lambda: api.compress(str(asm), str(tmp_path / "out"), lib=emu)) == (EIO, f"cannot write {tmp_path / 'out' / 'input_assemblies.gfa'}")
    assert _raises(lambda: api.decompress(str(good / "in.gfa"), out_file=str(tmp_path / "o.fa"), lib=emu)) == (EIO, f"cannot write {tmp_path / 'o.fa'}")
    assert _raises(lambda: api.trim(str(good), lib=emu)) == (EIO, f"cannot write {good / '2_trimmed.gfa'}")
    (good / "2_trimmed.gfa").unlink()
    (good / "2_trimmed.gfa").write_text(GFA)
    assert _raises(lambda: api.resolve(str(good), lib=emu)) == (EIO, f"cannot write the output files under {good}")


def test_outputs_written(emu, tmp_path):
    """The same calls with the directories out of the way succeed (the test above fails for the reason it names)."""
    _layout(tmp_path)
    good = tmp_path / "good"
    api.decompress(str(good / "in.gfa"), out_dir=str(tmp_path / "d" / "e"), out_file=str(tmp_path / "o.fa"), lib=emu)
    assert (tmp_path / "o.fa").read_text() == ">a.fasta__c1\nACGTTTGCA\n"
    assert (tmp_path / "d" / "e" / "a.fasta").read_text() == ">c1\nACGTTTGCA\n"
    api.trim(str(good), lib=emu)
    assert (good / "2_trimmed.gfa").exists() and (good / "2_trimmed.yaml").exists()
    api.resolve(str(good), lib=emu)
    assert all((good / f).exists() for f in ("3_bridged.gfa", "4_merged.gfa", "5_final.gfa"))
    api.combine(str(tmp_path / "c"), [str(good / "5_final.gfa")], lib=emu)
    assert all((tmp_path / "c" / f"consensus_assembly.{e}").exists() for e in ("gfa", "fasta", "yaml"))


# ---- malformed input graphs -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("command", ["decompress", "trim", "cluster", "resolve"])
def test_malformed_gfa(emu, tmp_path, command):
    name = {"decompress": "in.gfa", "trim": "1_untrimmed.gfa", "cluster": "input_assemblies.gfa", "resolve": "2_trimmed.gfa"}[command]
    (tmp_path / name).write_text(BAD_GFA)
    call = {"decompress": lambda: api.decompress(str(tmp_path / name), out_file=str(tmp_path / "o.fa"), lib=emu),
            "trim": lambda: api.trim(str(tmp_path), lib=emu), "cluster": lambda: api.cluster(str(tmp_path), lib=emu),
            "resolve": lambda: api.resolve(str(tmp_path), lib=emu)}[command]
    code, message = _raises(call)
    assert message == BAD_GFA_MESSAGE
    assert code == EINPUT          # decompress reported AC_EINVAL before the commands shared one loader


# ---- the two-call text getters ----------------------------------------------------------------------------------------------------

def test_text_getters(emu):
    g, _ = api.UnitigGraph.from_gfa_lines(GFA, lib=emu)
    h = g._h
    getters = {"ac_distance_matrix_text": (), "ac_trim_yaml": (), "ac_cluster_text": (0, 0), "ac_resolve_text": (2,)}
    # before the call that makes the text
    for fn, msg in (("ac_trim_yaml", "ac_trim must precede ac_trim_yaml"), ("ac_cluster_text", "ac_cluster must precede ac_cluster_text"),
                    ("ac_resolve_text", "ac_resolve must precede ac_resolve_text")):
        n = C.c_uint64()
        assert getattr(emu, fn)(h.ptr, *getters[fn], None, 0, C.byref(n)) == EINVAL and emu.ac_last_error(h.ptr).decode() == msg
    want = {"ac_distance_matrix_text": g.distance_matrix_text()}
    g.cluster()
    want["ac_cluster_text"] = g.cluster_text("phylip")
    g.resolve()
    want["ac_resolve_text"] = g.resolve_text("final")
    g.trim()
    want["ac_trim_yaml"] = g.trimmed_yaml()
    for fn, args in getters.items():
        f = getattr(emu, fn)
        n = C.c_uint64(12345)
        assert f(h.ptr, *args, None, 0, C.byref(n)) == 0 and n.value == len(want[fn]) > 0, fn
        assert emu.ac_last_error(h.ptr) == b""
        buf = C.create_string_buffer(n.value)
        assert f(h.ptr, *args, buf, n.value - 1, C.byref(n)) == ERANGE, fn
        assert emu.ac_last_error(h.ptr).decode() == emu.ac_last_error(None).decode() == "buffer too small"
        assert buf.raw == b"\0" * len(buf.raw)                  # nothing was copied
        assert f(h.ptr, *args, buf, n.value, C.byref(n)) == 0 and buf.raw.decode() == want[fn], fn
        assert f(h.ptr, *args, None, 0, None) == EINVAL and emu.ac_last_error(h.ptr).decode() == "null argument"
    for fn, args, code, msg in (("ac_cluster_text", (9, 0), EINVAL, "unknown cluster text"), ("ac_cluster_text", (4, 99), ERANGE, "no cluster 99"),
                                ("ac_resolve_text", (7,), EINVAL, "unknown resolve text")):
        n = C.c_uint64()
        assert getattr(emu, fn)(h.ptr, *args, None, 0, C.byref(n)) == code and emu.ac_last_error(h.ptr).decode() == msg


def test_path_validation(emu):
    """ac_trim_paths and ac_bridge_best_paths check the caller's paths the same way: offsets that do not decrease, a weight per entry."""
    h = api._Handle(emu, 51)
    w = (C.c_uint32 * 3)(0, 10, 20)
    u64 = lambda *v: (C.c_uint64 * len(v))(*v)
    out, out_off, trimmed = (C.c_int32 * 8)(), u64(0, 0, 0), (C.c_uint8 * 2)()

    def trim(paths, off):
        rc = emu.ac_trim_paths(h.ptr, 0, (C.c_int32 * len(paths))(*paths), u64(*off), len(off) - 1, w, 3, 0.75, 5000, out, out_off, trimmed)
        return rc, emu.ac_last_error(h.ptr).decode()

    def bridge(paths, off, goff):
        totals, best, best_off = (C.c_uint32 * 4)(), (C.c_int32 * 8)(), u64(0, 0, 0)
        rc = emu.ac_bridge_best_paths(h.ptr, (C.c_int32 * len(paths))(*paths), u64(*off), len(off) - 1, u64(*goff), len(goff) - 1, w, 3,
                                      totals, best, best_off)
        return rc, emu.ac_last_error(h.ptr).decode()

    assert trim([1, 2], [0, 2, 1]) == (EINVAL, "path offsets must not decrease")
    assert trim([1, -3], [0, 1, 2]) == (EINVAL, "path entry -3 has no weight")
    assert trim([1, 0], [0, 1, 2]) == (EINVAL, "path entry 0 has no weight")
    assert trim([1, 2], [0, 1, 2])[0] == 0
    assert bridge([1, 2], [0, 2, 1], [0, 2]) == (EINVAL, "path offsets must not decrease")
    assert bridge([1, 3], [0, 1, 2], [0, 2]) == (EINVAL, "path entry 3 has no weight")
    assert bridge([1, 2], [0, 1, 2], [0, 2, 1, 2]) == (EINVAL, "group offsets must not decrease")
    assert bridge([1, 2], [0, 1, 2], [0, 1]) == (EINVAL, "the groups must cover the paths in order")
    assert bridge([1, 2], [0, 1, 2], [0, 2])[0] == 0
