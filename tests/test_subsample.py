"""`autocycler subsample` (subsample.rs): the product's sample_XX.fastq files and subsample.yaml against the CPU oracle
(tests/subsample_oracle.py) byte for byte; the reference's unit-test data (tests/golden/subsample_kats.json); the RNG, the shuffle and
the genome size on their own; window boundaries at every byte; the errors through the library and the CLI; and `table` over the result.
The CPU tests run the product's code through the host-emulation library (the kernels' bodies, serially); the tests marked gpu run the
CUDA build on the H100."""
import gzip
import json
import os
import subprocess

import pytest

import clean_oracle
import subsample_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "subsample_kats.json")))
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
GENOME = synth.make_genome(synth.SplitMix64(0x5AB5), 40_000)


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def builds():
    return [pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]


@pytest.fixture
def lib(request, emu):
    return request.getfixturevalue("gpu") if request.param == "gpu" else emu


def reads_of(lengths, seed=1):
    """One read per length, cut from GENOME (longer reads wrap around it)."""
    out = []
    for i, L in enumerate(lengths):
        name, seq, qual = next(synth.make_reads(GENOME, n_reads=1, length=L, seed=seed * 7919 + i))
        out.append((f"r{i} len={L}", seq, qual))
    return out


def check(lib, path, out_dir, genome_size="40k", count=4, depth=25.0, seed=0):
    """The product's files against the oracle's; returns the info."""
    info = api.subsample(path, out_dir, genome_size, count, depth, seed, lib=lib)
    want = O.subsample(path, genome_size, count, depth, seed)
    got = {f: open(os.path.join(out_dir, f), "rb").read() for f in sorted(os.listdir(out_dir))}
    assert sorted(got) == sorted(want)
    for f in want:
        assert got[f] == want[f], f
    return info


# ---- the reference's unit tests and the pieces on their own ----------------------------------------------------------------------
def test_oracle_kats():
    for text, value in KATS["parse_genome_size"]:
        assert O.parse_genome_size(text) == value, text
    for text in KATS["parse_genome_size_refused"]:
        with pytest.raises(O.GenomeSizeError):
            O.parse_genome_size(text)
    order = KATS["subsample_indices"]["read_order"]
    assert len(KATS["subsample_indices"]["cases"]) == 11
    for c in KATS["subsample_indices"]["cases"]:
        assert sorted(O.subsample_indices(c["count"], c["reads_per_subset"], order, c["i"])[0]) == c["expected"]


EXTRA_SIZES = [("inf", 2**64 - 1), ("-5", 0), ("nan", 0), ("+2.5", 3), ("-2.5", 0), ("1e3", 1000), ("1.25e-1k", 125), (".5", 1), ("5.", 5),
               ("2.5K", 2500), ("infk", 2**64 - 1), ("0.0000005g", 500), ("\t7m\n", 7000000)]
EXTRA_REFUSED = ["", "k", "0x10", "1e", "1_000", "5 k", "--5", "1.2.3"]


@pytest.mark.parametrize("build", builds(), indirect=False)
def test_genome_size_product(build, request, emu, tmp_path):
    lib = request.getfixturevalue("gpu") if build == "gpu" else emu
    for text, value in KATS["parse_genome_size"] + EXTRA_SIZES:
        assert O.parse_genome_size(text) == value, text
        assert api.genome_size(text, lib=lib) == value, text
    for text in KATS["parse_genome_size_refused"] + EXTRA_REFUSED:
        with pytest.raises(O.GenomeSizeError):
            O.parse_genome_size(text)
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.subsample(str(tmp_path / "missing.fq"), str(tmp_path / "o"), text, lib=lib)
        assert e.value.code == -6 and "cannot interpret genome size" in str(e.value)
    # valid sizes reach the settings checks and the info
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads_of([3000] * 40), path)
    for text, value in KATS["parse_genome_size"][:3]:
        info = api.subsample(path, str(tmp_path / f"o_{value}"), text, min_read_depth=1.0, lib=lib)
        assert info["genome_size"] == value


def test_chacha20_against_cryptography():
    cr = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    import struct
    import numpy as np
    for seed in (0, 1, 2**64 - 1):
        key = O.pcg32_key(seed)
        ks = cr.Cipher(cr.algorithms.ChaCha20(struct.pack("<8I", *key), bytes(16)), mode=None).encryptor().update(bytes(64 * 70))
        want = np.frombuffer(ks, dtype="<u4").tolist()
        assert O.chacha_blocks(key, 0, 70, rounds=20).tolist() == want


@pytest.mark.parametrize("seed", [0, 1, 2**53 + 1, 2**64 - 1])
def test_rng_and_shuffle_product(emu, seed):
    r = O.StdRng(seed)
    assert api.subsample_words(seed, 1100, lib=emu) == [r.next_u32() for _ in range(1100)]
    r20 = O.StdRng(seed, rounds=20)
    assert api.subsample_words(seed, 100, rounds=20, lib=emu) == [r20.next_u32() for _ in range(100)]
    for n in (0, 1, 2, 3, 13, 14, 100, 5000):
        assert api.subsample_shuffle(n, seed, lib=emu) == O.shuffle_order(n, seed)


def test_range_draw_rejects_and_carries():
    """random_range(..bound): the second word is drawn only when the low half exceeds bound.wrapping_neg(), and carries into the result."""
    class Words:
        def __init__(self, w): self.w = list(w)
        def next_u32(self): return self.w.pop(0)
    w = Words([0xFFFFFFFF, 7])
    assert O.random_below_u32(w, 3) == 2 and w.w == [7]                # low half 0xFFFFFFFD is not above 2^32 - 3: one word
    assert O.random_below_u32(Words([0x55555555, 0]), 3) == 0          # low half 0xFFFFFFFF: a second word, no carry
    assert O.random_below_u32(Words([0x55555555, 0xFFFFFFFF]), 3) == 1  # ... whose high half 2 carries
    assert O.random_below_u32(Words([0x80000000]), 2) == 1


# ---- the command against the oracle ------------------------------------------------------------------------------------------------
def case_reads(name):
    """-> (reads, write_reads options)"""
    if name == "lengths_0_to_200k":
        return reads_of([0, 1, 2, 0, 5, 17, 1000, 65535, 65536, 65537, 131072, 200_000] + [3000 + 97 * i for i in range(60)]), {}
    if name == "crlf":
        return reads_of([0] + [2000 + 13 * i for i in range(80)]), {"crlf": True}
    if name == "plus_header":
        return reads_of([1500] * 90), {"plus_header": True}
    if name == "no_final_newline":
        return reads_of([1800 + i for i in range(70)]), {"final_newline": False}
    if name == "no_final_newline_crlf":
        return reads_of([0] + [1800 + i for i in range(70)]), {"final_newline": False, "crlf": True}
    if name == "lower_iupac":
        reads = reads_of([2500] * 60)
        odd = bytes(b"acgtnRYKMSWBDHVN"[i % 16] for i in range(2500))
        return [(n, odd if i % 3 == 0 else s.lower(), q) for i, (n, s, q) in enumerate(reads)], {}
    if name.startswith("gz"):
        return reads_of([2200 + 31 * i for i in range(75)]), {"gz": True}
    raise KeyError(name)


CASES = ["lengths_0_to_200k", "crlf", "plus_header", "no_final_newline", "no_final_newline_crlf", "lower_iupac", "gz", "gz_two_members"]


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("name", CASES)
def test_inputs(lib, name, tmp_path):
    reads, opts = case_reads(name)
    path = str(tmp_path / ("r.fq.gz" if opts.get("gz") else "r.fq"))
    if name == "gz_two_members":
        synth.write_reads(reads[:30], str(tmp_path / "a.gz"), gz=True)
        synth.write_reads(reads[30:], str(tmp_path / "b.gz"), gz=True)
        with open(path, "wb") as f:
            f.write(open(tmp_path / "a.gz", "rb").read() + open(tmp_path / "b.gz", "rb").read())
    else:
        synth.write_reads(reads, path, **opts)
    info = check(lib, path, str(tmp_path / "out"), genome_size="5k", depth=20.0, seed=3)
    assert info["input_count"] == len(reads) and info["windows"] == 1


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("count", [2, 3, 4, 7, 64, 65, 100, 128, 129])
def test_counts(lib, count, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(synth.make_reads(GENOME, depth=60, n50=2500, seed=count), path)
    check(lib, path, str(tmp_path / "out"), count=count, seed=count)
    if count == 100:
        assert os.path.exists(tmp_path / "out" / "sample_100.fastq")


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("setting", ["equal", "just_above", "rps_zero", "n1", "n2", "n3"])
def test_subset_sizes(lib, setting, tmp_path):
    import math
    path = str(tmp_path / "r.fq")
    n = {"n1": 1, "n2": 2, "n3": 3, "rps_zero": 1}.get(setting, 50)
    reads = reads_of([1000 + 10 * i for i in range(n)])
    synth.write_reads(reads, path)
    bases = sum(len(r[1]) for r in reads)
    gsize = 100 if setting != "rps_zero" else 1
    depth = bases / gsize
    if setting == "just_above":
        depth = math.nextafter(depth, 0.0)
    if setting == "rps_zero":
        depth = 0.001
    info = check(lib, path, str(tmp_path / "out"), genome_size=str(gsize), count=3, depth=depth, seed=5)
    if setting == "equal":
        assert info["reads_per_subset"] == n
    if setting == "rps_zero":
        assert info["reads_per_subset"] == 0


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("crlf,gz", [(False, False), (True, False), (False, True), (True, True)], ids=["False", "True", "False-gz", "True-gz"])
def test_window_at_every_byte(lib, crlf, gz, tmp_path, monkeypatch):
    path = str(tmp_path / ("r.fq.gz" if gz else "r.fq"))
    synth.write_reads(reads_of([7, 0, 12, 3]), path, gz=gz, crlf=crlf, plus_header=True)
    size = len(O.read_bytes(path))
    want = O.subsample(path, "10", count=3, min_read_depth=1.0, seed=9)
    for w in range(1, size + 2):
        monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(w))
        out = tmp_path / f"o{w}"
        info = api.subsample(path, str(out), "10", 3, 1.0, 9, lib=lib)
        for f, data in want.items():
            assert open(out / f, "rb").read() == data, (w, f)
        assert (info["windows"] == 1) == (w > size - 1)


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_record_longer_than_window_and_one_pass_reuse(lib, tmp_path, monkeypatch):
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads_of([300, 5000, 20, 40_000, 2, 700] * 5), path)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", "100")
    small = check(lib, path, str(tmp_path / "small"), genome_size="1k", depth=3.0, seed=2)
    assert small["windows"] > 1
    monkeypatch.delenv("AC_SUBSAMPLE_WINDOW")
    one = check(lib, path, str(tmp_path / "one"), genome_size="1k", depth=3.0, seed=2)
    assert one["windows"] == 1 and one["bytes_scanned"] == small["bytes_scanned"] == os.path.getsize(path)


# ---- the shapes only the GPU reaches ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_more_reads_than_one_grid(gpu, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(synth.make_reads(GENOME, n_reads=(1 << 20) + 77, n50=30, sigma=0.8, seed=11), path)
    info = check(gpu, path, str(tmp_path / "out"), genome_size="100k", count=3, depth=3.0, seed=2**64 - 1)
    assert info["input_count"] == (1 << 20) + 77


@pytest.mark.gpu
def test_gpu_long_read_and_many_windows(gpu, tmp_path, monkeypatch):
    path = str(tmp_path / "r.fq")
    big = synth.make_genome(synth.SplitMix64(44), 5_000_000)
    reads = [next(synth.make_reads(big, n_reads=1, length=4_000_000, seed=1))] + list(synth.make_reads(big, n_reads=3000, n50=2000, seed=2))
    synth.write_reads(reads, path)
    check(gpu, path, str(tmp_path / "one"), genome_size="100k", count=4, depth=10.0, seed=1)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(1 << 20))
    info = check(gpu, path, str(tmp_path / "many"), genome_size="100k", count=100, depth=10.0, seed=1)
    assert info["windows"] > 1


# ---- errors ---------------------------------------------------------------------------------------------------------------------
def run_cli(*args):
    p = subprocess.run([AUTOCYCLER, "subsample", *args], capture_output=True, text=True)
    return p.returncode, p.stderr


@pytest.fixture(scope="module")
def cli():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc")], check=True)
    return AUTOCYCLER


SETTINGS = [  # (genome size, count, depth, what the first failing check says); the reads file and out_dir are valid
    ("abc", 1, 0.0, "cannot interpret genome size"),
    ("0", 1, 0.0, "--genome_size must be at least 1"),
    ("-3k", 4, 25.0, "--genome_size must be at least 1"),
    ("5k", 1, 0.0, "--count must be at least 2"),
    ("5k", 2, 0.0, "--min_read_depth must be greater than 0"),
    ("5k", 2, -1.0, "--min_read_depth must be greater than 0"),
]


@pytest.mark.parametrize("gsize,count,depth,msg", SETTINGS)
def test_settings_errors(emu, cli, tmp_path, gsize, count, depth, msg):
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads_of([100]), path)
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.subsample(path, str(tmp_path / "o"), gsize, count, depth, lib=emu)
    assert e.value.code == -6 and e.value.message == msg
    rc, err = run_cli("-r", path, "-o", str(tmp_path / "o2"), "-g", gsize, "-c", str(count), "-d", str(depth))
    assert rc == 1 and err.endswith(f"Error: {msg}\n")
    assert not os.path.exists(tmp_path / "o") and not os.path.exists(tmp_path / "o2")


def test_path_errors(emu, cli, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads_of([100]), path)
    open(tmp_path / "afile", "w").close()
    cases = [(str(tmp_path / "nope.fq"), str(tmp_path / "o"), f"file does not exist: {tmp_path / 'nope.fq'}", -6),
             (str(tmp_path), str(tmp_path / "o"), f"{tmp_path} is not a file", -6),
             (path, str(tmp_path / "afile"), f"{tmp_path / 'afile'} exists but is not a directory", -6),
             (path, str(tmp_path / "afile" / "sub"), f"failed to create directory {tmp_path / 'afile' / 'sub'}", -6)]
    for reads, out, msg, code in cases:
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.subsample(reads, out, "0", 1, 0.0, lib=emu)     # the path checks come before the settings'
        if "failed to create" in msg:
            with pytest.raises(api.AutocyclerGpuError) as e:
                api.subsample(reads, out, "5k", lib=emu)
        assert e.value.code == code and msg in str(e.value), (msg, str(e.value))
        rc, err = run_cli("-r", reads, "-o", out, "-g", "0" if "failed" not in msg else "5k", "-c", "1" if "failed" not in msg else "4")
        assert rc == 1 and msg in err


MALFORMED = [
    (b"@a\nAC\n+\nII\nb\nAC\n+\nII\n", 2, "expected '@' at the start of the header line"),
    (b"@a\nAC\n+\nII\n\n@b\nAC\n+\nII\n", 2, "expected '@' at the start of the header line"),
    (b"@a\nAC\n+\nII\n@b\nAC\n-\nII\n", 2, "expected '+' at the start of the separator line"),
    (b"@a\nAC\n+\nII\n@b\nACG\n+\nII\n@c\nA\n+\nI\n", 2, "sequence and quality lengths differ"),
    (b"@a\nAC\n+\nII\n@b\nAC\n+\n", 2, "truncated record"),
    (b"@a\nAC\n+\nII\n@b\nAC", 2, "truncated record"),
    (b"@a\r\nAC\r\n+\r\nII\r\n@b\r\nAC\r\n+\r\nI\r\n", 2, "sequence and quality lengths differ"),
    (b"@a\nAC\n+\nII\n\n", 2, "expected '@' at the start of the header line"),
]


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("k", range(len(MALFORMED)))
def test_malformed_fastq(lib, k, tmp_path):
    data, rec, why = MALFORMED[k]
    path = str(tmp_path / "r.fq")
    open(path, "wb").write(data)
    with pytest.raises(O.FastqError) as oe:
        O.parse_fastq(data)
    assert str(oe.value) == f"record {rec}: {why}"
    out = tmp_path / "out"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.subsample(path, str(out), "1", lib=lib)
    assert e.value.code == -6 and e.value.message == f"Error reading FASTQ file: record {rec}: {why}"
    assert out.is_dir() and os.listdir(out) == []


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_too_shallow(lib, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads_of([1000] * 10), path)
    for reads_path in (path, str(tmp_path / "empty.fq")):
        open(tmp_path / "empty.fq", "wb").close()
        with pytest.raises(O.TooShallow):
            O.subsample(reads_path, "1k")
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.subsample(reads_path, str(tmp_path / "out"), "1k", lib=lib)
        assert e.value.code == -6 and e.value.message == "input reads are too shallow to subset"
        assert os.listdir(tmp_path / "out") == []


def test_cli_surface(cli, tmp_path):
    usage = "Usage: autocycler subsample"
    rc, err = run_cli("-h")
    assert rc == 0 and err.startswith(usage)
    for args in ([], ["-r", "x"], ["-r", "x", "-o", "y"], ["-o", "y", "-g", "5k"]):
        rc, err = run_cli(*args)
        assert rc == 2 and err.startswith(usage), args
    rc, err = run_cli("-r", "x", "-o", "y", "-g", "5k", "--bogus")
    assert rc == 2 and err.startswith("error: unexpected argument '--bogus'")
    for flag, value in (("-c", "-1"), ("-c", "2.5"), ("-s", "1.5"), ("-s", "18446744073709551616"), ("-s", "-1"), ("-s", ""), ("-d", "abc"),
                        ("--count", "x")):
        rc, err = run_cli("-r", "x", "-o", "y", "-g", "5k", flag, value)
        assert rc == 2 and err.startswith(f"error: invalid value '{value}' for '{flag}'"), (flag, value)
    rc, err = run_cli("-r", "x", "-o", "y", "-g", "5k", "-c")
    assert rc == 2 and "a value is required for '-c'" in err


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2**53 + 1, 2**64 - 1])
def test_cli_seeds(gpu, cli, seed, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(synth.make_reads(GENOME, depth=50, n50=3000, seed=seed % 1000 + 1), path)
    rc, err = run_cli("-r", path, "-o", str(tmp_path / "out"), "-g", "40k", "-s", str(seed))
    assert rc == 0, err
    assert f"  --seed {seed}\n" in err
    for f, data in O.subsample(path, "40k", seed=seed).items():
        assert open(tmp_path / "out" / f, "rb").read() == data, f


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_table_over_subsample(lib, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(synth.make_reads(GENOME, depth=40, n50=4000, seed=8), path)
    d = tmp_path / "auto"
    api.subsample(path, str(d), "40k", lib=lib)
    row = api.table(str(d), name="s1")
    assert row == clean_oracle.table(str(d), name="s1")
    fields = row.rstrip("\n").split("\t")
    want = O.read_set_details([len(r[1]) for r in O.parse_fastq(open(path, "rb").read())])
    assert fields[1:4] == [str(v) for v in want]
