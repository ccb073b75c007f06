"""`autocycler helper genome_size`: the genome size from the reads' canonical k-mer depth spectrum, counted on the GPU (DESIGN.md §18).
This command departs from the reference on purpose (the reference prints the length of a Raven assembly), so nothing here is compared
with the reference: the histogram and the estimate are pinned against the numpy oracle of the rule (tests/genome_size_oracle.py), the
rule alone on crafted histograms, and the estimate's accuracy on synthetic genomes of known size.  The CPU tests run the product's code
through the host-emulation library (the kernels' bodies, serially); the tests marked gpu run the CUDA build on the H100."""
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import genome_size_oracle as O
import subsample_oracle
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
GOLDENS = json.load(open(os.path.join(ROOT, "tests", "golden", "genome_size_goldens.json")))
H = O.H
GENOME = synth.make_genome(synth.SplitMix64(0x65A1), 30_000)


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", CSRC, "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def builds():
    return [pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]


@pytest.fixture
def lib(request, emu):
    return request.getfixturevalue("gpu") if request.param == "gpu" else emu


def check(lib, path, k, **kw):
    """The product's histogram and estimate against the oracle's; returns the info."""
    info = api.genome_size_estimate(path, k, lib=lib, **kw)
    want_hist, want_w = O.histogram(path, k)
    assert info["windows"] == want_w
    assert info["histogram"] == want_hist
    want = O.estimate(want_hist, want_w)
    for f in ("estimate", "valley", "peak", "peak_refined", "solid", "distinct"):
        assert info[f] == want[f], f
    return info


def deep_reads(genome=GENOME, depth=30, n50=2000, seed=1, err=0.01):
    return synth.make_noisy_reads(genome, depth=depth, n50=n50, seed=seed, sub=err / 2, ins=err / 4, dele=err / 4)


def oddities(seed):
    """Reads that exercise the packing: N and IUPAC bases, lowercase, short and empty reads, homopolymers, 32m-1 / 32m / 32m+1 lengths."""
    rng = np.random.default_rng(seed)
    out = []
    for i, (name, seq, qual) in enumerate(deep_reads(depth=20, seed=seed)):
        s = bytearray(seq)
        if i % 5 == 1:
            for at in rng.integers(0, max(1, len(s)), 3):
                if at < len(s):
                    s[at] = b"NRYKMSWBDHV"[int(at) % 11]
        if i % 7 == 2:
            s = bytearray(bytes(s).lower())
        if i % 11 == 3 and len(s) > 40:
            s[10:40] = s[10:40].lower()
        out.append((name, bytes(s), qual[:len(s)]))
    for L in (0, 1, 10, 20, 21, 22, 30, 31, 32, 33, 63, 64, 65, 95, 96, 97):
        name, seq, qual = next(synth.make_reads(GENOME, n_reads=1, length=L, seed=seed * 31 + L))
        out.append((f"len{L}", seq, qual))
    for L in (40, 64, 200):
        out.append((f"homo{L}", b"A" * L, b"I" * L))
        out.append((f"homoT{L}", b"t" * L, b"I" * L))
        out.append((f"di{L}", b"AC" * (L // 2), b"I" * (L // 2 * 2)))
    return out


# ---- the histogram and the estimate against the oracle ------------------------------------------------------------------------------
@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("k", [11, 13, 21, 31])
@pytest.mark.parametrize("form", ["plain", "crlf", "gz2"])
def test_oracle_parity(lib, k, form, tmp_path):
    reads = oddities(k)
    path = str(tmp_path / "r.fq")
    if form == "gz2":                                 # two gzip members
        half = len(reads) // 2
        synth.write_reads(reads[:half], str(tmp_path / "a.fq"))
        synth.write_reads(reads[half:], str(tmp_path / "b.fq"))
        path = str(tmp_path / "r.fq.gz")
        with open(path, "wb") as f:
            f.write(gzip.compress(open(tmp_path / "a.fq", "rb").read()) + gzip.compress(open(tmp_path / "b.fq", "rb").read()))
    else:
        synth.write_reads(reads, path, crlf=form == "crlf")
    info = check(lib, path, k)
    assert info["k"] == k and info["reads"] == len(reads)
    assert info["bases"] == sum(len(r[1]) for r in reads)


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_one_read_and_window_boundaries(lib, tmp_path, monkeypatch):
    path = str(tmp_path / "one.fq")
    synth.write_reads([next(synth.make_reads(GENOME, n_reads=1, length=5000, seed=3))], path)
    with pytest.raises(api.AutocyclerGpuError) as e:         # one error-free read: every k-mer once, no depth peak
        api.genome_size_estimate(path, 21, lib=lib)
    assert e.value.code == -6 and e.value.message.startswith("no k-mer depth peak")
    with pytest.raises(O.NoPeak):
        O.estimate(*O.histogram(path, 21))
    # the same histogram whatever the windows: boundaries inside records, a record longer than the window
    path = str(tmp_path / "r.fq")
    synth.write_reads(oddities(5), path)
    want = api.genome_size_estimate(path, 15, lib=lib)
    for w in (1000, 7777, 100_000):
        monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(w))
        got = api.genome_size_estimate(path, 15, lib=lib)
        assert got["histogram"] == want["histogram"] and got["estimate"] == want["estimate"], w
    assert want["histogram"] == O.histogram(path, 15)[0]


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_partitions_and_reruns(lib, tmp_path, monkeypatch):
    path = str(tmp_path / "r.fq")
    synth.write_reads(deep_reads(seed=9), path)
    base = check(lib, path, 17)
    assert base["partitions"] == 1 and base["reruns"] == 0
    for parts in (1, 2, 3, 8):
        monkeypatch.setenv("AC_GS_PARTITIONS", str(parts))
        got = api.genome_size_estimate(path, 17, lib=lib)
        assert got["partitions"] == parts and got["histogram"] == base["histogram"] and got["estimate"] == base["estimate"]
    monkeypatch.delenv("AC_GS_PARTITIONS")
    # a budget of ceil(W / 2) slots: P = 4, each table ceil(2 W / 4) slots
    monkeypatch.setenv("AC_GS_TABLE_SLOTS", str((base["windows"] + 1) // 2))
    got = api.genome_size_estimate(path, 17, lib=lib)
    assert got["partitions"] == 4 and got["reruns"] == 0 and got["histogram"] == base["histogram"]
    # one partition in a table far smaller than the distinct k-mers: reruns with twice the slots until it fits
    monkeypatch.setenv("AC_GS_PARTITIONS", "1")
    monkeypatch.setenv("AC_GS_TABLE_SLOTS", str(base["distinct"] // 5))
    got = api.genome_size_estimate(path, 17, lib=lib)
    assert got["partitions"] == 1 and got["reruns"] >= 2 and got["histogram"] == base["histogram"]
    assert got["table_bytes"] >= base["distinct"] * 16


# ---- the rule on crafted histograms -------------------------------------------------------------------------------------------------
def rule(emu, hist, W):
    got = api.genome_size_from_histogram(hist, W, lib=emu)
    want = O.estimate(hist, W)
    for f in want:
        assert got[f] == want[f], f
    return got


def bimodal(peak=30, genome=100_000, errors=400_000):
    h = [0] * 200
    h[1], h[2], h[3] = errors, errors // 10, errors // 100
    for c in range(5, 120):
        h[c] = int(genome * np.exp(-0.5 * ((c - peak) / (peak ** 0.5)) ** 2) / (2.5 * peak ** 0.5))
    return h


def test_rule_crafted(emu):
    h = bimodal()
    W = sum(c * x for c, x in enumerate(h))
    r = rule(emu, h, W)
    assert r["valley"] < 10 and r["peak"] == 30 and abs(r["estimate"] - 100_000) < 2_000
    # a tie at the peak: the smaller count wins, and the parabola moves toward the larger neighbour
    h = [0, 100, 10, 1, 5, 50, 50, 20, 3]
    r = rule(emu, h, 2000)
    assert (r["valley"], r["peak"]) == (3, 5) and r["peak_refined"] == 5 + (5 - 50) / (2 * (5 - 100 + 50))
    # a zero denominator: p* = p
    h = [0, 100, 10, 1, 10, 20, 30, 20, 0]
    r = rule(emu, h, 1000)
    assert r["peak"] == 6 and r["peak_refined"] == 6.0 and r["estimate"] == round((1000 - 100 - 20) / 6)
    # a valley at 1 (error-free reads): nothing is subtracted
    h = [0, 0, 0, 5, 40, 80, 40, 5]
    r = rule(emu, h, 1000)
    assert r["valley"] == 1 and r["solid"] == 1000 and r["peak"] == 5 and r["estimate"] == 200
    # the half-way rounding goes away from zero
    h = [0, 0, 0, 10, 20, 10]
    r = rule(emu, h, 9)
    assert r["peak_refined"] == 4.0 and r["estimate"] == 2      # 9 / 4 = 2.25
    r = rule(emu, h, 10)
    assert r["estimate"] == 3                                   # 10 / 4 = 2.5


def test_rule_refusals(emu):
    # a monotone spectrum has no valley
    for h in ([0, 1000, 500, 250, 125, 60, 30, 15, 7, 3, 1], [0], [0, 5]):
        with pytest.raises(O.NoPeak):
            O.estimate(h, 10_000)
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.genome_size_from_histogram(h, 10_000, lib=emu)
        assert e.value.code == -6 and e.value.message == "no k-mer depth peak: the reads are too shallow or too noisy for a k-mer estimate"
    # a peak at the cap (H - 2) or in the overflow bin's neighbour
    h = [0] * H
    h[1], h[2], h[3], h[H - 2] = 100, 10, 1, 500
    with pytest.raises(O.PeakAtCap):
        O.estimate(h, 10 ** 9)
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.genome_size_from_histogram(h, 10 ** 9, lib=emu)
    assert e.value.code == -4
    h[H - 2], h[H - 3] = 0, 500                               # one below the cap is still a peak
    r = rule(emu, h, 10 ** 9)
    assert r["peak"] == H - 3
    # more occurrences below the valley than windows
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.genome_size_from_histogram(bimodal(), 10, lib=emu)
    assert e.value.code == -6


# ---- accuracy on synthetic genomes of known size -------------------------------------------------------------------------------------
# The target, set before any run, is an estimate within 2% of the true length.  The rule misses it in four of these five cases; what it
# gives instead is recorded here (estimate, and its deviation) and in DESIGN.md §18, not hidden behind a wider tolerance.  The runs are
# seeded, so each estimate is exact; a change to the rule or the reads shows up here.
TARGET = 0.02
MISSED = {(17, 0.01): 1_020_108, (21, 0.01): 1_042_794, (17, 0.05): 1_042_769, (21, 0.05): 1_035_288, "two_replicons": 738_317}


def accuracy_case(key, length, info):
    rel = info["estimate"] / length - 1
    if key in MISSED:
        assert info["estimate"] == MISSED[key] and abs(rel) >= TARGET, (key, info["estimate"], rel)
    else:
        assert abs(rel) < TARGET, (key, info["estimate"], rel)


@pytest.mark.parametrize("k", [17, 21])
@pytest.mark.parametrize("err", [0.01, 0.05])
def test_accuracy(emu, k, err, tmp_path):
    """1 Mbp genomes with make_genome's repeat families (7 x 5 kbp and 10 x 1.3 kbp) at 40x."""
    genome = synth.make_genome(synth.SplitMix64(0xACC0 + k), 1_000_000)
    path = str(tmp_path / "r.fq")
    synth.write_reads(synth.make_noisy_reads(genome, depth=40, n50=8000, seed=k, sub=err / 2, ins=err / 4, dele=err / 4), path)
    accuracy_case((k, err), len(genome), api.genome_size_estimate(path, k, lib=emu))


def test_accuracy_two_replicons(emu, tmp_path):
    """A 600 kbp chromosome and a 40 kbp plasmid present in 3 copies per genome: the estimate counts the plasmid three times."""
    rng = synth.SplitMix64(0x2E91)
    chrom, plasmid = synth.make_genome(rng, 600_000), synth.make_genome(rng, 40_000)
    reads = list(synth.make_noisy_reads(chrom, depth=40, n50=8000, seed=1, sub=0.005, ins=0.0025, dele=0.0025))
    reads += list(synth.make_noisy_reads(plasmid, depth=120, n50=8000, seed=2, sub=0.005, ins=0.0025, dele=0.0025))
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads, path)
    accuracy_case("two_replicons", 600_000 + 3 * 40_000, api.genome_size_estimate(path, 21, lib=emu))


# ---- errors ----------------------------------------------------------------------------------------------------------------------
MALFORMED = [
    (b"@a\nAC\n+\nII\nb\nAC\n+\nII\n", 2, "expected '@' at the start of the header line"),
    (b"@a\nAC\n+\nII\n@b\nAC\n-\nII\n", 2, "expected '+' at the start of the separator line"),
    (b"@a\nAC\n+\nII\n@b\nACG\n+\nII\n@c\nA\n+\nI\n", 2, "sequence and quality lengths differ"),
    (b"@a\nAC\n+\nII\n@b\nAC", 2, "truncated record"),
]


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_errors(lib, tmp_path):
    for data, rec, why in MALFORMED:
        path = str(tmp_path / "bad.fq")
        open(path, "wb").write(data)
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.genome_size_estimate(path, 21, lib=lib)
        assert e.value.code == -6 and e.value.message == f"Error reading FASTQ file: record {rec}: {why}"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.genome_size_estimate(str(tmp_path / "nope.fq"), 21, lib=lib)
    assert e.value.code == -6 and e.value.message == f"file does not exist: {tmp_path / 'nope.fq'}"
    path = str(tmp_path / "short.fq")
    synth.write_reads([("a", b"ACGTN" * 8, b"I" * 40), ("b", b"", b""), ("c", b"ACGT" * 5, b"I" * 20)], path)
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.genome_size_estimate(path, 21, lib=lib)
    assert e.value.code == -6 and e.value.message == "no k-mer windows: no read holds 21 consecutive A, C, G or T bases"
    open(tmp_path / "empty.fq", "wb").close()
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.genome_size_estimate(str(tmp_path / "empty.fq"), 21, lib=lib)
    assert e.value.code == -6 and e.value.message.startswith("no k-mer windows")
    for k in (9, 10, 12, 22, 33, 0):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.genome_size_estimate(path, k, lib=lib)
        assert e.value.code == -6 and e.value.message == "--kmer must be odd and between 11 and 31"
    open(tmp_path / "afile", "w").close()
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.genome_size_estimate(path, 21, dir=str(tmp_path / "afile"), lib=lib)
    assert e.value.code == -6 and e.value.message.endswith("exists but is not a directory")


# ---- the CLI ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def emu_cli(emu, tmp_path_factory):
    """The CLI built against the emulation library, so that its successful runs can be checked without a GPU."""
    out = str(tmp_path_factory.mktemp("cli") / "autocycler")
    emu_dir = os.path.join(ROOT, "tests", "emu")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", out, os.path.join(CSRC, "cli_main.cpp"), f"-L{emu_dir}", "-l:libautocycler_emu.so",
                    f"-Wl,-rpath,{emu_dir}"], check=True)
    return out


@pytest.fixture(scope="session")
def cli():
    subprocess.run(["make", "-s", "-C", CSRC], check=True)
    return AUTOCYCLER


def run(binary, *args):
    return subprocess.run([binary, *map(str, args)], capture_output=True, text=True)


def test_cli_end_to_end(emu_cli, tmp_path):
    path = str(tmp_path / "reads.fastq.gz")
    reads = list(deep_reads(depth=40, seed=4))
    synth.write_reads(reads, path, gz=True)
    r = run(emu_cli, "helper", "genome_size", "-r", path, "-t", "8", "-d", tmp_path / "hist")
    assert r.returncode == 0, r.stderr
    hist, W = O.histogram(path, 21)
    want = O.estimate(hist, W)["estimate"]
    assert r.stdout == f"{want}\n"
    assert "Starting autocycler helper genome_size" in r.stderr and "Raven" in r.stderr
    tsv = open(tmp_path / "hist" / "kmer_histogram.tsv").read()
    assert tsv == "".join(f"{c}\t{x}\n" for c, x in enumerate(hist) if c and x)
    r = run(emu_cli, "helper", "genome_size", "--reads", path, "--kmer", "17")
    assert r.returncode == 0 and r.stdout == f"{O.estimate(*O.histogram(path, 17))['estimate']}\n"
    # the pipelines' two lines: subsample takes the number as its genome size
    size = run(emu_cli, "helper", "genome_size", "--reads", path, "--threads", "4").stdout.strip()
    r = run(emu_cli, "subsample", "--reads", path, "--out_dir", tmp_path / "sub", "--genome_size", size, "--min_read_depth", "5")
    assert r.returncode == 0, r.stderr
    files = subsample_oracle.subsample(path, size, 4, 5.0, 0)
    for f, data in files.items():
        assert open(tmp_path / "sub" / f, "rb").read() == data, f


def test_cli_surface(cli, tmp_path):
    usage = "Usage: autocycler helper genome_size"
    for args in (["helper"], ["helper", "genome_size"], ["helper", "genome_size", "-t", "4"], ["helper", "-r", "x"]):
        r = run(cli, *args)
        assert r.returncode == 2 and r.stderr.startswith(usage) and r.stdout == "", args
    r = run(cli, "helper", "-h")
    assert r.returncode == 0 and r.stderr.startswith(usage) and "departs from the reference" in r.stderr
    r = run(cli, "helper", "genome_size", "--help")
    assert r.returncode == 0 and r.stderr.startswith(usage)
    for task in ("raven", "flye", "canu", "bogus"):
        r = run(cli, "helper", task, "-r", "x", "-o", "y")
        assert r.returncode == 1 and f"helper task '{task}' runs an external assembler" in r.stderr and r.stdout == "", task
    for flag, value in (("--args", "-x"), ("-o", "prefix"), ("-g", "5m"), ("--read_type", "ont_r10"), ("--min_depth_abs", "3"),
                        ("--min_depth_rel", "0.1"), ("--bogus", "1")):
        r = run(cli, "helper", "genome_size", "-r", "x", flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: unexpected argument '{flag}'\n{usage}"), flag
    for flag, value in (("--kmer", "x"), ("-t", "-1"), ("--kmer", "2.5")):
        r = run(cli, "helper", "genome_size", "-r", "x", flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'"), (flag, value)
    r = run(cli, "helper", "genome_size", "-r", tmp_path / "nope.fq")
    assert r.returncode == 1 and r.stdout == "" and r.stderr.endswith(f"Error: file does not exist: {tmp_path / 'nope.fq'}\n")


# ---- the shapes only the GPU reaches ------------------------------------------------------------------------------------------------
def bench_input(tmp_path, gz=False):
    import bench_genome_size as B
    return B.write_input("b" if gz else "a", str(tmp_path))


@pytest.mark.gpu
def test_gpu_full_size_against_golden(gpu, tmp_path, monkeypatch):
    """5 Mbp at 100x with 1% errors (bench_genome_size.py's workload a): the histogram's SHA-256 and the estimate against the golden the
    oracle wrote, twice (determinism), then in several windows, and with four partitions and with reruns."""
    path = bench_input(tmp_path)
    g = GOLDENS["a"]

    def same(info):
        assert hashlib.sha256(np.asarray(info["histogram"], dtype="<u8").tobytes()).hexdigest() == g["histogram_sha256"]
        assert info["estimate"] == g["estimate"] and info["windows"] == g["windows"]

    first = api.genome_size_estimate(path, 21, lib=gpu)
    same(first)
    second = api.genome_size_estimate(path, 21, lib=gpu)
    assert second["histogram"] == first["histogram"] and second["estimate"] == first["estimate"]
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(64 << 20))
    same(api.genome_size_estimate(path, 21, lib=gpu))
    monkeypatch.delenv("AC_SUBSAMPLE_WINDOW")
    monkeypatch.setenv("AC_GS_TABLE_SLOTS", str((first["windows"] + 1) // 2))
    p4 = api.genome_size_estimate(path, 21, lib=gpu)
    assert p4["partitions"] == 4
    same(p4)
    monkeypatch.setenv("AC_GS_PARTITIONS", "3")
    monkeypatch.setenv("AC_GS_TABLE_SLOTS", str(first["distinct"] // 12))
    rr = api.genome_size_estimate(path, 21, lib=gpu)
    assert rr["partitions"] == 3 and rr["reruns"] >= 3
    same(rr)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [11, 21, 31])
def test_gpu_parity_oddities(gpu, k, tmp_path):
    path = str(tmp_path / "r.fq")
    synth.write_reads(oddities(k), path, crlf=True)
    check(gpu, path, k)


@pytest.mark.gpu
def test_gpu_read_longer_than_window(gpu, tmp_path, monkeypatch):
    big = synth.make_genome(synth.SplitMix64(77), 400_000)
    reads = [("long", big.tobytes()[:300_000], b"I" * 300_000)] + list(synth.make_noisy_reads(big, depth=30, n50=5000, seed=6, sub=0.005))
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads, path)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(100_000))
    info = check(gpu, path, 21)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(1 << 20))
    assert api.genome_size_estimate(path, 21, lib=gpu)["histogram"] == info["histogram"]
