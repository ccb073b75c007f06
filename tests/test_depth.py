"""`autocycler depth`: each contig's read depth from the reads' k-mers, counted on the GPU, and the reference's helper depth filter
(DESIGN.md §19).  Read-measured depth is not in the reference, so it is pinned against the numpy oracle of the rule
(tests/depth_oracle.py) and, on synthetic replicons of known copy number, by what it means.  The filter and the header parser are the
reference's: they are replayed against the data of its unit tests (tests/golden/helper_depth_kats.json).  The CPU tests run the product's
code through the host-emulation library (the kernels' bodies, serially); the tests marked gpu run the CUDA build on the H100."""
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import depth_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "helper_depth_kats.json")))


def goldens():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "depth_goldens.json")))


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", CSRC, "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def noisy(genome, depth, seed, err=0.01, n50=3000):
    return list(synth.make_noisy_reads(genome, depth=depth, n50=n50, seed=seed, sub=err / 2, ins=err / 4, dele=err / 4))


def write_fasta(path, records):
    with open(path, "w") as f:
        for header, seq in records:
            f.write(f">{header}\n{seq}\n")


def check(lib, asm, reads, k, tmp_path, min_abs=None, min_rel=None):
    """The product's output FASTA, TSV, depths and unique counts against the oracle's; returns the info."""
    out, tsv = str(tmp_path / "out.fasta"), str(tmp_path / "out.tsv")
    if os.path.exists(out):
        os.remove(out)
    info = api.depth(asm, out, reads=reads, k=k, min_depth_abs=min_abs, min_depth_rel=min_rel, tsv=tsv, lib=lib)
    want = O.run(asm, reads, k, min_abs, min_rel)
    assert info["depths"] == want["depths"]
    assert info["unique"] == want["unique"]
    assert info["unique_kmers"] == sum(want["unique"])
    assert open(tsv).read() == want["tsv"]
    assert info["filtered"] == int(want["filtered"])
    if want["fasta"] is None:
        assert not os.path.exists(out)
    else:
        assert open(out, "rb").read() == want["fasta"]
    return info


def parity_case(tmp_path):
    """Contigs that share a repeat, one whose keys are all shared, a palindromic and homopolymer-rich one, circular and linear ones
    (one shorter than k), N/IUPAC and lowercase in contigs and reads; reads in two gzip members."""
    rng = synth.SplitMix64(0xD3)
    a, b, rep = synth.make_genome(rng, 6000), synth.make_genome(rng, 4000), synth.make_genome(rng, 800)
    a, b, rep = a.tobytes().decode(), b.tobytes().decode(), rep.tobytes().decode()
    pal = "ACGTTGCA" * 20 + "A" * 60 + "GAATTC" * 15 + "T" * 40 + "CCGG" * 25
    contigs = [
        ("ctgA circular=true", a[:3000] + rep + a[3000:]),
        ("ctgB length=4800", b[:2000] + rep + b[2000:]),
        ("shared", rep[100:700]),                                   # every key also in ctgA and ctgB: no depth
        ("pal Circular=TRUE", pal),
        ("tiny circular=true", a[100:112]),                         # shorter than k: no junction windows
        ("mixed", a[200:900].lower() + "NNRYK" + a[900:1500] + "N" + b[100:700].lower()),
    ]
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, contigs)
    genome = np.frombuffer((a + b + pal + rep).encode(), dtype=np.uint8)
    reads = noisy(genome, 12, 5, n50=1500)
    odd = []
    for i, (n, s, q) in enumerate(reads):
        s = bytearray(s)
        if i % 4 == 1 and len(s) > 50:
            s[20:23] = b"NRY"
        if i % 5 == 2:
            s = bytearray(bytes(s).lower())
        odd.append((n, bytes(s), q))
    half = len(odd) // 2
    synth.write_reads(odd[:half], str(tmp_path / "r1.fq"))
    synth.write_reads(odd[half:], str(tmp_path / "r2.fq"))
    path = str(tmp_path / "reads.fq.gz")
    with open(path, "wb") as f:
        f.write(gzip.compress(open(tmp_path / "r1.fq", "rb").read()) + gzip.compress(open(tmp_path / "r2.fq", "rb").read()))
    return asm, path


# ---- the rule against the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_oracle_parity(emu, k, tmp_path):
    asm, reads = parity_case(tmp_path)
    info = check(emu, asm, reads, k, tmp_path)
    assert info["depths"][2] is None and info["unique"][2] == 0          # the shared contig
    assert info["k"] == k and info["contigs"] == 6
    # a contig without a depth: the filter is skipped and every record is kept
    info = check(emu, asm, reads, k, tmp_path, min_rel=0.5)
    assert info["filtered"] == 0 and info["kept"] == 6


def test_filter_and_medians(emu, tmp_path):
    """Even and odd medians, the filter on read depths, and windows split inside records."""
    rng = synth.SplitMix64(0xD4)
    chrom, plas = synth.make_genome(rng, 5000), synth.make_genome(rng, 1200)
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("chrom circular=true", chrom.tobytes().decode()), ("plas", plas.tobytes().decode())])
    reads = str(tmp_path / "r.fq")
    synth.write_reads(noisy(chrom, 20, 7) + noisy(plas, 5, 8), reads)
    for abs_, rel in ((None, 0.5), (3.0, None), (1e9, None), (None, None)):
        check(emu, asm, reads, 21, tmp_path, abs_, rel)
    base = api.depth(asm, str(tmp_path / "o.fasta"), reads=reads, k=15, lib=emu)
    for w in (1000, 7777):
        os.environ["AC_SUBSAMPLE_WINDOW"] = str(w)
        try:
            got = api.depth(asm, str(tmp_path / "o.fasta"), reads=reads, k=15, lib=emu)
        finally:
            del os.environ["AC_SUBSAMPLE_WINDOW"]
        assert got["depths"] == base["depths"] and got["unique"] == base["unique"]


def test_even_and_odd_median(emu, tmp_path):
    """Crafted reads: a contig of 4 unique keys seen 1, 2, 5 and 9 times (median 3.5) and one of 3 keys seen 0, 4, 4 times (median 4)."""
    rng = synth.SplitMix64(0xD5)
    g = synth.make_genome(rng, 200).tobytes().decode()
    c1, c2 = g[:14], g[100:113]                                      # k = 11: 4 and 3 windows
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("c1", c1), ("c2", c2)])
    reads = []
    for i, times in enumerate((1, 2, 5, 9)):
        reads += [(f"a{i}_{j}", c1[i:i + 11].encode(), b"I" * 11) for j in range(times)]
    for i, times in enumerate((0, 4, 4)):
        reads += [(f"b{i}_{j}", c2[i:i + 11].encode(), b"I" * 11) for j in range(times)]
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads, path)
    info = check(emu, asm, path, 11, tmp_path)
    assert info["depths"] == [3.5, 4.0]
    assert open(tmp_path / "out.fasta").read().startswith(">c1 depth=3.50\n")


def test_meaning_copy_number(emu, tmp_path):
    """A 600 kbp chromosome and a 40 kbp plasmid in 3 copies per genome, reads at 40x with 1% errors, the assembly holding one copy of
    each: the plasmid's depth over the chromosome's lands within 3.0 +- 0.15.  The run is seeded, so the depths are pinned exactly."""
    import bench_depth as B
    asm, reads = B.write_input("c", str(tmp_path))
    info = api.depth(asm, str(tmp_path / "out.fasta"), reads=reads, k=21, lib=emu)
    chrom, plasmid = info["depths"]
    assert abs(plasmid / chrom - 3.0) <= 0.15
    assert info["depths"] == goldens()["c"]["depths"] and info["unique"] == goldens()["c"]["unique"]


# ---- the reference's filter and header parser ---------------------------------------------------------------------------------------
def test_kat_depth_from_header(emu):
    for header, want in KATS["depth_from_header"]:
        assert api.depth_from_header(header, lib=emu) == want, header
        assert O.depth_from_header(header) == want, header
    for header, want in (("x depth=", None), ("x depth=-5", None), ("x depth=1e-5", None), ("x depth=1e5_y", 1e5), ("x depth=INF", float("inf")),
                         ("x coverage=.5", 0.5), ("x depth=5. y", 5.0), ("x depth=0x10", None), ("x depth=abc depth-3", None)):
        assert api.depth_from_header(header, lib=emu) == want, header


def test_kat_depth_filter_text(emu):
    text = KATS["depth_filter"]["fasta"]
    for step in KATS["depth_filter"]["steps"]:
        text = api.depth_filter_text(text, step["min_abs"], step["min_rel"], lib=emu)
        if step["records"] is None:
            assert text == ""
        else:
            assert text.count(">") == step["records"], step


def test_kat_depth_filter_cli(emu_cli, tmp_path):
    """The reference's test_depth_filter through the CLI: the file filtered in place, its state checked after every step."""
    fasta = str(tmp_path / "test.fasta")
    open(fasta, "w").write(KATS["depth_filter"]["fasta"])
    for step in KATS["depth_filter"]["steps"]:
        args = ["depth", "-i", fasta, "-o", fasta, "--source", "header"]
        if step["min_abs"] is not None:
            args += ["--min_depth_abs", step["min_abs"]]
        if step["min_rel"] is not None:
            args += ["--min_depth_rel", step["min_rel"]]
        r = run(emu_cli, *args)
        assert r.returncode == 0 and r.stdout == "", r.stderr
        if step["records"] is None:
            assert not os.path.exists(fasta)
        else:
            assert open(fasta).read().count(">") == step["records"], step
            if step["min_abs"] is not None or step["min_rel"] is not None:
                assert "Autocycler helper depth filter\nthreshold = " in r.stderr


# ---- errors -------------------------------------------------------------------------------------------------------------------------
def test_errors(emu, tmp_path):
    asm, reads = str(tmp_path / "a.fasta"), str(tmp_path / "r.fq")
    write_fasta(asm, [("a", "ACGT" * 20)])
    synth.write_reads([("r", b"ACGT" * 20, b"I" * 80)], reads)
    out = str(tmp_path / "o.fasta")

    def err(code, message, **kw):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.depth(kw.pop("assembly", asm), out, lib=emu, **kw)
        assert e.value.code == code and (e.value.message == message if isinstance(message, str) else message(e.value.message)), e.value.message

    err(-6, f"file does not exist: {tmp_path / 'nope.fasta'}", assembly=str(tmp_path / "nope.fasta"), reads=reads)
    err(-6, f"file does not exist: {tmp_path / 'nope.fq'}", reads=str(tmp_path / "nope.fq"))
    err(-6, "--reads is required with --source reads (or use --source header)")
    for k in (9, 10, 12, 22, 33, 0):
        err(-6, "--kmer must be odd and between 11 and 31", reads=reads, k=k)
    write_fasta(str(tmp_path / "d.fasta"), [("a", "ACGT" * 20), ("b depth=5.0", "ACGA" * 20)])
    err(-6, lambda m: m.endswith("the header of b already carries a depth; use --source header to filter by it"),
        assembly=str(tmp_path / "d.fasta"), reads=reads)
    open(tmp_path / "empty.fasta", "w").close()
    err(-6, f"{tmp_path / 'empty.fasta'} is an empty file", assembly=str(tmp_path / "empty.fasta"), reads=reads)
    for data, rec, why in ((b"@a\nAC\n+\nII\nb\nAC\n+\nII\n", 2, "expected '@' at the start of the header line"),
                           (b"@a\nAC\n+\nII\n@b\nAC", 2, "truncated record")):
        open(tmp_path / "bad.fq", "wb").write(data)
        err(-6, f"Error reading FASTQ file: record {rec}: {why}", reads=str(tmp_path / "bad.fq"))
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.depth(asm, str(tmp_path / "no_dir" / "o.fasta"), reads=reads, lib=emu)
    assert e.value.code == -5 and e.value.message == f"cannot write {tmp_path / 'no_dir' / 'o.fasta'}"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.depth(asm, out, reads=reads, tsv=str(tmp_path / "no_dir" / "t.tsv"), lib=emu)
    assert e.value.code == -5
    os.environ["AC_DEPTH_TABLE_SLOTS"] = "100"                     # 2 x 61 windows do not fit 100 slots
    try:
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.depth(asm, out, reads=reads, lib=emu)
        assert e.value.code == -4 and "does not fit" in e.value.message
    finally:
        del os.environ["AC_DEPTH_TABLE_SLOTS"]


# ---- the CLI ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def emu_cli(emu, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cli") / "autocycler")
    emu_dir = os.path.join(ROOT, "tests", "emu")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", out, os.path.join(CSRC, "cli_main.cpp"), f"-L{emu_dir}", "-l:libautocycler_emu.so",
                    f"-Wl,-rpath,{emu_dir}"], check=True)
    return out


def run(binary, *args):
    return subprocess.run([binary, *map(str, args)], capture_output=True, text=True)


def test_cli(emu_cli, tmp_path):
    asm, reads = parity_case(tmp_path)
    out, tsv = tmp_path / "cli.fasta", tmp_path / "cli.tsv"
    r = run(emu_cli, "depth", "-i", asm, "-r", reads, "-o", out, "--tsv", tsv, "--kmer", "15")
    assert r.returncode == 0 and r.stdout == "", r.stderr
    want = O.run(asm, reads, 15)
    assert open(out, "rb").read() == want["fasta"] and open(tsv).read() == want["tsv"]
    assert "Starting autocycler depth" in r.stderr and "Note: not every contig has a depth" not in r.stderr
    r = run(emu_cli, "depth", "-i", asm, "-r", reads, "-o", out, "--kmer", "15", "--min_depth_abs", "2")
    assert r.returncode == 0 and "Note: not every contig has a depth" in r.stderr
    usage = "Usage: autocycler depth"
    for args in (["depth"], ["depth", "-i", asm], ["depth", "-i", asm, "-o", out], ["depth", "-o", out, "-r", reads]):
        r = run(emu_cli, *args)
        assert r.returncode == 2 and r.stderr.startswith(usage) and r.stdout == "", args
    r = run(emu_cli, "depth", "-h")
    assert r.returncode == 0 and r.stderr.startswith(usage) and "not in the reference" in r.stderr
    for flag, value in (("--kmer", "x"), ("--min_depth_abs", "y"), ("--min_depth_rel", "1.5x"), ("--source", "both")):
        r = run(emu_cli, "depth", "-i", asm, "-o", out, "-r", reads, flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'"), (flag, value)
    r = run(emu_cli, "depth", "-i", asm, "-o", out, "-r", reads, "--bogus", "1")
    assert r.returncode == 2 and r.stderr.startswith("error: unexpected argument '--bogus'")
    r = run(emu_cli, "depth", "-i", tmp_path / "nope.fasta", "-o", out, "-r", reads)
    assert r.returncode == 1 and r.stderr.endswith(f"Error: file does not exist: {tmp_path / 'nope.fasta'}\n")
    r = run(emu_cli, "depth", "-i", asm, "-o", out, "-r", reads, "--kmer", "20")
    assert r.returncode == 1 and r.stderr.endswith("Error: --kmer must be odd and between 11 and 31\n")


# ---- the GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_bench_input_against_golden(gpu, tmp_path, monkeypatch):
    """bench_depth.py's workload a (5 Mbp at 100x, the genome as the assembly) against the oracle's golden, three times
    (determinism), then in several read windows."""
    import bench_depth as B
    asm, reads = B.write_input("a", str(tmp_path))
    g = goldens()["a"]
    out = str(tmp_path / "out.fasta")
    for _ in range(3):
        info = api.depth(asm, out, reads=reads, k=21, lib=gpu)
        assert hashlib.sha256(open(out, "rb").read()).hexdigest() == g["fasta_sha256"]
        assert info["depths"] == g["depths"] and info["unique"] == g["unique"]
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(64 << 20))
    info = api.depth(asm, out, reads=reads, k=21, lib=gpu)
    assert info["depths"] == g["depths"] and hashlib.sha256(open(out, "rb").read()).hexdigest() == g["fasta_sha256"]


@pytest.mark.gpu
@pytest.mark.parametrize("k", [11, 21, 31])
def test_gpu_oracle_parity(gpu, k, tmp_path):
    asm, reads = parity_case(tmp_path)
    check(gpu, asm, reads, k, tmp_path)
    check(gpu, asm, reads, k, tmp_path, min_abs=1.0)


@pytest.mark.gpu
def test_gpu_read_longer_than_window(gpu, tmp_path, monkeypatch):
    big = synth.make_genome(synth.SplitMix64(78), 300_000)
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("big circular=true", big.tobytes().decode())])
    reads = [("long", big.tobytes()[:250_000], b"I" * 250_000)] + noisy(big, 20, 9, n50=5000)
    path = str(tmp_path / "r.fq")
    synth.write_reads(reads, path)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(100_000))
    info = check(gpu, asm, path, 21, tmp_path)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(1 << 20))
    assert api.depth(asm, str(tmp_path / "o2.fasta"), reads=path, k=21, lib=gpu)["depths"] == info["depths"]


@pytest.mark.gpu
def test_gpu_large_assembly(gpu, tmp_path):
    """A 10 Mbp assembly in five contigs, reads at 8x over half of it: the depths against the oracle."""
    rng = synth.SplitMix64(0xD6)
    contigs = [synth.make_genome(rng, 2_000_000) for _ in range(5)]
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [(f"c{i} circular=true", c.tobytes().decode()) for i, c in enumerate(contigs)])
    path = str(tmp_path / "r.fq")
    synth.write_reads(noisy(contigs[0], 8, 11, n50=8000) + noisy(contigs[3], 4, 12, n50=8000), path)
    info = check(gpu, asm, path, 21, tmp_path)
    assert info["assembly_windows"] == 10_000_000 and info["depths"][1] == 0.0
