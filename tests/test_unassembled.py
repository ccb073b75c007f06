"""`autocycler unassembled`: the reads an assembly does not explain, and the depth of the sequence it misses, counted on the GPU (DESIGN.md
§21).  `unassembled` is not in the reference, so it is pinned against the numpy oracle of the rule (tests/unassembled_oracle.py) and, on
synthetic genomes with sequence missing from the assembly at known places, by what the rule means.  The CPU tests run the product's code
through the host-emulation library (the kernels' bodies, serially); the tests marked gpu run the CUDA build on the H100."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import unassembled_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
H = api.GENOME_SIZE_BINS
FILES = ["absent_histogram.tsv", "fraction_histogram.tsv", "kmer_histogram.tsv", "summary.tsv", "unassembled.fastq", "unassembled.tsv"]


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", CSRC, "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def write_fasta(path, records):
    with open(path, "w") as f:
        for header, seq in records:
            f.write(f">{header}\n{seq}\n")


def noisy(genome, depth, seed, err=0.01, n50=3000):
    g = np.frombuffer(genome.encode(), dtype=np.uint8) if isinstance(genome, str) else genome
    return list(synth.make_noisy_reads(g, depth=depth, n50=n50, seed=seed, sub=err / 2, ins=err / 4, dele=err / 4))


def out_files(out_dir):
    files = {}
    for dirpath, _, names in os.walk(out_dir):
        for n in names:
            p = os.path.join(dirpath, n)
            files[os.path.relpath(p, out_dir)] = open(p, "rb").read()
    return files


def check(lib, reads, assemblies, k, out_dir, **kw):
    """Every file the product writes against the oracle's (and no other file); returns (info, oracle result)."""
    info = api.unassembled(reads, assemblies, str(out_dir), k=k, lib=lib, **kw)
    want = O.run(reads, assemblies, k, **kw)
    got = out_files(out_dir)
    assert sorted(got) == sorted(want["files"]) == FILES
    for name, data in want["files"].items():
        assert got[name] == data, name
    assert info["min_count"] == want["t"] and info["read_windows"] == want["W"] and info["valley"] == (want["valley"] or 0)
    assert info["selected_reads"] == len(want["selected"]) and info["absent_kmers"] == want["absent_kmers"]
    return info, want


def parity_case(tmp_path):
    """A circular chromosome and a linear replicon, held by a directory input (the chromosome without a 20 kbp stretch) and a file input
    (the replicon); a circular plasmid missing from both, at 4 copies, its reads drawn from the plasmid repeated end to end so that some
    cross its junction; N/IUPAC and lowercase in reads and contigs; reads in two gzip members."""
    rng = synth.SplitMix64(0xB1)
    chrom, lin, plas = (synth.make_genome(rng, n).tobytes().decode() for n in (60_000, 8_000, 4_000))
    held = chrom[:15_000] + chrom[35_000:]
    d = tmp_path / "asm"
    d.mkdir()
    write_fasta(d / "chrom.fasta", [("chrom circular=true", held[:9_000].lower() + "NNRYK" + held[9_005:])])
    write_fasta(d / "notes.txt", [("x", "ACGT")])                        # not an assembly file: the directory skips it
    other = str(tmp_path / "replicon.fa")
    write_fasta(other, [("lin", lin[:3_000] + "nnnn" + lin[3_004:]), ("tiny circular=true", chrom[100:115])])
    reads = noisy(chrom, 25, 11, n50=2500) + noisy(lin, 25, 12, n50=2500) + noisy(plas * 3, 4 * 25 / 3, 13, n50=2500)
    odd = []
    for i, (n, s, q) in enumerate(reads):
        s = bytearray(s)
        if i % 4 == 1 and len(s) > 50:
            s[20:23] = b"NRY"
        if i % 5 == 2:
            s = bytearray(bytes(s).lower())
        odd.append((n, bytes(s), q))
    order = np.argsort(np.array(synth.SplitMix64(0xB2).u64(len(odd)), dtype=np.uint64), kind="stable")
    odd = [odd[i] for i in order]                                         # the sources interleaved
    half = len(odd) // 2
    synth.write_reads(odd[:half], str(tmp_path / "r1.fq"))
    synth.write_reads(odd[half:], str(tmp_path / "r2.fq"))
    path = str(tmp_path / "reads.fq.gz")
    with open(path, "wb") as f:
        f.write(gzip.compress(open(tmp_path / "r1.fq", "rb").read()) + gzip.compress(open(tmp_path / "r2.fq", "rb").read()))
    return path, [str(d), other]


# ---- the rule against the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_oracle_parity(emu, k, tmp_path):
    reads, asm = parity_case(tmp_path)
    info, want = check(emu, reads, asm, k, tmp_path / "out")
    assert info["assemblies"] == 2 and info["contigs"] == 3 and info["selected_reads"] > 0 and info["peak"] is not None
    # kmer_histogram.tsv is genome_size -d's file
    gs_dir = tmp_path / "gs"
    api.genome_size_estimate(reads, k, dir=str(gs_dir), lib=emu)
    assert open(gs_dir / "kmer_histogram.tsv", "rb").read() == open(tmp_path / "out" / "kmer_histogram.tsv", "rb").read()
    # the fraction histogram covers every scored read; the selected reads are a tail of it
    rows = [list(map(int, line.split("\t"))) for line in open(tmp_path / "out" / "fraction_histogram.tsv").read().splitlines()[1:]]
    assert [r[0] for r in rows] == list(range(101)) and sum(r[1] for r in rows) == info["scored_reads"]
    assert sum(r[1] for r in rows[50:]) == info["selected_reads"]


def test_same_outputs_with_min_count_partitions_and_windows(emu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path)
    base_info = api.unassembled(reads, asm, str(tmp_path / "base"), k=21, lib=emu)
    base = out_files(tmp_path / "base")
    assert base_info["partitions"] == 1 and base_info["read_passes"] == 1
    info = api.unassembled(reads, asm, str(tmp_path / "given"), k=21, min_count=base_info["min_count"], lib=emu)
    assert out_files(tmp_path / "given") == base
    settings = [{"AC_GS_PARTITIONS": "1"}, {"AC_GS_TABLE_SLOTS": str(2 * base_info["read_windows"] // 4 + 1)},
                {"AC_SUBSAMPLE_WINDOW": "20000"}, {"AC_SUBSAMPLE_WINDOW": "77777", "AC_GS_PARTITIONS": "2"}]
    for i, env in enumerate(settings):
        for name, value in env.items():
            monkeypatch.setenv(name, value)
        info = api.unassembled(reads, asm, str(tmp_path / f"o{i}"), k=21, lib=emu)
        for name in env:
            monkeypatch.delenv(name)
        assert out_files(tmp_path / f"o{i}") == base, env
        if "AC_GS_TABLE_SLOTS" in env:
            assert info["partitions"] == 4
        if "AC_SUBSAMPLE_WINDOW" in env:
            assert info["read_passes"] == 2


# ---- what the rule means: sequence missing at known places ---------------------------------------------------------------------------
CHROM, PLAS, DEL = 150_000, 6_000, (60_000, 80_000)


def meaning_case(tmp_path, copies):
    """A 150 kbp circular chromosome at 40x and a 6 kbp circular plasmid at `copies` copies, 1% errors; the chromosome's reads first,
    then the plasmid's.  Assemblies: the truth, the chromosome alone, and the chromosome alone without a 20 kbp stretch."""
    rng = synth.SplitMix64(0xB5)
    chrom = synth.make_genome(rng, CHROM, repeats=False).tobytes().decode()
    plas = synth.make_genome(rng, PLAS, repeats=False).tobytes().decode()
    paths = {}
    for name, recs in {"truth": [("chrom circular=true", chrom), ("plasmid circular=true", plas)],
                       "chrom": [("chrom circular=true", chrom)],
                       "deleted": [("chrom circular=true", chrom[:DEL[0]] + chrom[DEL[1]:])]}.items():
        paths[name] = str(tmp_path / f"{name}.fasta")
        write_fasta(paths[name], recs)
    chrom_reads, plas_reads = noisy(chrom, 40, 51, n50=4000), noisy(plas, 40 * copies, 52, n50=3000)
    reads = str(tmp_path / f"reads_{copies}.fq")
    synth.write_reads(chrom_reads + plas_reads, reads)
    return reads, paths, len(chrom_reads), len(plas_reads)


@pytest.mark.parametrize("copies", [3, 8])
def test_missing_plasmid(emu, copies, tmp_path):
    reads, paths, n_chrom, n_plas = meaning_case(tmp_path, copies)
    info, want = check(emu, reads, [paths["chrom"]], 21, tmp_path / "out")
    sel = np.array(want["selected"])
    plas_sel, chrom_sel = int((sel >= n_chrom).sum()), int((sel < n_chrom).sum())
    # targets fixed before the first run
    assert plas_sel >= 0.95 * n_plas
    assert chrom_sel <= 0.001 * n_chrom
    assert abs(info["absent_copy_ratio"] - copies) <= 0.15 * copies
    # seeded, so pinned exactly: (chromosome reads, plasmid reads, plasmid reads selected, chromosome reads selected, absent_kmers,
    # absent_median, p*, absent_copy_ratio)
    pinned = {3: (1720, 269, 269, 0, 6000, 97.0, 32.088235294117645, 3.022914757103575),
              8: (1720, 743, 743, 0, 6000, 258.0, 32.088235294117645, 8.040329972502292)}
    assert (n_chrom, n_plas, plas_sel, chrom_sel, info["absent_kmers"], info["absent_median"], info["peak"],
            info["absent_copy_ratio"]) == pinned[copies]


def test_deletion_plus_plasmid_and_complete(emu, tmp_path):
    reads, paths, n_chrom, n_plas = meaning_case(tmp_path, 3)
    info, _ = check(emu, reads, [paths["deleted"]], 21, tmp_path / "deleted")
    want = (DEL[1] - DEL[0]) + PLAS
    assert abs(info["absent_kmers"] - want) <= 0.02 * want
    assert (info["absent_kmers"], info["selected_reads"], info["absent_median"]) == (26019, 510, 35.0)     # seeded, so pinned exactly
    info, _ = check(emu, reads, [paths["truth"]], 21, tmp_path / "truth")
    assert info["selected_reads"] == 0 and open(tmp_path / "truth" / "unassembled.fastq", "rb").read() == b""
    assert open(tmp_path / "truth" / "unassembled.tsv").read() == "read\tlength\tsolid_kmers\tabsent_kmers\n"


# ---- errors -------------------------------------------------------------------------------------------------------------------------
def test_errors(emu, tmp_path):
    asm, reads = str(tmp_path / "a.fasta"), str(tmp_path / "r.fq")
    write_fasta(asm, [("a", "ACGT" * 20)])
    synth.write_reads([("r", b"ACGT" * 20, b"I" * 80)], reads)
    out = str(tmp_path / "o")

    def err(code, message, assemblies=(asm,), reads=reads, out=out, **kw):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.unassembled(reads, list(assemblies), out, lib=emu, **kw)
        assert e.value.code == code and (e.value.message == message if isinstance(message, str) else message(e.value.message)), e.value.message

    for k in (9, 10, 12, 22, 33):
        err(-6, "--kmer must be odd and between 11 and 31", k=k)
    for t in (0, H):
        err(-6, f"--min_count must be between 1 and {H - 1}", min_count=t)
    err(-6, "--min_solid must be at least 1", min_solid=0)
    for f in (0.0, -0.5, 1.0001, float("nan")):
        err(-6, "--min_fraction must be above 0 and at most 1", min_fraction=f)
    err(-6, f"file does not exist: {tmp_path / 'nope.fq'}", reads=str(tmp_path / "nope.fq"))
    write_fasta(str(tmp_path / "short.fasta"), [("s", "ACGTNACGTACGTACGTACG"), ("t", "ACG")])
    (tmp_path / "d").mkdir()
    write_fasta(str(tmp_path / "d" / "x.fasta"), [("x", "ACGTACGTAC")])
    err(-6, f"no k-mer windows: no contig of {tmp_path / 'short.fasta'}, {tmp_path / 'd' / 'x.fasta'} holds 21 consecutive A, C, G or T bases",
        assemblies=[str(tmp_path / "short.fasta"), str(tmp_path / "d")])
    synth.write_reads([("r", b"ACGTN" * 20, b"I" * 100)], str(tmp_path / "short.fq"))
    err(-6, "no k-mer windows: no read holds 21 consecutive A, C, G or T bases", reads=str(tmp_path / "short.fq"))
    for data, rec, why in ((b"@a\nAC\n+\nII\nb\nAC\n+\nII\n", 2, "expected '@' at the start of the header line"),
                           (b"@a\nAC\n+\nII\n@b\nAC", 2, "truncated record"), (b"@a\nACG\n+\nII\n", 1, "sequence and quality lengths differ")):
        open(tmp_path / "bad.fq", "wb").write(data)
        err(-6, f"Error reading FASTQ file: record {rec}: {why}", reads=str(tmp_path / "bad.fq"))
    rng = synth.SplitMix64(0xBA)                                  # error-free reads at 1x over each base: no valley
    g = synth.make_genome(rng, 5_000, repeats=False).tobytes().decode()
    synth.write_reads([(f"r{i}", g[i:i + 1000].encode(), b"I" * 1000) for i in range(0, 4_000, 1000)], str(tmp_path / "flat.fq"))
    err(-6, lambda m: m.startswith("no k-mer depth peak") and "--min_count" in m, reads=str(tmp_path / "flat.fq"))
    open(tmp_path / "file", "w").close()
    err(-6, f"{tmp_path / 'file'} exists but is not a directory", out=str(tmp_path / "file"), min_count=1)
    err(-6, lambda m: m.startswith(f"failed to create directory {tmp_path / 'file' / 'sub'}"), out=str(tmp_path / "file" / "sub"), min_count=1)
    os.environ["AC_UNASSEMBLED_TABLE_SLOTS"] = "100"              # 2 x 60 windows do not fit 100 slots
    try:
        err(-4, lambda m: "does not fit" in m, min_count=1)
        os.environ["AC_UNASSEMBLED_TABLE_SLOTS"] = "121"          # the set (120 slots) fits; with the read's counters and words it does not
        err(-4, lambda m: "do not fit" in m, min_count=1)
    finally:
        del os.environ["AC_UNASSEMBLED_TABLE_SLOTS"]
    assert os.listdir(out) == []


def test_unwritable_out_dir(emu, tmp_path):
    reads, asm = parity_case(tmp_path)
    out = tmp_path / "ro"
    out.mkdir()
    os.chmod(out, 0o500)
    try:
        if os.access(out, os.W_OK):
            pytest.skip("the directory stays writable (running as root)")
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.unassembled(reads, asm, str(out), k=21, lib=emu)
        assert e.value.code == -5 and e.value.message == f"cannot write {out}/unassembled.fastq"
    finally:
        os.chmod(out, 0o700)


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
    reads, asm = parity_case(tmp_path)
    out = tmp_path / "cli"
    r = run(emu_cli, "unassembled", "-r", reads, "-i", *asm, "-o", out, "--kmer", "15")
    assert r.returncode == 0, r.stderr
    assert r.stdout == open(out / "summary.tsv").read()
    want = O.run(reads, asm, 15)
    assert out_files(out) == want["files"]
    assert "Starting autocycler unassembled" in r.stderr and "not in the reference" in r.stderr and f"valley: {want['valley']}" in r.stderr
    assert f"k-mer depth peak: {want['peak']:.2f}" in r.stderr and r.stderr.rstrip().endswith("unassembled.fastq")
    r = run(emu_cli, "unassembled", "--reads", reads, "--assemblies", asm[1], "--out_dir", out, "--kmer", "15", "--min_count", "3",
            "--min_solid", "50", "--min_fraction", "0.25")
    assert r.returncode == 0 and r.stdout == O.run(reads, [asm[1]], 15, 3, 50, 0.25)["files"]["summary.tsv"].decode()
    assert "min_count: 3 (given)" in r.stderr and "--min_fraction 0.25" in r.stderr
    usage = "Usage: autocycler unassembled"
    for args in (["unassembled"], ["unassembled", "-r", reads], ["unassembled", "-r", reads, "-i", asm[1]], ["unassembled", "-i", asm[1], "-o", out]):
        r = run(emu_cli, *args)
        assert r.returncode == 2 and r.stderr.startswith(usage) and r.stdout == "", args
    r = run(emu_cli, "unassembled", "-h")
    assert r.returncode == 0 and r.stderr.startswith(usage) and "not in the reference" in r.stderr
    for flag, value in (("--kmer", "x"), ("--kmer", "9"), ("--kmer", "22"), ("--kmer", "33"), ("--min_solid", "0"), ("--min_solid", "-1"),
                        ("--min_fraction", "0"), ("--min_fraction", "1.5"), ("--min_fraction", "-0.1"), ("--min_fraction", "nan"),
                        ("--min_fraction", "x"), ("--min_count", "2.5")):
        r = run(emu_cli, "unassembled", "-r", reads, "-i", asm[1], "-o", out, flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'") and usage in r.stderr, (flag, value)
    r = run(emu_cli, "unassembled", "-r", reads, "-i", asm[1], "-o", out, "--bogus", "1")
    assert r.returncode == 2 and r.stderr.startswith("error: unexpected argument '--bogus'")
    r = run(emu_cli, "unassembled", "-r", tmp_path / "nope.fq", "-i", asm[1], "-o", out)
    assert r.returncode == 1 and r.stderr.endswith(f"Error: file does not exist: {tmp_path / 'nope.fq'}\n") and r.stdout == ""
    r = run(emu_cli, "unassembled", "-r", reads, "-i", asm[1], "-o", out, "--min_count", "0")
    assert r.returncode == 1 and r.stderr.endswith(f"Error: --min_count must be between 1 and {H - 1}\n")


# ---- the GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_gpu_oracle_parity(gpu, k, tmp_path):
    reads, asm = parity_case(tmp_path)
    check(gpu, reads, asm, k, tmp_path / "out")


@pytest.mark.gpu
def test_gpu_partitions_and_windows(gpu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path)
    base_info, _ = check(gpu, reads, asm, 21, tmp_path / "base")
    base = out_files(tmp_path / "base")
    monkeypatch.setenv("AC_GS_TABLE_SLOTS", str(2 * base_info["read_windows"] // 4 + 1))
    info = api.unassembled(reads, asm, str(tmp_path / "p4"), k=21, lib=gpu)
    assert info["partitions"] == 4 and out_files(tmp_path / "p4") == base
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", "50000")
    info = api.unassembled(reads, asm, str(tmp_path / "w"), k=21, lib=gpu)
    assert info["read_passes"] == 2 and out_files(tmp_path / "w") == base


@pytest.mark.gpu
def test_gpu_two_missing_plasmids(gpu, tmp_path):
    """A 2 Mbp chromosome at 40x with a 5 kbp plasmid at 6 copies and a 12 kbp plasmid at 2, neither in the assembly, 1% errors."""
    rng = synth.SplitMix64(0xB9)
    chrom = synth.make_genome(rng, 2_000_000).tobytes().decode()
    p1 = synth.make_genome(rng, 5_000, repeats=False).tobytes().decode()
    p2 = synth.make_genome(rng, 12_000, repeats=False).tobytes().decode()
    asm = str(tmp_path / "chrom.fasta")
    write_fasta(asm, [("chrom circular=true", chrom)])
    chrom_reads, r1, r2 = noisy(chrom, 40, 61, n50=8000), noisy(p1, 240, 62), noisy(p2, 80, 63)
    reads = str(tmp_path / "r.fq")
    synth.write_reads(chrom_reads + r1 + r2, reads)
    info, want = check(gpu, reads, [asm], 21, tmp_path / "out")
    sel = np.array(want["selected"])
    assert (sel >= len(chrom_reads)).sum() >= 0.95 * (len(r1) + len(r2)) and (sel < len(chrom_reads)).sum() <= 0.001 * len(chrom_reads)
