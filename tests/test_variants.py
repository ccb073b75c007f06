"""`autocycler variants`: the alleles the reads carry beside the consensus, with every position's alternatives screened on the GPU
(DESIGN.md §23).  `variants` is not in the reference, so it is pinned against the numpy oracle of the rule (tests/variants_oracle.py) and,
on mixtures of reads from a truth genome and from a copy with variants planted at known places, by what the rule means.  The CPU tests
run the product's code through the host-emulation library (the kernels' bodies, serially); the tests marked gpu run the CUDA build on the
H100."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import variants_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
H = api.GENOME_SIZE_BINS
FILES = ["summary.tsv", "variants.vcf"]
OTHER = {b: "ACGT"[("ACGT".index(b) + 1) % 4] for b in "ACGT"}


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


def noisy(genome, depth, seed, n50=3000):
    g = genome.encode() if isinstance(genome, str) else genome.tobytes()
    return list(synth.make_noisy_reads(np.frombuffer(g, dtype=np.uint8), depth=depth, n50=n50, seed=seed, sub=0.005, ins=0.0025,
                                       dele=0.0025))


def out_files(out_dir):
    return {n: open(os.path.join(out_dir, n), "rb").read() for n in sorted(os.listdir(out_dir))}


def check(lib, reads, assembly, k, out_dir, **kw):
    """Every file the product writes against the oracle's (and no other file); returns (info, oracle result)."""
    info = api.variants(reads, assembly, str(out_dir), k=k, lib=lib, **kw)
    want = O.run(reads, assembly, k, **kw)
    got = out_files(out_dir)
    assert sorted(got) == sorted(want["files"]) == FILES
    for name, data in want["files"].items():
        assert got[name] == data, name
    assert info["min_count"] == want["t"] and info["read_windows"] == want["W"] and info["valley"] == (want["valley"] or 0)
    assert (info["positions"], info["screened"], info["candidates"], info["passing"], info["variants"]) == \
        (want["positions"], want["screened"], want["candidates"], want["passing"], len(want["rows"]))
    return info, want


def two_members(tmp_path, reads, name="reads.fq.gz"):
    half = len(reads) // 2
    synth.write_reads(reads[:half], str(tmp_path / "r1.fq"))
    synth.write_reads(reads[half:], str(tmp_path / "r2.fq"))
    path = str(tmp_path / name)
    with open(path, "wb") as f:
        f.write(gzip.compress(open(tmp_path / "r1.fq", "rb").read()) + gzip.compress(open(tmp_path / "r2.fq", "rb").read()))
    return path


def parity_case(tmp_path, k, length=20_000):
    """A circular chromosome, a linear contig, and pieces of the chromosome k + 31, k + 32 and k + 33 bases long (so that S(p, b) straddles
    packed words at every offset), with lowercase and N/IUPAC bases in the assembly; reads of the truth at 40x and of a copy with 0.3%
    differences at 15x, both with 1% errors, in two gzip members."""
    rng = synth.SplitMix64(0x7A1)
    chrom, lin = synth.make_genome(rng, length + k, repeats=False), synth.make_genome(rng, 5_000 + 3 * k, repeats=False)
    var = synth.mutate(synth.SplitMix64(0x7A2), chrom, sub=2e-3, ins=5e-4, dele=5e-4)
    var_lin = synth.mutate(synth.SplitMix64(0x7A3), lin, sub=2e-3, ins=5e-4, dele=5e-4)
    c, ln = chrom.tobytes().decode(), lin.tobytes().decode()
    asm = str(tmp_path / "asm.fasta")
    pieces = [(f"piece{j} length={k + 31 + j}", c[3_000 + 500 * j:3_000 + 500 * j + k + 31 + j]) for j in range(3)]
    write_fasta(asm, [("chrom length=x circular=TRUE", c[:4_000].lower() + c[4_000:]), ("lin", ln[:2_000] + "NRY" + ln[2_003:])] + pieces)
    reads = noisy(chrom, 40, 0x7A4) + noisy(var, 15, 0x7A5) + noisy(lin, 40, 0x7A6, n50=2000) + noisy(var_lin, 15, 0x7A7, n50=2000)
    return two_members(tmp_path, reads), asm


# ---- the rule against the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_oracle_parity(emu, k, tmp_path):
    reads, asm = parity_case(tmp_path, k)
    info, want = check(emu, reads, asm, k, tmp_path / "out")
    assert info["variants"] > 10 and info["screened"] < info["positions"] // 10
    assert info["insertions"] > 0 and info["deletions"] > 0 and info["substitutions"] > 0


def test_same_outputs_with_partitions_windows_tight_tables_and_min_count(emu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path, 21)
    base_info, _ = check(emu, reads, asm, 21, tmp_path / "base", max_indel=3)
    base = out_files(tmp_path / "base")
    assert base_info["partitions"] == 1 and base_info["batches"] == 1
    api.variants(reads, asm, str(tmp_path / "given"), k=21, min_count=base_info["min_count"], max_indel=3, lib=emu)
    assert out_files(tmp_path / "given") == base
    # a budget of the window table's slots, which holds a few dozen positions' candidates (2 x 2,118 slots each at k = 21, L = 3)
    tight = str(base_info["table_bytes"] // 16)
    assert base_info["loci"] > int(tight) // (2 * 2_118)
    settings = [{"AC_GS_PARTITIONS": "2"}, {"AC_GS_PARTITIONS": "4"}, {"AC_SUBSAMPLE_WINDOW": "30000"}, {"AC_VARIANTS_TABLE_SLOTS": tight},
                {"AC_GS_PARTITIONS": "2", "AC_VARIANTS_TABLE_SLOTS": tight}]
    for i, env in enumerate(settings):
        for name, value in env.items():
            monkeypatch.setenv(name, value)
        info = api.variants(reads, asm, str(tmp_path / f"o{i}"), k=21, max_indel=3, lib=emu)
        for name in env:
            monkeypatch.delenv(name)
        assert out_files(tmp_path / f"o{i}") == base, env
        assert (info["screened"], info["candidates"], info["passing"]) == (base_info["screened"], base_info["candidates"], base_info["passing"])
        if "AC_GS_PARTITIONS" in env:
            assert info["partitions"] == int(env["AC_GS_PARTITIONS"])
        if "AC_VARIANTS_TABLE_SLOTS" in env:
            assert info["batches"] > base_info["batches"]


# ---- what the rule means: variants planted at known places --------------------------------------------------------------------------
def plant(truth, events):
    """truth with events (position, kind, argument) in ascending position, far apart: ("sub", base), ("ins", bases) put before the
    position, ("del", d) bases removed there."""
    out, at = [], 0
    for x, kind, arg in events:
        out.append(truth[at:x])
        if kind == "sub":
            out.append(arg)
            at = x + 1
        elif kind == "ins":
            out.append(arg)
            at = x
        else:
            at = x + arg
    out.append(truth[at:])
    return "".join(out)


def normalized(truth, x, kind, arg):
    """The VCF (POS, REF, ALT) of an event on truth, indels shifted left over the bases they repeat and anchored on the base before."""
    if kind == "sub":
        return x + 1, truth[x], arg
    if kind == "del":
        while x > 1 and truth[x - 1] == truth[x + arg - 1]:
            x -= 1
        return x, truth[x - 1:x + arg], truth[x - 1]
    s = arg
    while x > 1 and truth[x - 1] == s[-1]:
        s, x = s[-1] + s[:-1], x - 1
    return x, truth[x - 1], truth[x - 1] + s


def homopolymer(s, x, n=3):
    while len(set(s[x:x + n])) != 1:
        x += 1
    return x


def meaning_events(chrom, step, count):
    """count events `step` apart, every kind in turn, the first across the circular junction (a substitution at position 3)."""
    ev = [(3, "sub", OTHER[chrom[3]])]
    for i in range(1, count):
        x = i * step
        kind = i % 8
        if kind == 0:
            ev.append((x, "sub", OTHER[chrom[x]]))
        elif kind <= 3:
            ev.append((x, "ins", "GATTACA"[:kind]))
        elif kind <= 6:
            ev.append((x, "del", kind - 3))
        else:
            h = homopolymer(chrom, x)
            ev.append((h, "ins", chrom[h]))                  # a homopolymer run one base longer in the minority
    return ev


def meaning_case(tmp_path, length=40_000, step=800, truth_depth=40, minority_depth=15):
    """A circular chromosome and reads of it at truth_depth, with reads of a copy carrying planted variants at minority_depth; the copy also
    has two substitutions 5 bp apart (closer than k), which give no row."""
    chrom = synth.make_genome(synth.SplitMix64(0x7B1), length, repeats=False).tobytes().decode()
    events = meaning_events(chrom, step, length // step - 2)
    close = length - step
    minority = plant(chrom, events + [(close, "sub", OTHER[chrom[close]]), (close + 5, "sub", OTHER[chrom[close + 5]])])
    truth, var = str(tmp_path / "truth.fasta"), str(tmp_path / "minority.fasta")
    write_fasta(truth, [("chrom circular=true", chrom)])
    write_fasta(var, [("chrom circular=true", minority)])
    reads = str(tmp_path / "reads.fq")
    synth.write_reads(noisy(chrom, truth_depth, 0x7B2) + noisy(minority, minority_depth, 0x7B3), reads)
    return reads, truth, var, chrom, events, close


def check_meaning(lib, tmp_path, oracle=True, **case):
    reads, truth, _, chrom, events, close = meaning_case(tmp_path, **case)
    out = tmp_path / "out"
    if oracle:
        info, _ = check(lib, reads, truth, 21, out, max_indel=3)
    else:
        info = api.variants(reads, truth, str(out), k=21, max_indel=3, lib=lib)
    got = [(r["pos"], r["ref"], r["alt"]) for r in info["rows"]]
    want = [normalized(chrom, *e) for e in events]
    assert sorted(got) == sorted(want)                       # each planted variant exactly once, and nothing else
    assert not any(close - 21 < r["pos"] <= close + 26 for r in info["rows"])
    # the fraction of reads that carry the minority is 15 / 55; a minimum over k-mer counts is biased by read errors (an error in any
    # of the k + s k-mers lowers one count), so the band is loose
    assert all(0.12 < r["af"] < 0.45 for r in info["rows"]), [r["af"] for r in info["rows"]]
    # PK counts the checked k-mers the assembly holds: a substitution's are all new, but an indel in a repeat (here the homopolymer runs and
    # the insertions whose bases repeat the ones before them) has windows that slide onto the assembly's own
    assert info["alt_major"] == 0 and all(r["pk"] == 0 for r in info["rows"] if len(r["ref"]) == len(r["alt"]))
    return reads, truth, out, info


def test_planted_variants(emu, tmp_path):
    reads, truth, out, info = check_meaning(emu, tmp_path)
    kinds = {"sub": 0, "ins": 0, "del": 0}
    for _, kind, _ in meaning_events(open(truth).read().split("\n")[1], 800, 40_000 // 800 - 2):
        kinds[kind] += 1
    assert (info["substitutions"], info["insertions"], info["deletions"]) == (kinds["sub"], kinds["ins"], kinds["del"])
    assert any(r["pos"] == 4 for r in info["rows"])         # the site across the junction
    # --max_indel 0: the substitutions only
    info0, _ = check(emu, reads, truth, 21, tmp_path / "l0", max_indel=0)
    assert info0["variants"] == kinds["sub"] and info0["insertions"] == info0["deletions"] == 0


def test_truth_only_reads_give_a_header_only_vcf(emu, tmp_path):
    chrom = synth.make_genome(synth.SplitMix64(0x7C1), 20_000, repeats=False).tobytes().decode()
    asm, reads = str(tmp_path / "asm.fasta"), str(tmp_path / "reads.fq")
    write_fasta(asm, [("chrom circular=true", chrom)])
    synth.write_reads(noisy(chrom, 50, 0x7C2), reads)
    info, _ = check(emu, reads, asm, 21, tmp_path / "out", max_indel=3)
    vcf = open(tmp_path / "out" / "variants.vcf").read()
    assert info["variants"] == 0 and vcf.splitlines()[-1].startswith("#CHROM") and "##contig=<ID=chrom,length=20000>" in vcf


def test_assembly_with_the_minority_allele(emu, tmp_path):
    """The minority copy as the assembly: every planted site is a row whose alternative is the majority, counted in alt_major."""
    reads, _, var, _, events, _ = meaning_case(tmp_path, length=20_000)
    info, _ = check(emu, reads, var, 21, tmp_path / "out", max_indel=3)
    assert info["alt_major"] >= len(events) and all(r["af"] > 0.55 for r in info["rows"] if r["ak"] > r["rk"])


def test_two_copy_repeat_gives_pk(emu, tmp_path):
    """A 200 bp repeat twice in a circular genome, its copies differing at one base.  Error-free reads that start at every base give every
    k-mer the same count, so each copy carries the other's base as an alternative at AF 0.5, whose k-mers are the assembly's own."""
    rng = synth.SplitMix64(0x7D1)
    g = list(synth.make_genome(rng, 3_000, repeats=False).tobytes().decode())
    rep = synth.make_genome(rng, 200, repeats=False).tobytes().decode()
    g[500:700], g[2000:2200] = rep, rep
    g[600], g[2100] = "C", "G"
    truth = "".join(g)
    reads = str(tmp_path / "reads.fq")
    synth.write_reads([(f"r{i}", (truth + truth)[i:i + 120].encode(), b"I" * 120) for i in range(len(truth))], reads)
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("genome circular=true", truth)])
    info, _ = check(emu, reads, asm, 21, tmp_path / "out", min_count=2)
    assert [(r["pos"], r["ref"], r["alt"], r["af"], r["pk"]) for r in info["rows"]] == [(601, "C", "G", 0.5, 21), (2101, "G", "C", 0.5, 21)]
    assert info["paralog"] == 2


# ---- errors -------------------------------------------------------------------------------------------------------------------------
def test_errors(emu, tmp_path):
    asm, reads = str(tmp_path / "a.fasta"), str(tmp_path / "r.fq")
    write_fasta(asm, [("a", "ACGT" * 20)])
    synth.write_reads([("r", b"ACGT" * 20, b"I" * 80)], reads)
    out = str(tmp_path / "o")

    def err(code, message, assembly=asm, reads=reads, out=out, **kw):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.variants(reads, assembly, out, lib=emu, **kw)
        assert e.value.code == code and (e.value.message == message if isinstance(message, str) else message(e.value.message)), e.value.message

    for k in (9, 10, 12, 22, 33):
        err(-6, "--kmer must be odd and between 11 and 31", k=k)
    for t in (0, H):
        err(-6, f"--min_count must be between 1 and {H - 1}", min_count=t)
    err(-6, "--max_indel must be between 0 and 3", max_indel=4)
    for f in (0.0, -0.1, 1.5, float("nan")):
        err(-6, "--min_fraction must be above 0 and at most 1", min_fraction=f)
    err(-6, f"file does not exist: {tmp_path / 'nope.fq'}", reads=str(tmp_path / "nope.fq"))
    err(-6, f"file does not exist: {tmp_path / 'nope.fasta'}", assembly=str(tmp_path / "nope.fasta"))
    write_fasta(str(tmp_path / "short.fasta"), [("s", "ACGTNACGTACGTACGTACG"), ("t", "ACG")])
    err(-6, f"{tmp_path / 'short.fasta'}: no k-mer windows: no contig holds 21 consecutive A, C, G or T bases", assembly=str(tmp_path / "short.fasta"))
    synth.write_reads([("r", b"ACGTN" * 20, b"I" * 100)], str(tmp_path / "short.fq"))
    err(-6, "no k-mer windows: no read holds 21 consecutive A, C, G or T bases", reads=str(tmp_path / "short.fq"))
    g = synth.make_genome(synth.SplitMix64(0x7E1), 5_000, repeats=False).tobytes().decode()
    synth.write_reads([(f"r{i}", g[i:i + 1000].encode(), b"I" * 1000) for i in range(0, 4_000, 1000)], str(tmp_path / "flat.fq"))
    err(-6, lambda m: m.startswith("no k-mer depth peak") and "--min_count" in m, reads=str(tmp_path / "flat.fq"))
    open(tmp_path / "file", "w").close()
    err(-6, f"{tmp_path / 'file'} exists but is not a directory", out=str(tmp_path / "file"), min_count=1)
    os.environ["AC_VARIANTS_TABLE_SLOTS"] = "100"                 # 2 x 60 windows and more do not fit 100 slots
    try:
        err(-4, lambda m: m.startswith("variants: the contigs' k-mer table") and "does not fit" in m, min_count=1)
    finally:
        del os.environ["AC_VARIANTS_TABLE_SLOTS"]
    assert os.listdir(out) == []


def test_one_position_candidates_do_not_fit(emu, tmp_path, monkeypatch):
    """A budget of 3,000 slots holds the window table of a 1 kbp contig and one position's candidates at k = 21, L = 1 (2 x 176), but not
    one position's at k = 31, L = 3 (2 x 2,628)."""
    g = synth.make_genome(synth.SplitMix64(0x7E2), 1_000, repeats=False).tobytes().decode()
    var = g[:500] + OTHER[g[500]] + g[501:]
    asm, reads = str(tmp_path / "a.fasta"), str(tmp_path / "r.fq")
    write_fasta(asm, [("a", g)])
    synth.write_reads([(f"r{i}", s[i:i + 100].encode(), b"I" * 100) for s in (g, var) for i in range(0, 900, 3)], reads)
    monkeypatch.setenv("AC_VARIANTS_TABLE_SLOTS", "3000")
    info = api.variants(reads, asm, str(tmp_path / "ok"), k=21, min_count=2, lib=emu)
    assert info["variants"] == 1 and info["rows"][0]["pos"] == 501
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.variants(reads, asm, str(tmp_path / "big"), k=31, max_indel=3, min_count=2, lib=emu)
    assert e.value.code == -4 and "one locus's candidate table" in e.value.message


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
    reads, asm = parity_case(tmp_path, 15, length=8_000)
    out = tmp_path / "cli"
    r = run(emu_cli, "variants", "-r", reads, "-i", asm, "-o", out, "--kmer", "15")
    assert r.returncode == 0, r.stderr
    assert r.stdout == open(out / "summary.tsv").read()
    want = O.run(reads, asm, 15)
    assert out_files(out) == want["files"]
    assert "Starting autocycler variants" in r.stderr and "not in the reference" in r.stderr and f"valley: {want['valley']}" in r.stderr
    assert f"screened: {want['screened']}" in r.stderr and r.stderr.rstrip().endswith("variants.vcf")
    r = run(emu_cli, "variants", "--reads", reads, "--input", asm, "--out_dir", out, "--kmer", "15", "--min_count", "3", "--max_indel", "2",
            "--min_fraction", "0.25")
    assert r.returncode == 0 and r.stdout == O.run(reads, asm, 15, 3, 2, 0.25)["files"]["summary.tsv"].decode()
    assert "min_count: 3 (given)" in r.stderr and "--max_indel 2" in r.stderr and "--min_fraction 0.25" in r.stderr
    usage = "Usage: autocycler variants"
    for args in (["variants"], ["variants", "-r", reads], ["variants", "-r", reads, "-i", asm], ["variants", "-i", asm, "-o", out]):
        r = run(emu_cli, *args)
        assert r.returncode == 2 and r.stderr.startswith(usage) and r.stdout == "", args
    r = run(emu_cli, "variants", "-h")
    assert r.returncode == 0 and r.stderr.startswith(usage) and "not in the reference" in r.stderr
    for flag, value in (("--kmer", "x"), ("--kmer", "9"), ("--kmer", "22"), ("--kmer", "33"), ("--min_count", "0"), ("--min_count", "16384"),
                        ("--min_count", "2.5"), ("--max_indel", "4"), ("--max_indel", "-1"), ("--max_indel", "x"), ("--min_fraction", "0"),
                        ("--min_fraction", "1.01"), ("--min_fraction", "-0.5"), ("--min_fraction", "x"), ("--min_fraction", "nan")):
        r = run(emu_cli, "variants", "-r", reads, "-i", asm, "-o", out, flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'") and usage in r.stderr, (flag, value)
    r = run(emu_cli, "variants", "-r", reads, "-i", asm, "-o", out, "--bogus", "1")
    assert r.returncode == 2 and r.stderr.startswith("error: unexpected argument '--bogus'")
    r = run(emu_cli, "variants", "-r", tmp_path / "nope.fq", "-i", asm, "-o", out)
    assert r.returncode == 1 and r.stderr.endswith(f"Error: file does not exist: {tmp_path / 'nope.fq'}\n") and r.stdout == ""
    write_fasta(str(tmp_path / "short.fasta"), [("s", "ACGTACGT")])
    r = run(emu_cli, "variants", "-r", reads, "-i", tmp_path / "short.fasta", "-o", out)
    assert r.returncode == 1 and r.stderr.endswith("holds 21 consecutive A, C, G or T bases\n")


# ---- the GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [21, 31])
def test_gpu_oracle_parity(gpu, k, tmp_path):
    reads, asm = parity_case(tmp_path, k)
    check(gpu, reads, asm, k, tmp_path / "out")


@pytest.mark.gpu
def test_gpu_partitions(gpu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path, 21)
    monkeypatch.setenv("AC_GS_PARTITIONS", "2")
    info, _ = check(gpu, reads, asm, 21, tmp_path / "out")
    assert info["partitions"] == 2


@pytest.mark.gpu
def test_gpu_1mbp_mixture_equals_emulation(gpu, emu, tmp_path):
    reads, truth, _, _, events, _ = meaning_case(tmp_path, length=1_000_000, step=5_000)
    info = api.variants(reads, truth, str(tmp_path / "gpu"), k=21, max_indel=3, lib=gpu)
    api.variants(reads, truth, str(tmp_path / "emu"), k=21, max_indel=3, lib=emu)
    assert out_files(tmp_path / "gpu") == out_files(tmp_path / "emu")
    assert info["variants"] >= len(events) * 0.95
