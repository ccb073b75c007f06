"""`autocycler polish`: the consensus corrected where the reads' k-mers do not support it, with candidate edits scored on the GPU (DESIGN.md
§22).  `polish` is not in the reference, so it is pinned against the numpy oracle of the rule (tests/polish_oracle.py) and, on synthetic
assemblies with errors planted at known positions, by what the rule means.  The CPU tests run the product's code through the
host-emulation library (the kernels' bodies, serially); the tests marked gpu run the CUDA build on the H100."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import polish_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
H = api.GENOME_SIZE_BINS
FILES = ["edits.tsv", "polished.fasta", "remaining.bed", "rounds.tsv", "summary.tsv"]


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
    info = api.polish(reads, assembly, str(out_dir), k=k, lib=lib, **kw)
    want = O.run(reads, assembly, k, **kw)
    got = out_files(out_dir)
    assert sorted(got) == sorted(want["files"]) == FILES
    for name, data in want["files"].items():
        assert got[name] == data, name
    assert info["min_count"] == want["t"] and info["read_windows"] == want["W"] and info["valley"] == (want["valley"] or 0)
    assert info["edits"] == len(want["edits"]) and info["rounds"] == len(want["rounds"])
    return info, want


def parity_case(tmp_path, length=24_000):
    """A circular chromosome and a linear contig with seeded errors at 0.4% (some close together, some at the linear ends), lowercase
    and N bases in the assembly, reads at 40x with 1% errors in two gzip members."""
    rng = synth.SplitMix64(0xC1)
    chrom, lin = synth.make_genome(rng, length, repeats=False), synth.make_genome(rng, 6_000, repeats=False)
    m = synth.mutate(synth.SplitMix64(0xC2), chrom, sub=2e-3, ins=1e-3, dele=1e-3).tobytes().decode()
    ml = synth.mutate(synth.SplitMix64(0xC3), lin, sub=2e-3, ins=1e-3, dele=1e-3).tobytes().decode()
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("chrom length=x circular=TRUE", m[:5_000].lower() + m[5_000:]), ("lin", ml[:3_000] + "NRY" + ml[3_003:])])
    reads = noisy(chrom, 40, 0xC4) + noisy(lin, 40, 0xC5, n50=2000)
    half = len(reads) // 2
    synth.write_reads(reads[:half], str(tmp_path / "r1.fq"))
    synth.write_reads(reads[half:], str(tmp_path / "r2.fq"))
    path = str(tmp_path / "reads.fq.gz")
    with open(path, "wb") as f:
        f.write(gzip.compress(open(tmp_path / "r1.fq", "rb").read()) + gzip.compress(open(tmp_path / "r2.fq", "rb").read()))
    return path, asm


# ---- the rule against the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_oracle_parity(emu, k, tmp_path):
    reads, asm = parity_case(tmp_path)
    info, want = check(emu, reads, asm, k, tmp_path / "out")
    rows = want["rounds"]
    assert info["edits"] > 20 and info["unsupported_after"] < info["unsupported_before"]
    assert sum(r["none"] for r in rows) > 0 and sum(r["deferred"] for r in rows) > 0


def test_same_outputs_with_min_count_partitions_windows_and_tight_tables(emu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path)
    base_info, _ = check(emu, reads, asm, 21, tmp_path / "base", max_indel=2, rounds=4)
    base = out_files(tmp_path / "base")
    assert base_info["partitions"] == 1
    api.polish(reads, asm, str(tmp_path / "given"), k=21, min_count=base_info["min_count"], max_indel=2, rounds=4, lib=emu)
    assert out_files(tmp_path / "given") == base
    # a budget of the window table's slots: one locus's candidates take 2 x 1,064 of them at k = 21, L = 2, so a batch holds a few dozen
    tight = str(base_info["table_bytes"] // 16)
    settings = [{"AC_GS_PARTITIONS": "4"}, {"AC_SUBSAMPLE_WINDOW": "30000"}, {"AC_POLISH_TABLE_SLOTS": tight},
                {"AC_GS_PARTITIONS": "2", "AC_POLISH_TABLE_SLOTS": tight}]
    for i, env in enumerate(settings):
        for name, value in env.items():
            monkeypatch.setenv(name, value)
        info = api.polish(reads, asm, str(tmp_path / f"o{i}"), k=21, max_indel=2, rounds=4, lib=emu)
        for name in env:
            monkeypatch.delenv(name)
        assert out_files(tmp_path / f"o{i}") == base, env
        if "AC_GS_PARTITIONS" in env:
            assert info["partitions"] == int(env["AC_GS_PARTITIONS"])
        if "AC_POLISH_TABLE_SLOTS" in env:
            assert info["batches"] > base_info["batches"]


# ---- what the rule means: errors planted at known places -----------------------------------------------------------------------------
def plant(truth, errors):
    """truth with errors (truth position, kind, argument) applied, far apart and in ascending position: ("sub", base), ("ins", bases)
    put before the position, ("del", d) bases removed there.  -> (assembly, the edit polish should make for each: (position in the
    assembly, ref, alt), at the first base where the assembly and the truth differ)."""
    out, want, at, off = [], [], 0, 0
    for x, kind, arg in errors:
        out.append(truth[at:x])
        if kind == "sub":
            out.append(arg)
            want.append((x + off, arg, truth[x]))
            at = x + 1
            continue
        local = truth[x:x + 50]
        a = arg + local if kind == "ins" else local[arg:]
        i = next(j for j in range(50) if a[j] != local[j])     # the first base where they differ
        if kind == "ins":
            out.append(arg)
            want.append((x + off + i, a[i:i + len(arg)], "-"))
            at, off = x, off + len(arg)
        else:
            want.append((x + off + i, "-", local[i:i + arg]))
            at, off = x + arg, off - arg
    out.append(truth[at:])
    return "".join(out), want


def homopolymer(s, x, n=3):
    """The first position from x where a run of n equal bases starts."""
    while len(set(s[x:x + n])) != 1:
        x += 1
    return x


def meaning_errors(chrom, step, count):
    """count errors `step` apart on chrom, every kind in turn; the first is across the circular junction (position 3)."""
    errs = [(3, "sub", "ACGT"[("ACGT".index(chrom[3]) + 1) % 4])]
    for i in range(1, count):
        x = i * step
        kind = i % 9
        if kind == 0:
            errs.append((x, "sub", "ACGT"[("ACGT".index(chrom[x]) + 2) % 4]))
        elif kind <= 3:
            errs.append((x, "ins", "GATTACA"[:kind]))
        elif kind <= 6:
            errs.append((x, "del", kind - 3))
        elif kind == 7:
            h = homopolymer(chrom, x)
            errs.append((h, "ins", chrom[h]))                   # a homopolymer run one base long
        else:
            errs.append((homopolymer(chrom, x), "del", 1))       # ... and one base short
    return errs


def meaning_case(tmp_path, length=40_000, step=700):
    rng = synth.SplitMix64(0xC7)
    chrom = synth.make_genome(rng, length, repeats=False).tobytes().decode()
    lin = synth.make_genome(rng, 8_000, repeats=False).tobytes().decode()
    reads = str(tmp_path / "reads.fq")
    synth.write_reads(noisy(chrom, 40, 0xC8) + noisy(lin, 40, 0xC9, n50=2000), reads)
    asm_chrom, want = plant(chrom, meaning_errors(chrom, step, length // step - 1))
    # the linear contig: an error in its first k bases, and two errors 5 bp apart
    asm_lin, _ = plant(lin, [(5, "sub", "ACGT"[("ACGT".index(lin[5]) + 1) % 4]), (4_000, "sub", "ACGT"[("ACGT".index(lin[4_000]) + 1) % 4]),
                             (4_005, "sub", "ACGT"[("ACGT".index(lin[4_005]) + 1) % 4])])
    truth, asm = str(tmp_path / "truth.fasta"), str(tmp_path / "asm.fasta")
    write_fasta(truth, [("chrom circular=true", chrom), ("lin", lin)])
    write_fasta(asm, [("chrom circular=true", asm_chrom), ("lin", asm_lin)])
    return reads, truth, asm, chrom, lin, asm_lin, want


def check_meaning(lib, tmp_path, **case):
    reads, truth, asm, chrom, lin, asm_lin, want = meaning_case(tmp_path, **case)
    info, oracle = check(lib, reads, asm, 21, tmp_path / "out")
    polished = open(tmp_path / "out" / "polished.fasta").read()
    assert polished == f">chrom circular=true\n{chrom}\n>lin\n{asm_lin}\n"
    got = [(e["position"], e["ref"], e["alt"]) for e in info["applied"]]
    assert all(e["round"] == 1 and e["contig"] == "chrom" for e in info["applied"]) and got == want
    first = oracle["rounds"][0]
    assert (first["edited"], first["ambiguous"], first["deferred"], first["edge"], first["none"]) == (len(want), 0, 0, 1, 1)
    assert info["rounds"] == 2 and oracle["rounds"][1]["edited"] == 0
    bed = open(tmp_path / "out" / "remaining.bed").read().splitlines()
    assert "lin\t0\t26" in bed and any(line.startswith("lin\t") and int(line.split("\t")[1]) <= 4_000 < int(line.split("\t")[2]) for line in bed)
    assert not any(line.startswith("chrom\t") for line in bed)
    # the true genome as input: no edit, and polished.fasta is the input
    info, _ = check(lib, reads, truth, 21, tmp_path / "truth")
    assert info["edits"] == 0 and info["rounds"] == 1 and info["unsupported_before"] == 0
    assert open(tmp_path / "truth" / "polished.fasta", "rb").read() == open(truth, "rb").read()
    return reads, asm, info


def test_planted_errors(emu, tmp_path):
    reads, asm, _ = check_meaning(emu, tmp_path)
    # qv agrees: QV before and after and the remaining BED are qv's for the input and for polished.fasta, with the same reads, k and t
    summary = dict(zip(*(line.split("\t") for line in open(tmp_path / "out" / "summary.tsv").read().splitlines())))
    t = int(summary["min_count"])
    for path, field in ((asm, "qv_before"), (str(tmp_path / "out" / "polished.fasta"), "qv_after")):
        q = api.qv(reads, [path], str(tmp_path / f"qv_{field}"), k=21, min_count=t, lib=emu)
        assert q["assemblies"][0]["qv"] == (None if summary[field] == "" else float(summary[field]))
        row = open(tmp_path / f"qv_{field}" / "qv.tsv").read().splitlines()[1].split("\t")
        assert row[3] == summary[field]
    assert open(tmp_path / "qv_qv_after" / "unsupported" / "1.bed", "rb").read() == open(tmp_path / "out" / "remaining.bed", "rb").read()


def test_ambiguous_two_allele_repeat(emu, tmp_path):
    """A 200 bp repeat twice in a circular genome, its copies differing at one base (C and G); the assembly has a T there in the first
    copy.  Error-free reads that start at every base give every genome k-mer the same count, so both alleles score the same."""
    rng = synth.SplitMix64(0xCA)
    g = list(synth.make_genome(rng, 3_000, repeats=False).tobytes().decode())
    rep = synth.make_genome(rng, 200, repeats=False).tobytes().decode()
    g[500:700], g[2000:2200] = rep, rep
    g[600], g[2100] = "C", "G"
    truth = "".join(g)
    asm_seq = truth[:600] + "T" + truth[601:]
    reads = str(tmp_path / "reads.fq")
    doubled = truth + truth
    synth.write_reads([(f"r{i}", doubled[i:i + 120].encode(), b"I" * 120) for i in range(len(truth))], reads)
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("genome circular=true", asm_seq)])
    info, want = check(emu, reads, asm, 21, tmp_path / "out", min_count=2)
    assert info["edits"] == 0 and want["rounds"][0]["ambiguous"] == 1 and want["rounds"][0]["loci"] == 1
    assert open(tmp_path / "out" / "remaining.bed").read() == "genome\t580\t621\n"


# ---- errors -------------------------------------------------------------------------------------------------------------------------
def test_errors(emu, tmp_path):
    asm, reads = str(tmp_path / "a.fasta"), str(tmp_path / "r.fq")
    write_fasta(asm, [("a", "ACGT" * 20)])
    synth.write_reads([("r", b"ACGT" * 20, b"I" * 80)], reads)
    out = str(tmp_path / "o")

    def err(code, message, assembly=asm, reads=reads, out=out, **kw):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.polish(reads, assembly, out, lib=emu, **kw)
        assert e.value.code == code and (e.value.message == message if isinstance(message, str) else message(e.value.message)), e.value.message

    for k in (9, 10, 12, 22, 33):
        err(-6, "--kmer must be odd and between 11 and 31", k=k)
    for t in (0, H):
        err(-6, f"--min_count must be between 1 and {H - 1}", min_count=t)
    for n in (0, 5):
        err(-6, "--max_indel must be between 1 and 4", max_indel=n)
    for n in (0, 11):
        err(-6, "--rounds must be between 1 and 10", rounds=n)
    err(-6, f"file does not exist: {tmp_path / 'nope.fq'}", reads=str(tmp_path / "nope.fq"))
    err(-6, f"file does not exist: {tmp_path / 'nope.fasta'}", assembly=str(tmp_path / "nope.fasta"))
    write_fasta(str(tmp_path / "short.fasta"), [("s", "ACGTNACGTACGTACGTACG"), ("t", "ACG")])
    err(-6, f"{tmp_path / 'short.fasta'}: no k-mer windows: no contig holds 21 consecutive A, C, G or T bases", assembly=str(tmp_path / "short.fasta"))
    synth.write_reads([("r", b"ACGTN" * 20, b"I" * 100)], str(tmp_path / "short.fq"))
    err(-6, "no k-mer windows: no read holds 21 consecutive A, C, G or T bases", reads=str(tmp_path / "short.fq"))
    rng = synth.SplitMix64(0xBA)                                  # error-free reads at 1x over each base: no valley
    g = synth.make_genome(rng, 5_000, repeats=False).tobytes().decode()
    synth.write_reads([(f"r{i}", g[i:i + 1000].encode(), b"I" * 1000) for i in range(0, 4_000, 1000)], str(tmp_path / "flat.fq"))
    err(-6, lambda m: m.startswith("no k-mer depth peak") and "--min_count" in m, reads=str(tmp_path / "flat.fq"))
    open(tmp_path / "file", "w").close()
    err(-6, f"{tmp_path / 'file'} exists but is not a directory", out=str(tmp_path / "file"), min_count=1)
    err(-6, lambda m: m.startswith(f"failed to create directory {tmp_path / 'file' / 'sub'}"), out=str(tmp_path / "file" / "sub"), min_count=1)
    os.environ["AC_POLISH_TABLE_SLOTS"] = "100"                   # 2 x 60 windows and more do not fit 100 slots
    try:
        err(-4, lambda m: "does not fit" in m, min_count=1)
    finally:
        del os.environ["AC_POLISH_TABLE_SLOTS"]
    assert os.listdir(out) == []


def test_one_locus_candidates_do_not_fit(emu, tmp_path, monkeypatch):
    """A 2 kbp piece of the parity case's chromosome with one substitution: a budget of 10,000 slots holds its window table and two loci's
    candidates at k = 21, L = 3 (2 x 2,118 slots each), but not one locus's at k = 31, L = 4 (2 x 12,009)."""
    reads, _ = parity_case(tmp_path, length=8_000)
    chrom = synth.make_genome(synth.SplitMix64(0xC1), 8_000, repeats=False).tobytes().decode()[1_000:3_000]
    asm = str(tmp_path / "piece.fasta")
    write_fasta(asm, [("piece", chrom[:1_000] + "ACGT"[("ACGT".index(chrom[1_000]) + 1) % 4] + chrom[1_001:])])
    monkeypatch.setenv("AC_POLISH_TABLE_SLOTS", "10000")
    info = api.polish(reads, asm, str(tmp_path / "ok"), k=21, lib=emu)
    assert info["edits"] == 1
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.polish(reads, asm, str(tmp_path / "big"), k=31, max_indel=4, lib=emu)
    assert e.value.code == -4 and "one locus's candidate table" in e.value.message


def test_unwritable_out_dir(emu, tmp_path):
    reads, asm = parity_case(tmp_path, length=8_000)
    out = tmp_path / "ro"
    out.mkdir()
    os.chmod(out, 0o500)
    try:
        if os.access(out, os.W_OK):
            pytest.skip("the directory stays writable (running as root)")
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.polish(reads, asm, str(out), k=21, lib=emu)
        assert e.value.code == -5 and e.value.message == f"cannot write {out}/polished.fasta"
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
    reads, asm = parity_case(tmp_path, length=8_000)
    out = tmp_path / "cli"
    r = run(emu_cli, "polish", "-r", reads, "-i", asm, "-o", out, "--kmer", "15")
    assert r.returncode == 0, r.stderr
    assert r.stdout == open(out / "summary.tsv").read()
    want = O.run(reads, asm, 15)
    assert out_files(out) == want["files"]
    assert "Starting autocycler polish" in r.stderr and "not in the reference" in r.stderr and f"valley: {want['valley']}" in r.stderr
    assert "  round 1: " in r.stderr and r.stderr.rstrip().endswith("polished.fasta")
    r = run(emu_cli, "polish", "--reads", reads, "--input", asm, "--out_dir", out, "--kmer", "15", "--min_count", "3", "--max_indel", "1",
            "--rounds", "1")
    assert r.returncode == 0 and r.stdout == O.run(reads, asm, 15, 3, 1, 1)["files"]["summary.tsv"].decode()
    assert "min_count: 3 (given)" in r.stderr and "--max_indel 1" in r.stderr and "--rounds 1" in r.stderr
    usage = "Usage: autocycler polish"
    for args in (["polish"], ["polish", "-r", reads], ["polish", "-r", reads, "-i", asm], ["polish", "-i", asm, "-o", out]):
        r = run(emu_cli, *args)
        assert r.returncode == 2 and r.stderr.startswith(usage) and r.stdout == "", args
    r = run(emu_cli, "polish", "-h")
    assert r.returncode == 0 and r.stderr.startswith(usage) and "not in the reference" in r.stderr
    for flag, value in (("--kmer", "x"), ("--kmer", "9"), ("--kmer", "22"), ("--kmer", "33"), ("--min_count", "0"), ("--min_count", "16384"),
                        ("--min_count", "2.5"), ("--max_indel", "0"), ("--max_indel", "5"), ("--max_indel", "-1"), ("--rounds", "0"),
                        ("--rounds", "11"), ("--rounds", "x")):
        r = run(emu_cli, "polish", "-r", reads, "-i", asm, "-o", out, flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'") and usage in r.stderr, (flag, value)
    r = run(emu_cli, "polish", "-r", reads, "-i", asm, "-o", out, "--bogus", "1")
    assert r.returncode == 2 and r.stderr.startswith("error: unexpected argument '--bogus'")
    r = run(emu_cli, "polish", "-r", tmp_path / "nope.fq", "-i", asm, "-o", out)
    assert r.returncode == 1 and r.stderr.endswith(f"Error: file does not exist: {tmp_path / 'nope.fq'}\n") and r.stdout == ""
    write_fasta(str(tmp_path / "short.fasta"), [("s", "ACGTACGT")])
    r = run(emu_cli, "polish", "-r", reads, "-i", tmp_path / "short.fasta", "-o", out)
    assert r.returncode == 1 and r.stderr.endswith("holds 21 consecutive A, C, G or T bases\n")


# ---- the GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_gpu_oracle_parity(gpu, k, tmp_path):
    reads, asm = parity_case(tmp_path)
    check(gpu, reads, asm, k, tmp_path / "out")


@pytest.mark.gpu
def test_gpu_partitions_windows_and_tight_tables(gpu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path)
    base_info, _ = check(gpu, reads, asm, 21, tmp_path / "base")
    base = out_files(tmp_path / "base")
    tight = str(base_info["table_bytes"] // 16)
    for i, env in enumerate([{"AC_GS_PARTITIONS": "4"}, {"AC_SUBSAMPLE_WINDOW": "50000"}, {"AC_POLISH_TABLE_SLOTS": tight}]):
        for name, value in env.items():
            monkeypatch.setenv(name, value)
        info = api.polish(reads, asm, str(tmp_path / f"o{i}"), k=21, lib=gpu)
        for name in env:
            monkeypatch.delenv(name)
        assert out_files(tmp_path / f"o{i}") == base, env
        if "AC_GS_PARTITIONS" in env:
            assert info["partitions"] == 4
        if "AC_POLISH_TABLE_SLOTS" in env:
            assert info["batches"] > base_info["batches"]


@pytest.mark.gpu
def test_gpu_planted_errors_1mbp(gpu, tmp_path):
    check_meaning(gpu, tmp_path, length=1_000_000, step=5_000)
