"""`autocycler qv`: each assembly's k-mer QV and completeness against the reads, counted on the GPU (DESIGN.md §20).  `qv` is not in the
reference, so it is pinned against the numpy oracle of the rule (tests/qv_oracle.py) and, on synthetic assemblies with errors planted at
known positions, by what the rule means.  The CPU tests run the product's code through the host-emulation library (the kernels' bodies,
serially); the tests marked gpu run the CUDA build on the H100."""
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import qv_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
H = api.GENOME_SIZE_BINS


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


def check(lib, reads, assemblies, k, out_dir, min_count=None):
    """Every file the product writes against the oracle's (and no other file); returns (info, oracle result)."""
    info = api.qv(reads, assemblies, str(out_dir), k=k, min_count=min_count, lib=lib)
    want = O.run(reads, assemblies, k, min_count)
    got = out_files(out_dir)
    assert sorted(got) == sorted(want["files"])
    for name, data in want["files"].items():
        assert got[name] == data, name
    assert info["min_count"] == want["t"] and info["solid_kmers"] == want["S"] and info["read_windows"] == want["W"]
    assert info["valley"] == (want["valley"] or 0)
    return info, want


def parity_case(tmp_path):
    """Three assemblies, two of them in a directory: a true genome of a circular chromosome and a linear replicon, a copy with planted
    errors, a contig repeated 2, 3 and 5 times, circular, linear and too-short contigs, N/IUPAC and lowercase; reads in two gzip
    members, with N/IUPAC and lowercase too."""
    rng = synth.SplitMix64(0xA1)
    chrom, lin, rep = (synth.make_genome(rng, n).tobytes().decode() for n in (12_000, 3_000, 2_000))
    bad = list(chrom)
    for p in range(300, 12_000, 1_700):
        bad[p] = "ACGT"[("ACGT".index(bad[p]) + 1) % 4]
    bad = "".join(bad)
    d = tmp_path / "asm"
    d.mkdir()
    write_fasta(d / "a_true.fasta", [("chrom circular=true", chrom), ("lin", lin)])
    write_fasta(d / "b_errors.fa", [("chrom Circular=TRUE", bad[:6000].lower() + "NNRYK" + bad[6005:]), ("lin", lin[:2500])])
    write_fasta(d / "notes.txt", [("x", "ACGT")])                        # not an assembly file: the directory skips it
    third = str(tmp_path / "repeats.fasta")
    write_fasta(third, [("r2a", rep[:700]), ("r2b circular=true", rep[:700]), ("r3", rep[800:1200] * 3), ("r5", (rep[1300:1600] + "N") * 5),
                        ("tiny circular=true", chrom[100:115]), ("lin_part", lin[500:1500])])
    reads = noisy(chrom + lin + rep, 25, 7, n50=2000)
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
    return path, [str(d), third]


def spectrum_rows(data):
    rows = {}
    for line in data.decode().splitlines()[1:]:
        c, *x = map(int, line.split("\t"))
        rows[c] = x
    return rows


# ---- the rule against the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [11, 15, 21, 31])
def test_oracle_parity(emu, k, tmp_path):
    reads, asm = parity_case(tmp_path)
    info, want = check(emu, reads, asm, k, tmp_path / "out")
    assert info["assemblies"][0]["path"].endswith("asm/a_true.fasta") and info["assemblies"][2]["path"] == asm[1]
    assert [a["kmers"] for a in info["assemblies"]] == [a["kmers"] for a in want["assemblies"]]
    # the repeats reach every copy-number column
    cn = want["assemblies"][2]["spectrum"]
    assert cn[:, 2].sum() and cn[:, 3].sum() and cn[:, 4].sum()
    # invariants: each spectra-cn row sums to genome_size's h[c], and kmer_histogram.tsv is genome_size -d's file
    gs_dir = tmp_path / "gs"
    gs = api.genome_size_estimate(reads, k, dir=str(gs_dir), lib=emu)
    assert open(gs_dir / "kmer_histogram.tsv", "rb").read() == open(tmp_path / "out" / "kmer_histogram.tsv", "rb").read()
    for n in (1, 2, 3):
        for c, row in spectrum_rows(open(tmp_path / "out" / "spectra_cn" / f"{n}.tsv", "rb").read()).items():
            assert min(row) >= 0
            if c:
                assert sum(row) == gs["histogram"][c]
            else:
                assert row[0] == 0


def test_same_outputs_across_windows_partitions_and_reruns(emu, tmp_path, monkeypatch):
    reads, asm = parity_case(tmp_path)
    api.qv(reads, asm, str(tmp_path / "base"), k=15, lib=emu)
    base = out_files(tmp_path / "base")
    settings = [{"AC_SUBSAMPLE_WINDOW": "1000"}, {"AC_SUBSAMPLE_WINDOW": "7777"}, {"AC_GS_PARTITIONS": "1"}, {"AC_GS_PARTITIONS": "2"},
                {"AC_GS_PARTITIONS": "4"}, {"AC_GS_PARTITIONS": "2", "AC_GS_TABLE_SLOTS": "5000"}]    # the last: tables too small, rerun
    for i, env in enumerate(settings):
        for name, value in env.items():
            monkeypatch.setenv(name, value)
        info = api.qv(reads, asm, str(tmp_path / f"o{i}"), k=15, lib=emu)
        for name in env:
            monkeypatch.delenv(name)
        assert out_files(tmp_path / f"o{i}") == base, env
        if "AC_GS_PARTITIONS" in env:
            assert info["partitions"] == int(env["AC_GS_PARTITIONS"])
        assert (info["reruns"] > 0) == ("AC_GS_TABLE_SLOTS" in env)


# ---- what the rule means: errors planted at known positions -------------------------------------------------------------------------
def planted_case(tmp_path):
    """A 40 kbp circular chromosome and a 6 kbp linear plasmid (no repeats), reads at 40x with 1% errors, and five assemblies: the truth,
    4 substitutions more than 2k apart, also across the junction (the last one's windows wrap), 12 substitutions, the truth without a
    4 kbp stretch, and 3 substitutions on the linear plasmid, two of them near its ends (clipped)."""
    rng = synth.SplitMix64(0xA7)
    chrom = synth.make_genome(rng, 40_000, repeats=False).tobytes().decode()
    plas = synth.make_genome(rng, 6_000, repeats=False).tobytes().decode()

    def sub(seq, positions):
        s = list(seq)
        for p in positions:
            s[p] = "ACGT"[("ACGT".index(s[p]) + 2) % 4]
        return "".join(s)

    few = [30, 10_000, 25_000, 39_985]
    many = list(range(1_000, 37_000, 3_000))
    plas_subs = [3, 3_000, 5_990]
    files = {
        "truth": [("chrom circular=true", chrom), ("plasmid", plas)],
        "few": [("chrom circular=true", sub(chrom, few)), ("plasmid", plas)],
        "many": [("chrom circular=true", sub(chrom, many)), ("plasmid", plas)],
        "gap": [("chrom circular=true", chrom[:20_000] + chrom[24_000:]), ("plasmid", plas)],
        "linear": [("chrom circular=true", chrom), ("plasmid", sub(plas, plas_subs))],
    }
    paths = []
    for name, recs in files.items():
        paths.append(str(tmp_path / f"{name}.fasta"))
        write_fasta(paths[-1], recs)
    reads = str(tmp_path / "reads.fq")
    synth.write_reads(noisy(chrom, 40, 21, n50=4000) + noisy(plas, 40, 22, n50=2000), reads)
    return reads, paths, few, many, plas_subs


def test_planted_errors(emu, tmp_path):
    k = 21
    reads, paths, few, many, plas_subs = planted_case(tmp_path)
    info, want = check(emu, reads, paths, k, tmp_path / "out")
    truth, a_few, a_many, gap, linear = info["assemblies"]
    L = 40_000
    # the truth: every window supported
    assert truth["unsupported"] == 0 and truth["qv"] == float("inf")
    assert open(tmp_path / "out" / "unsupported" / "1.bed").read() == ""
    # s substitutions more than 2k apart: exactly k s unsupported windows, and s intervals [p-k+1, p+k) wrapped at the junction
    assert a_few["unsupported"] == k * len(few) and a_many["unsupported"] == k * len(many)
    p0, p1, p2, p3 = few                                                 # p3's interval wraps: [p3-k+1, L) and [0, p3+k-L)
    assert open(tmp_path / "out" / "unsupported" / "2.bed").read().splitlines() == [
        f"chrom\t0\t{p3 + k - L}", f"chrom\t{p0 - k + 1}\t{p0 + k}", f"chrom\t{p1 - k + 1}\t{p1 + k}", f"chrom\t{p2 - k + 1}\t{p2 + k}",
        f"chrom\t{p3 - k + 1}\t{L}"]
    many_bed = open(tmp_path / "out" / "unsupported" / "3.bed").read().splitlines()
    assert many_bed == [f"chrom\t{p - k + 1}\t{p + k}" for p in many]
    # the linear plasmid: substitutions near its ends are clipped, with fewer windows
    plas_len = 6_000
    assert linear["unsupported"] == sum(min(p, plas_len - k) - max(0, p - k + 1) + 1 for p in plas_subs)
    assert open(tmp_path / "out" / "unsupported" / "5.bed").read().splitlines() == [
        f"plasmid\t{max(0, p - k + 1)}\t{min(plas_len, p + k)}" for p in plas_subs]
    # a missing stretch: fewer solid read k-mers found; the truth finds them all
    # a missing stretch: fewer solid read k-mers found.  The reads come from a circular plasmid, so the truth, whose plasmid is linear,
    # misses only the k-1 solid keys across its junction
    assert truth["solid_found"] == info["solid_kmers"] - (k - 1)
    assert gap["solid_found"] < a_few["solid_found"] < truth["solid_found"] and gap["completeness"] < 92.0
    # the rows rank as planted: 0 errors, one deletion, 3 substitutions (clipped), 4 substitutions, 12 substitutions
    assert truth["qv"] > gap["qv"] > linear["qv"] > a_few["qv"] > a_many["qv"]
    # contig rows: only the chromosome of `few` and the plasmid of `linear` carry errors
    rows = {(c["assembly"], c["contig"]): c for c in info["contigs"]}
    assert rows[(paths[1], "chrom")]["unsupported"] == k * len(few) and rows[(paths[1], "plasmid")]["qv"] == float("inf")
    assert rows[(paths[4], "chrom")]["unsupported"] == 0
    # seeded, so pinned exactly
    assert [(a["unsupported"], a["qv"], a["solid_found"], a["completeness"]) for a in info["assemblies"]] == [
        (0, float("inf"), 45980, 99.96), (84, 40.6, 45896, 99.77), (252, 35.82, 45728, 99.41), (19, 46.66, 41961, 91.22),
        (35, 44.41, 45945, 99.88)]
    assert (info["valley"], info["min_count"], info["solid_kmers"]) == (13, 13, 46000)




def test_min_count(emu, tmp_path):
    """--min_count overrides the valley; t = 1 is Merqury's QV.  Reads with no valley fail without it and succeed with it."""
    reads, paths, *_ = planted_case(tmp_path)
    info, want = check(emu, reads, paths[:2], 21, tmp_path / "o1", min_count=1)
    assert info["min_count"] == 1 and info["valley"] == want["valley"] != 1
    check(emu, reads, paths[:2], 21, tmp_path / "o2", min_count=3)
    # error-free reads at 1x over each base, so every k-mer is seen about once: no valley
    rng = synth.SplitMix64(0xA9)
    g = synth.make_genome(rng, 5_000, repeats=False).tobytes().decode()
    flat = str(tmp_path / "flat.fq")
    synth.write_reads([(f"r{i}", g[i:i + 1000].encode(), b"I" * 1000) for i in range(0, 4_000, 1000)], flat)
    asm = str(tmp_path / "g.fasta")
    write_fasta(asm, [("g", g)])
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.qv(flat, [asm], str(tmp_path / "o3"), k=21, lib=emu)
    assert e.value.code == -6 and e.value.message.startswith("no k-mer depth peak") and "--min_count" in e.value.message
    assert os.listdir(tmp_path / "o3") == []                             # created before the run, so a bad path fails fast
    info, _ = check(emu, flat, [asm], 21, tmp_path / "o4", min_count=1)
    assert info["valley"] == 0 and info["assemblies"][0]["unsupported"] == 1060     # the windows no read holds whole


# ---- errors -------------------------------------------------------------------------------------------------------------------------
def test_errors(emu, tmp_path):
    asm, reads = str(tmp_path / "a.fasta"), str(tmp_path / "r.fq")
    write_fasta(asm, [("a", "ACGT" * 20)])
    synth.write_reads([("r", b"ACGT" * 20, b"I" * 80)], reads)
    out = str(tmp_path / "o")

    def err(code, message, assemblies=(asm,), reads=reads, out=out, **kw):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.qv(reads, list(assemblies), out, lib=emu, **kw)
        assert e.value.code == code and (e.value.message == message if isinstance(message, str) else message(e.value.message)), e.value.message

    for k in (9, 10, 12, 22, 33, 0):
        err(-6, "--kmer must be odd and between 11 and 31", k=k)
    for t in (0, H):
        err(-6, f"--min_count must be between 1 and {H - 1}", min_count=t)
    err(-6, f"file does not exist: {tmp_path / 'nope.fq'}", reads=str(tmp_path / "nope.fq"))
    err(-6, f"file does not exist: {tmp_path / 'nope.fasta'}", assemblies=[asm, str(tmp_path / "nope.fasta")])
    (tmp_path / "empty_dir").mkdir()
    err(-6, f"no assemblies found in {tmp_path / 'empty_dir'}", assemblies=[str(tmp_path / "empty_dir")])
    write_fasta(str(tmp_path / "short.fasta"), [("s", "ACGTNACGTACGTACGTACG"), ("t", "ACG")])
    err(-6, f"{tmp_path / 'short.fasta'}: no k-mer windows: no contig holds 21 consecutive A, C, G or T bases",
        assemblies=[asm, str(tmp_path / "short.fasta")])
    open(tmp_path / "empty.fasta", "w").close()
    err(-6, f"{tmp_path / 'empty.fasta'} is an empty file", assemblies=[str(tmp_path / "empty.fasta")])
    synth.write_reads([("r", b"ACGTN" * 20, b"I" * 100)], str(tmp_path / "short.fq"))
    err(-6, "no k-mer windows: no read holds 21 consecutive A, C, G or T bases", reads=str(tmp_path / "short.fq"))
    for data, rec, why in ((b"@a\nAC\n+\nII\nb\nAC\n+\nII\n", 2, "expected '@' at the start of the header line"),
                           (b"@a\nAC\n+\nII\n@b\nAC", 2, "truncated record")):
        open(tmp_path / "bad.fq", "wb").write(data)
        err(-6, f"Error reading FASTQ file: record {rec}: {why}", reads=str(tmp_path / "bad.fq"))
    open(tmp_path / "file", "w").close()
    err(-6, f"{tmp_path / 'file'} exists but is not a directory", out=str(tmp_path / "file"), min_count=1)
    err(-6, lambda m: m.startswith(f"failed to create directory {tmp_path / 'file' / 'sub'}"), out=str(tmp_path / "file" / "sub"), min_count=1)
    os.environ["AC_QV_TABLE_SLOTS"] = "200"                       # 2 x 60 windows + 2 x 60 do not fit 200 slots
    try:
        err(-4, lambda m: "do not fit" in m, min_count=1)
    finally:
        del os.environ["AC_QV_TABLE_SLOTS"]
    assert os.listdir(out) == []


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
    r = run(emu_cli, "qv", "-r", reads, "-i", *asm, "-o", out, "--kmer", "15")
    assert r.returncode == 0, r.stderr
    assert r.stdout == open(out / "qv.tsv").read()
    want = O.run(reads, asm, 15)
    assert out_files(out) == want["files"]
    assert "Starting autocycler qv" in r.stderr and "not in the reference" in r.stderr and f"valley: {want['valley']}" in r.stderr
    r = run(emu_cli, "qv", "--reads", reads, "--assemblies", asm[1], "--out_dir", out, "--kmer", "15", "--min_count", "2")
    assert r.returncode == 0 and r.stdout.splitlines()[1].endswith("\t2") and "min_count: 2 (given)" in r.stderr
    usage = "Usage: autocycler qv"
    for args in (["qv"], ["qv", "-r", reads], ["qv", "-r", reads, "-i", asm[1]], ["qv", "-i", asm[1], "-o", out]):
        r = run(emu_cli, *args)
        assert r.returncode == 2 and r.stderr.startswith(usage) and r.stdout == "", args
    r = run(emu_cli, "qv", "-h")
    assert r.returncode == 0 and r.stderr.startswith(usage) and "not in the reference" in r.stderr
    for flag, value in (("--kmer", "x"), ("--min_count", "-1"), ("--min_count", "2.5")):
        r = run(emu_cli, "qv", "-r", reads, "-i", asm[1], "-o", out, flag, value)
        assert r.returncode == 2 and r.stderr.startswith(f"error: invalid value '{value}' for '{flag}'"), (flag, value)
    r = run(emu_cli, "qv", "-r", reads, "-i", asm[1], "-o", out, "--bogus", "1")
    assert r.returncode == 2 and r.stderr.startswith("error: unexpected argument '--bogus'")
    r = run(emu_cli, "qv", "-r", tmp_path / "nope.fq", "-i", asm[1], "-o", out)
    assert r.returncode == 1 and r.stderr.endswith(f"Error: file does not exist: {tmp_path / 'nope.fq'}\n") and r.stdout == ""
    r = run(emu_cli, "qv", "-r", reads, "-i", asm[1], "-o", out, "--min_count", "0")
    assert r.returncode == 1 and r.stderr.endswith(f"Error: --min_count must be between 1 and {H - 1}\n")


# ---- the GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [21, 31])
def test_gpu_oracle_parity(gpu, k, tmp_path):
    reads, asm = parity_case(tmp_path)
    check(gpu, reads, asm, k, tmp_path / "out")
    reads, paths, *_ = planted_case(tmp_path)
    check(gpu, reads, paths, k, tmp_path / "planted")


@pytest.mark.gpu
def test_gpu_read_longer_than_window_and_partitions(gpu, tmp_path, monkeypatch):
    big = synth.make_genome(synth.SplitMix64(0xAA), 300_000).tobytes().decode()
    asm = str(tmp_path / "asm.fasta")
    write_fasta(asm, [("big circular=true", big)])
    path = str(tmp_path / "r.fq")
    synth.write_reads([("long", big[:250_000].encode(), b"I" * 250_000)] + noisy(big, 20, 9, n50=5000), path)
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(100_000))
    check(gpu, path, [asm], 21, tmp_path / "o1")
    base = out_files(tmp_path / "o1")
    monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(1 << 20))
    monkeypatch.setenv("AC_GS_PARTITIONS", "4")
    info = api.qv(path, [asm], str(tmp_path / "o2"), k=21, lib=gpu)
    assert info["partitions"] == 4 and out_files(tmp_path / "o2") == base


@pytest.mark.gpu
def test_gpu_thirteen_assemblies(gpu, tmp_path):
    """13 assemblies of 1 Mbp: the truth and 12 copies with 0.01% to 0.12% substitutions, reads at 12x: the oracle's files, and QV
    falling as the planted rate rises."""
    rng = synth.SplitMix64(0xAB)
    g = synth.make_genome(rng, 1_000_000)
    d = tmp_path / "asm"
    d.mkdir()
    paths = []
    for i in range(13):
        a = g.copy()
        pos = np.array(rng.u64(100 * i), dtype=np.uint64) % np.uint64(len(a)) if i else np.zeros(0, dtype=np.uint64)
        a[pos.astype(np.int64)] = np.frombuffer(b"ACGT", dtype=np.uint8)[(np.searchsorted(np.frombuffer(b"ACGT", dtype=np.uint8),
                                                                                           a[pos.astype(np.int64)]) + 1) % 4]
        paths.append(str(d / f"{i:02d}.fasta"))
        write_fasta(paths[-1], [("chrom circular=true", a.tobytes().decode())])
    reads = str(tmp_path / "r.fq")
    synth.write_reads(noisy(g, 12, 31, n50=8000), reads)
    info, _ = check(gpu, reads, [str(d)], 21, tmp_path / "out")
    qv = [a["qv"] for a in info["assemblies"]]
    assert len(qv) == 13 and all(qv[i] > qv[i + 1] for i in range(1, 12))


def goldens():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "qv_goldens.json")))


@pytest.mark.gpu
def test_gpu_bench_input_against_golden(gpu, tmp_path, monkeypatch):
    """bench_qv.py's workload c (a chromosome and a 3-copy plasmid, and a variant) against the oracle's golden."""
    import bench_qv as B
    monkeypatch.chdir(tmp_path)                                          # the assembly paths are relative, as in the bench
    reads, asm = B.write_input("c", str(tmp_path))
    api.qv(reads, asm, str(tmp_path / "out"), k=B.K, lib=gpu)
    got = {n: hashlib.sha256(d).hexdigest() for n, d in out_files(tmp_path / "out").items()}
    assert got == goldens()["c"]["sha256"]
