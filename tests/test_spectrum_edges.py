"""The read-spectrum commands at the counts and warp shapes their other tests never reach: k-mers counted exactly 255, 256, 16,382,
16,383, 65,535, 65,536, 2^24 - 1, 2^24 and more, so that depth's radix-select median takes its upper digits and the histograms their top
bin; short reads by the thousand, so that many reads share one warp's packed words in unassembled's per-read adds; thousands of contigs
in depth's per-contig adds; spectrum tables whose last warp and CTA are partial; and polish candidates that tie within and across the
lanes of the choice's warp, at every largest indel.  Every case runs on the host-emulation build (which checks the generators, the
oracles and the shared bodies) and, marked gpu, on the CUDA build; each compares every output with its command's oracle and asserts
the shape it claims (the generators are in tests/spectrum_edges.py)."""
import os
import shutil
import subprocess

import pytest

import depth_oracle as DO
import genome_size_oracle as GO
import polish_oracle as PO
import qv_oracle as QO
import spectrum_edges as S
import unassembled_oracle as UO
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
H = GO.H
TOP = H - 1


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
def lib(request):
    return request.getfixturevalue(request.param)


def out_files(out_dir):
    files = {}
    for dirpath, _, names in os.walk(out_dir):
        for n in names:
            p = os.path.join(dirpath, n)
            files[os.path.relpath(p, out_dir)] = open(p, "rb").read()
    return files


def same_files(out_dir, want):
    got = out_files(out_dir)
    assert sorted(got) == sorted(want)
    for name, data in want.items():
        assert got[name] == data, name


def with_env(monkeypatch, env):
    for name in ("AC_GS_PARTITIONS", "AC_GS_TABLE_SLOTS", "AC_SUBSAMPLE_WINDOW"):
        monkeypatch.delenv(name, raising=False)
    for name, value in env.items():
        monkeypatch.setenv(name, value)


# ---- A. exact high counts --------------------------------------------------------------------------------------------------------------
K_HIGH = 15


@pytest.fixture(scope="session")
def high(tmp_path_factory):
    """The high-count reads (keys at 255/256, 16,382/16,383, 65,535/65,536, 20,000 and 30,000) and the oracle's histogram."""
    d = tmp_path_factory.mktemp("high")
    g, reads, cnt, units = S.high_counts(K_HIGH)
    path = str(d / "reads.fq")
    synth.write_reads(reads, path)
    hist, W = GO.histogram(path, K_HIGH)
    yield {"dir": d, "genome": g, "reads": path, "claim": cnt.histogram_claim(), "units": units, "hist": hist, "W": W}
    shutil.rmtree(d, ignore_errors=True)


def test_high_counts_claim(high):
    """The planted keys alone fill bins 255, 256, 16,382 and the top bin, and the oracle's histogram holds exactly them there."""
    claim, hist = high["claim"], high["hist"]
    assert claim == {255: 8, 256: 8, 16_382: 8, TOP: 27}
    for c in (255, 256, 16_382, TOP):
        assert hist[c] == claim[c], c
    assert sum(hist[100:]) == sum(claim.values())                   # no background key comes near them
    GO.estimate(hist, high["W"])                                     # the valley and the peak still hold


GS_SETTINGS = {
    "default": {},
    "p1": {"AC_GS_PARTITIONS": "1"},
    "p2": {"AC_GS_PARTITIONS": "2"},
    "p4": {"AC_GS_PARTITIONS": "4"},
    "rerun": {"AC_GS_PARTITIONS": "2", "AC_GS_TABLE_SLOTS": "40001"},      # tables of 40,001 x 2^n slots: partial last warp and CTA
}


@pytest.mark.parametrize("setting", sorted(GS_SETTINGS))
@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_genome_size_top_bins(lib, high, setting, monkeypatch):
    with_env(monkeypatch, GS_SETTINGS[setting])
    info = api.genome_size_estimate(high["reads"], K_HIGH, lib=lib)
    assert info["windows"] == high["W"] and info["histogram"] == high["hist"]
    want = GO.estimate(high["hist"], high["W"])
    for f in ("estimate", "valley", "peak", "peak_refined", "solid", "distinct"):
        assert info[f] == want[f], f
    for c, n in high["claim"].items():
        assert info["histogram"][c] == n, c
    if "AC_GS_PARTITIONS" in GS_SETTINGS[setting]:
        assert info["partitions"] == int(GS_SETTINGS[setting]["AC_GS_PARTITIONS"])
    if setting == "rerun":
        assert info["reruns"] > 0


def qv_assembly(high):
    """The background genome, a tandem array of U2 (5 copies of each rotation), a homopolymer (6 copies of A^k) and a dinucleotide
    (5 copies of each of its keys)."""
    k, u2 = K_HIGH, high["units"][1]
    path = str(high["dir"] / "qv_asm.fasta")
    S.write_fasta(path, [("bg circular=true", high["genome"]), ("tandem", (u2 * 8)[:5 * 16 + k - 1]), ("homo", "A" * (k + 5)),
                         ("di", ("AC" * k)[:k + 9])])
    return path


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_qv_top_bin(lib, high, tmp_path):
    asm = qv_assembly(high)
    info = api.qv(high["reads"], [asm], str(tmp_path / "out"), k=K_HIGH, lib=lib)
    want = QO.run(high["reads"], [asm], K_HIGH)
    same_files(tmp_path / "out", want["files"])
    assert info["min_count"] == want["t"] and info["solid_kmers"] == want["S"]
    rows = {}
    for line in want["files"]["spectra_cn/1.tsv"].decode().splitlines()[1:]:
        c, *x = map(int, line.split("\t"))
        rows[c] = x
    # the top bin: U3's 8 keys at 16,383 not in the assembly; U2's 16, A^k and the dinucleotide's 2 in it at 4+ copies
    assert rows[TOP] == [8, 0, 0, 0, 19] and rows[16_382] == [8, 0, 0, 0, 0]
    assert rows[255] == [8, 0, 0, 0, 0] and rows[256] == [8, 0, 0, 0, 0]


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_unassembled_absent_top_bin(lib, high, tmp_path):
    asm = str(high["dir"] / "ua_asm.fasta")
    S.write_fasta(asm, [("bg circular=true", high["genome"])])
    info = api.unassembled(high["reads"], [asm], str(tmp_path / "out"), k=K_HIGH, lib=lib)
    want = UO.run(high["reads"], [asm], K_HIGH)
    same_files(tmp_path / "out", want["files"])
    # the absent solid keys are the planted ones: bins 255, 256, 16,382 and the top bin; their median is the top bin
    absent = dict(tuple(map(int, line.split("\t"))) for line in want["files"]["absent_histogram.tsv"].decode().splitlines())
    assert absent == high["claim"]
    assert want["absent_median"] == float(TOP) and info["absent_median"] == float(TOP)
    assert want["ratio"] == TOP / want["peak"] and f"{info['absent_copy_ratio']:.2f}" == f"{want['ratio']:.2f}"


@pytest.fixture(scope="session")
def digits(tmp_path_factory):
    d = tmp_path_factory.mktemp("digits")
    contigs, reads, medians = S.depth_digits()
    asm, path = str(d / "asm.fasta"), str(d / "reads.fq")
    S.write_fasta(asm, contigs)
    synth.write_reads(reads, path)
    del reads
    yield asm, path, medians, DO.run(asm, path, 11)
    shutil.rmtree(d, ignore_errors=True)                               # 100 MB of reads


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_depth_digit_boundaries(lib, digits, tmp_path):
    """Medians of 255.5, 65,535.5 and 16,777,215.5 (middle counts on either side of a digit boundary) and 70,000 from counts that use
    all four digits: every pass of the radix select decides one of them."""
    asm, reads, medians, want = digits
    tsv = str(tmp_path / "out.tsv")
    info = api.depth(asm, str(tmp_path / "out.fasta"), reads=reads, k=11, tsv=tsv, lib=lib)
    assert info["depths"] == want["depths"] and info["unique"] == want["unique"]
    assert open(tsv).read() == want["tsv"] and open(tmp_path / "out.fasta", "rb").read() == want["fasta"]
    assert info["unique"][1:] == [16, 16, 2, 11]
    assert dict(zip(["d8", "d16", "d24", "dall"], info["depths"][1:])) == medians
    assert 20 <= info["depths"][0] <= 40


# ---- B. many addresses per warp ---------------------------------------------------------------------------------------------------------
K_SHORT = 17


@pytest.fixture(scope="session")
def short(tmp_path_factory):
    d = tmp_path_factory.mktemp("short")
    g, held, reads, names = S.short_reads(K_SHORT)
    asm, path = str(d / "asm.fasta"), str(d / "reads.fq")
    S.write_fasta(asm, [("held", held)])
    synth.write_reads(reads, path)
    kw = dict(min_solid=1, min_fraction=5e-324)
    yield asm, path, names, kw, UO.run(path, [asm], K_SHORT, **kw)
    shutil.rmtree(d, ignore_errors=True)


UA_SETTINGS = {
    "default": {},
    "p2": {"AC_GS_PARTITIONS": "2"},
    "p4": {"AC_GS_PARTITIONS": "4"},
    "windows_p2": {"AC_SUBSAMPLE_WINDOW": "20000", "AC_GS_PARTITIONS": "2"},
    "odd_slots": {"AC_GS_PARTITIONS": "4", "AC_GS_TABLE_SLOTS": "100003"},     # not a multiple of 32 or 1024
}


@pytest.mark.parametrize("setting", sorted(UA_SETTINGS))
@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_unassembled_short_reads(lib, short, setting, tmp_path, monkeypatch):
    """Every read with an absent solid window is listed with its exact solid and absent counts; thousands of them are shorter than one
    warp's 32 packed words, so many reads share a warp's adds."""
    asm, reads, names, kw, want = short
    with_env(monkeypatch, UA_SETTINGS[setting])
    info = api.unassembled(reads, [asm], str(tmp_path / "out"), k=K_SHORT, lib=lib, **kw)
    same_files(tmp_path / "out", want["files"])
    assert info["selected_reads"] == len(want["selected"])
    listed = [r for r in info["selected"] if r["read"] in names]
    assert sum(1 for r in listed if r["length"] // 32 + 1 < 32) >= 3000
    if setting == "windows_p2":
        assert info["read_passes"] > 1
    if "AC_GS_PARTITIONS" in UA_SETTINGS[setting]:
        assert info["partitions"] == int(UA_SETTINGS[setting]["AC_GS_PARTITIONS"])


@pytest.fixture(scope="session")
def contigs(tmp_path_factory):
    d = tmp_path_factory.mktemp("contigs")
    ctgs, reads = S.many_contigs(21)
    asm, path = str(d / "asm.fasta"), str(d / "reads.fq")
    S.write_fasta(asm, ctgs)
    synth.write_reads(reads, path)
    yield asm, path, DO.run(asm, path, 21)
    shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_depth_many_contigs(lib, contigs, tmp_path):
    asm, reads, want = contigs
    tsv = str(tmp_path / "out.tsv")
    info = api.depth(asm, str(tmp_path / "out.fasta"), reads=reads, k=21, tsv=tsv, lib=lib)
    assert info["depths"] == want["depths"] and info["unique"] == want["unique"]
    assert open(tsv).read() == want["tsv"]
    assert info["contigs"] == 3001 and sum(1 for u in info["unique"] if u) == 3001 and info["unique"][0] >= 199_000


# ---- C. polish ties at every warp layout -----------------------------------------------------------------------------------------------
# (L, name, candidates the repeat copies carry, the copy read twice as deep or None).  Candidates per L: 8, 25, 90 and 347, so a warp's
# lane holds candidates c, c + 32, ... from L = 3 on.
# A unique best comes with a weaker candidate that passes too: in the same lane (late_best, the best at c >= 32, at L = 4 c >= 256) or
# in another lane (best_other_lane), whose count must not join the best's.
TIES = [
    (1, "lanes", (1, 2), None), (1, "three", (0, 3, 5), None), (1, "best_other_lane", (1, 5), 1),
    (2, "lanes", (0, 10), None), (2, "three", (2, 3, 20), None), (2, "best_other_lane", (0, 20), 1),
    (3, "lanes", (1, 2), None), (3, "one_lane", (3, 35), None), (3, "three_two_lanes", (4, 36, 10), None), (3, "late_best", (8, 40), 1),
    (3, "best_other_lane", (9, 40), 1),
    (4, "lanes", (0, 2), None), (4, "one_lane", (5, 37), None), (4, "three_two_lanes", (6, 38, 7), None), (4, "late_best", (12, 300), 1),
    (4, "best_other_lane", (20, 300), 1),
]


def _tie_case(index, d):
    L, _, alleles, deep = TIES[index]
    asm_seq, reads, p0, cands = S.tie_case(L, alleles, seed=0x5E10 + index, deep=deep)
    asm, path = str(d / f"asm{index}.fasta"), str(d / f"reads{index}.fq")
    S.write_fasta(asm, [("genome circular=true", asm_seq)])
    synth.write_reads(reads, path)
    return L, alleles, deep, asm, path, p0, cands


@pytest.mark.parametrize("index", range(len(TIES)), ids=[f"L{t[0]}_{t[1]}" for t in TIES])
def test_tie_cases_claim(index, tmp_path):
    """The oracle's view of each case: one locus at the repeat's base 100, its best candidates exactly the planted ones (all of them on
    a tie, the deep copy's alone otherwise), their lanes as named."""
    L, alleles, deep, asm, reads, p0, cands = _tie_case(index, tmp_path)
    assert len(cands) == api_candidates(L)
    uk, uc, _ = QO.read_counts(reads, 21)
    seq = DO.load_fasta(asm)[0][2]
    best, count, first, _ = PO.choose([(0, p0 - 20)], [(seq, True)], 21, L, 2, PO.Counts(uk, uc))[0]
    if deep is None:
        assert (best, count, first) == (100, len(alleles), min(alleles))
    else:
        assert (best, count, first) == (200, 1, alleles[deep])
    lanes = {c % 32 for c in alleles}
    name = TIES[index][1]
    assert len(lanes) == {"lanes": len(alleles), "three": 3, "one_lane": 1, "three_two_lanes": 2, "late_best": 1, "best_other_lane": 2}[name]
    if name == "late_best":
        assert alleles[deep] >= (256 if L == 4 else 32)


def api_candidates(L):
    return 3 + L + sum(4 ** s for s in range(1, L + 1))


@pytest.mark.parametrize("index", range(len(TIES)), ids=[f"L{t[0]}_{t[1]}" for t in TIES])
@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_polish_ties(lib, index, tmp_path):
    L, alleles, deep, asm, reads, p0, cands = _tie_case(index, tmp_path)
    info = api.polish(reads, asm, str(tmp_path / "out"), k=21, min_count=2, max_indel=L, lib=lib)
    want = PO.run(reads, asm, 21, min_count=2, max_indel=L)
    same_files(tmp_path / "out", want["files"])
    first = want["rounds"][0]
    assert first["loci"] == 1
    if deep is None:
        assert (first["ambiguous"], first["edited"]) == (1, 0) and info["edits"] == 0
    else:
        mid, skip = cands[alleles[deep]]
        seq = DO.load_fasta(asm)[0][2]
        assert (first["ambiguous"], first["edited"]) == (0, 1)
        assert [(e["round"], e["position"], e["ref"], e["alt"], e["score"]) for e in info["applied"]] == \
            [(1, p0, seq[p0:p0 + skip] if skip else "-", mid or "-", 200)]
