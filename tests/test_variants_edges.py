"""`autocycler variants` (DESIGN.md §23) at the shapes its own tests never reach: exact AK, RK and PK from tiled reads for every kind
of event at max_indel 0 - 3, the PK rule's last window, the ref range's first window past it and its last window, substitutions at
every offset of a packed word and in many small contigs, the circular junction and the ends of linear contigs, multi-allelic sites,
counts past the histogram's top bin and 2^16, the min_fraction boundary, spectrum partitions, count reruns and candidate batches.
Every case runs on the host-emulation build and, marked gpu, on the CUDA build.  Each compares both files with the oracle
(tests/variants_oracle.py), asserts the exact rows the construction implies (tests/variants_edges.py), and asserts the shape it claims.
A count past 2^24 is left out: the tiled reads it takes would cost more time than the rest of this file."""
import math
import os
import shutil
import subprocess

import pytest

import variants_edges as V
import variants_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")


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


CASES = {
    "kinds_k21_L0": lambda: V.kinds(21, 0),
    "kinds_k21_L1": lambda: V.kinds(21, 1),
    "kinds_k21_L2": lambda: V.kinds(21, 2),
    "kinds_k21_L3": lambda: V.kinds(21, 3),
    "kinds_k11_L3": lambda: V.kinds(11, 3),
    "kinds_k31_L3": lambda: V.kinds(31, 3),
    "offsets_k21_L1": lambda: V.offsets(21, 1),
    "offsets_k31_L3": lambda: V.offsets(31, 3),
    "junction_k11": lambda: V.junction(11),
    "junction_k21": lambda: V.junction(21),
    "junction_k31": lambda: V.junction(31),
    "multi": V.multi,
    "high": V.high,
}


@pytest.fixture(scope="session")
def cases(tmp_path_factory):
    """Each case's FASTA and reads, written once on first use; the directory goes when the session ends."""
    d = tmp_path_factory.mktemp("variants_edges")
    made = {}

    def get(name):
        if name not in made:
            case = CASES[name]()
            case.asm, case.path = str(d / f"{name}.fasta"), str(d / f"{name}.fq")
            with open(case.asm, "w") as f:
                for _, header, seq, _ in case.contigs:
                    f.write(f">{header}\n{seq}\n")
            synth.write_reads(case.reads, case.path)
            case.reads = None
            made[name] = case
        return made[name]
    yield get
    shutil.rmtree(d, ignore_errors=True)


def out_files(out_dir):
    return {n: open(os.path.join(out_dir, n), "rb").read() for n in sorted(os.listdir(out_dir))}


def with_env(monkeypatch, env):
    for name in ("AC_GS_PARTITIONS", "AC_GS_TABLE_SLOTS", "AC_SUBSAMPLE_WINDOW", "AC_VARIANTS_TABLE_SLOTS"):
        monkeypatch.delenv(name, raising=False)
    for name, value in env.items():
        monkeypatch.setenv(name, value)


def check(lib, case, out_dir, min_fraction=None):
    """Both files against the oracle's, the counts against its, and the rows against the construction's; -> (info, rows)."""
    kw = dict(case.kw)
    if min_fraction is not None:
        kw["min_fraction"] = min_fraction
    info = api.variants(case.path, case.asm, str(out_dir), k=case.k, lib=lib, **kw)
    want = O.run(case.path, case.asm, case.k, **kw)
    got = out_files(out_dir)
    assert sorted(got) == sorted(want["files"])
    for name, data in want["files"].items():
        assert got[name] == data, name
    assert (info["positions"], info["screened"], info["candidates"], info["passing"], info["variants"]) == \
        (want["positions"], want["screened"], want["candidates"], want["passing"], len(want["rows"]))
    rows = [(r["contig"], r["pos"], r["ref"], r["alt"], r["ak"], r["rk"], r["pk"]) for r in info["rows"]]
    assert rows == case.rows(min_fraction), "the rows differ from the construction's"
    return info, rows


def measured(case):
    return [dict(ev, **case.measure(ev)) for ev in case.events]


def assert_shape(name, case, info):
    """What each case claims to reach, from its construction."""
    k = case.k
    ev = measured(case)
    if name.startswith("kinds"):
        m = case.R - k + 1
        by = {}
        for x in ev:
            by.setdefault(x["tag"], []).append(x)
        plain = by["plain"]
        assert all((x["ak"], x["rk"], x["pk"]) == (V.C2 * m, (V.C1 + V.C3) * m, 0) for x in plain)
        assert {(len(x["mid"]), x["skip"]) for x in plain} == \
            {(1, 1)} | {(0, d) for d in range(1, case.L + 1)} | {(d, 0) for d in range(1, case.L + 1)}
        # the held repeats: every checked window but the first few, the substitution's last one included, the deletion's left out
        assert by["held_sub"][0]["pk"] == 4 and by["held_sub"][0]["pk"] < len(by["held_sub"][0]["checked"])
        for x in by["ref_beyond"] + by.get("ref_beyond_del", []):
            # the truth window just past a .. p + d is read by fewer copies than every window in it
            after = case.count[V.canon((case.contigs[0][2] * 2)[x["p"] + x["skip"] * (x["mid"] == "") + 1:][:k])]
            assert x["rk"] == (V.C1 + V.C3) * m and after == (V.C1 + V.C2) * m < x["rk"]
        assert by["ref_last"][0]["rk"] == V.C1 * m
        if case.L:
            assert by["held_del"][0]["pk"] == 3 and by["hins"][0]["pk"] == 4 and by["hdel"][0]["pk"] == 4
            assert info["insertions"] == case.L + 1 and info["deletions"] == case.L + 3
        else:
            assert info["insertions"] == info["deletions"] == 0
    elif name.startswith("offsets"):
        words = [V.word_of(case, x) for x in ev if x["tag"] == "words"]
        assert sorted({o for _, o, _ in words}) == list(range(32))
        woff = V.layout(k, case.contigs)
        ci = [c[0] for c in case.contigs].index("words")
        assert max(w for w, _, _ in words) == woff[ci + 1] - 1 or max(w for w, _, _ in words) == woff[ci + 1] - 2
        assert any(V.word_of(case, x)[0] == 0 for x in ev if x["tag"] == "w0")
        names = {r["contig"] for r in info["rows"]}
        assert "tried" in names and "short" not in names and f"lin{k}" not in names and "lin65" in names
    elif name.startswith("junction"):
        names = {r["contig"] for r in info["rows"]}
        assert not names & set(case.shape["nothing"])
        assert all(V.word_of(case, x)[2] for x in ev if x["tag"] in ("sub0", "sub1", f"sub{k - 2}", "ins0", "del_cc"))
        assert not V.word_of(case, [x for x in ev if x["tag"] == f"sub{k - 1}"][0])[2]
        assert [r["pos"] for r in info["rows"] if r["contig"] == "homo"] == [1]
    elif name == "multi":
        sites = {}
        for r in info["rows"]:
            sites.setdefault(r["pos"], []).append(r)
        assert sum(len(s) == 3 for s in sites.values()) >= 6 and sum(len(s) == 2 for s in sites.values()) >= 6
        assert all(len({r["rk"] for r in s}) == 1 for s in sites.values())
        same_p = [x for x in ev if (len(x["mid"]), x["skip"]) == (1, 1)]
        assert any(a["p"] == b["p"] and a["c"] < b["c"] and a["ak"] > b["ak"] for a in same_p for b in same_p)
    elif name == "high":
        vcf = open(os.path.join(info["out"], "variants.vcf")).read()
        for (ak, rk) in case.shape["pairs"]:
            assert f"AF={ak / (ak + rk):.4f};AK={ak};RK={rk};PK=0" in vcf
        assert info["alt_major"] == 1


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_exact_rows(lib, cases, name, tmp_path, monkeypatch):
    with_env(monkeypatch, {})
    case = cases(name)
    info, rows = check(lib, case, tmp_path / "out")
    info["out"] = str(tmp_path / "out")
    assert rows
    assert_shape(name, case, info)


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_min_fraction_boundary(lib, cases, tmp_path, monkeypatch):
    """AF == F exactly (AK / (AK + RK) = 130 / 520 = 0.25) keeps the row; the next double above 0.25 drops it."""
    with_env(monkeypatch, {})
    case = cases("kinds_k21_L3")
    _, at = check(lib, case, tmp_path / "at", min_fraction=0.25)
    _, above = check(lib, case, tmp_path / "above", min_fraction=math.nextafter(0.25, 1.0))
    quarter = [r for r in at if r[4] * 4 == r[4] + r[5]]
    assert len(quarter) >= 9 and not set(quarter) & set(above) and set(above) == set(at) - set(quarter)


SWEEPS = {
    "p2": {"AC_GS_PARTITIONS": "2"},
    "p4": {"AC_GS_PARTITIONS": "4"},
    "p8": {"AC_GS_PARTITIONS": "8"},
    "rerun": {"AC_GS_PARTITIONS": "2", "AC_GS_TABLE_SLOTS": "1001"},     # tables too small for a partition's keys: count reruns
}


def split_alternatives(case, parts):
    """Substitution rows whose true alternative key S(p, e) lies in another spectrum partition than one of the window's two other
    alternatives, so that the screen's masks of that word are written by two partitions' sweeps."""
    out = []
    for x in measured(case):
        if (len(x["mid"]), x["skip"]) != (1, 1):
            continue
        first = x["checked"][0]                              # S(p, e)
        others = [first[:-1] + b for b in V.BASES if b not in (x["REF"], first[-1])]
        if any(V.partition(w, parts) != V.partition(first, parts) for w in others):
            out.append(x)
    return out


@pytest.mark.parametrize("name", ["kinds_k21_L3", "offsets_k21_L1", "junction_k21", "multi"])
@pytest.mark.parametrize("setting", sorted(SWEEPS))
@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_partitions_and_reruns(lib, cases, name, setting, tmp_path, monkeypatch):
    """The same files and rows with 2, 4 and 8 spectrum partitions and with count reruns: the screen's three masks per word are OR-ed
    over the partitions' sweeps."""
    case = cases(name)
    env = SWEEPS[setting]
    with_env(monkeypatch, env)
    info, _ = check(lib, case, tmp_path / "out")
    parts = int(env["AC_GS_PARTITIONS"])
    assert info["partitions"] == parts
    if setting == "rerun":
        assert info["reruns"] > 0
    assert split_alternatives(case, parts)


@pytest.mark.parametrize("per", [2, 3, 5])
@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_candidate_batches(lib, cases, per, tmp_path, monkeypatch):
    """Candidate tables of `per` positions each: batch boundaries fall between the loci of one contig, after multi-allelic sites whose
    candidates all sit in one locus."""
    case = cases("multi")
    with_env(monkeypatch, {"AC_VARIANTS_TABLE_SLOTS": str(2 * per * V.candidate_windows(case.k, case.L))})
    info, _ = check(lib, case, tmp_path / "out")
    assert info["loci"] > 2 * per and info["batches"] == -(-info["loci"] // per)
