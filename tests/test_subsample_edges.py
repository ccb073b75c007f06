"""`autocycler subsample` at the shapes its other tests never reach: an n50 whose running sum meets half the bases at the end of a
level-1 bucket, at the first length of a bucket, at the end of a run of equal lengths and one base past it, with odd bases, in buckets
up to 10, and on rows 63 and 64 across the 64-row batches; rows of 0 and 1 bases; bad records in later windows, after a window
doubled, and several in one window; gzip input in many windows; and the one byte a sample grows by when the last record lacks its
newline.  Every case runs on the host-emulation build and, marked gpu, on the CUDA build; each compares every file with
tests/subsample_oracle.py and asserts the shape it claims (the generators are in tests/subsample_edges.py)."""
import os
import subprocess

import pytest

import subsample_edges as E
import subsample_oracle as O
from autocycler_b200 import api, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = E.B


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
def lib(request):
    return request.getfixturevalue(request.param)


@pytest.fixture
def window(monkeypatch):
    def set_window(w):
        if w is None:
            monkeypatch.delenv("AC_SUBSAMPLE_WINDOW", raising=False)
        else:
            monkeypatch.setenv("AC_SUBSAMPLE_WINDOW", str(w))
    set_window(None)
    return set_window


def check(lib, path, out_dir, genome_size, count, depth, seed):
    """The product's files against the oracle's -> (info, the yaml's input row, its subset rows) as (count, bases, n50) tuples."""
    info = api.subsample(path, out_dir, genome_size, count, depth, seed, lib=lib)
    want = O.subsample(path, genome_size, count, depth, seed)
    got = {f: open(os.path.join(out_dir, f), "rb").read() for f in sorted(os.listdir(out_dir))}
    assert sorted(got) == sorted(want)
    for f in want:
        assert got[f] == want[f], f
    lines = got["subsample.yaml"].decode().splitlines()
    value = [int(x.split(": ")[1]) for x in lines if ": " in x]
    return info, tuple(value[:3]), [tuple(value[i:i + 3]) for i in range(3, len(value), 3)]


def write(lengths, path):
    synth.write_reads(E.reads_of(lengths), path)


# ---- n50 edges -------------------------------------------------------------------------------------------------------------------
SHAPE_OF = {  # shape -> (crossing bucket, the n50's cell in it, the next length in the row above z)
    "bucket0_end": (0, 0xFFFF, B),
    "bucket1_end": (1, 0xFFFF, 2 * B),
    "first_of_bucket": (3, 0, 200_000),
    "run_end": (2, 1234, 2 * B + 1235),
    "run_past": (2, 1235, 2 * B + 1235),
    "bucket10": (10, 0, 690_000),
}
N50_CASES = [  # (shape, n, count, seed, row); row None is the input
    ("bucket0_end", 200, 4, 3, None), ("bucket0_end", 200, 65, 3, 63), ("bucket0_end", 200, 65, 3, 64),
    ("bucket1_end", 200, 4, 4, None), ("bucket1_end", 200, 65, 4, 64),
    ("first_of_bucket", 200, 129, 5, 63), ("first_of_bucket", 200, 129, 5, 128),
    ("run_end", 200, 4, 6, None), ("run_end", 200, 65, 6, 64),
    ("run_past", 200, 65, 7, 63), ("run_past", 200, 129, 7, 64),
    ("bucket10", 200, 2, 8, None), ("bucket10", 200, 65, 8, 64),
]


def check_n50_case(lib, tmp_path, shape, n, count, seed, row, x=4, short=False):
    lengths, (gsize, depth), claim = E.n50_case(shape, n, count, seed, row, x, short)
    path = str(tmp_path / "r.fq")
    write(lengths, path)
    info, inp, outs = check(lib, path, str(tmp_path / "out"), gsize, count, depth, seed)
    assert info["reads_per_subset"] == claim["rps"] and len(outs) == count
    got = inp if row is None else outs[row]
    assert got[1:] == (claim["bases"], claim["n50"])
    bucket, cell, above = SHAPE_OF[shape]
    z, _, _, _, d, past = E.N50_SHAPES[shape]
    assert (claim["bucket"], claim["cell"]) == (bucket, cell)
    assert claim["bases"] % 2 == d and claim["sum_below"] < claim["half"] <= claim["sum_to_n50"]
    if past:       # half is one base past the end of z's run: the next length, in the same bucket, crosses
        assert claim["sum_to_z"] + 1 == claim["half"] and claim["n50"] == above and claim["n50"] >> 16 == z >> 16
    else:          # the running sum meets half exactly at the last read of the n50's run, and the next length is `above`
        assert claim["sum_to_n50"] == claim["half"] and claim["n50"] == z
        assert claim["ceil_n50"] == (above if d else z)          # odd bases: ceil(bases / 2) gives the next length
    if shape == "first_of_bucket":
        row_lengths = [L for i, L in enumerate(lengths) if row is None or i in set(E.row_members(n, seed, count, claim["rps"], row))]
        assert max(L for L in row_lengths if L < z) >> 16 < bucket


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("shape,n,count,seed,row", N50_CASES)
def test_n50_edges(lib, tmp_path, shape, n, count, seed, row):
    check_n50_case(lib, tmp_path, shape, n, count, seed, row)


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_rows_of_zero_and_one_base(lib, tmp_path):
    """Half the bases is 0: the n50 is 0 when the row holds a read of length 0, else 1."""
    path = str(tmp_path / "r.fq")
    write([0, 1], path)
    count = 65
    gsize, depth = E.settings(1, 4)
    info, inp, outs = check(lib, path, str(tmp_path / "out"), gsize, count, depth, 1)
    assert info["reads_per_subset"] == 1 and inp == (2, 1, 0)
    order = O.shuffle_order(2, 1)
    want = [(1, 1, 1) if order[O.subset_start(i, 2, count) % 2] == 1 else (1, 0, 0) for i in range(count)]
    assert outs == want and (1, 1, 1) in want and (1, 0, 0) in want


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("row,row_lengths", [(64, "zeros"), (63, "one_and_zeros")])
def test_subset_of_zero_length_reads(lib, tmp_path, row, row_lengths):
    n, count, seed = 200, 65, 9
    mem = E.row_members(n, seed, count, 100, row)
    built = [0] * 100 if row_lengths == "zeros" else [1] + [0] * 99
    lengths = E.place(n, mem, built, E.filler(n - 100))
    path = str(tmp_path / "r.fq")
    write(lengths, path)
    gsize, depth = E.settings(sum(lengths), 4)
    info, _, outs = check(lib, path, str(tmp_path / "out"), gsize, count, depth, seed)
    assert info["reads_per_subset"] == 100 and outs[row] == (100, sum(built), 0)


@pytest.mark.parametrize("lib", builds(), indirect=True)
def test_no_reads_per_subset(lib, tmp_path):
    n, count = 130, 129
    lengths = E.filler(n)
    path = str(tmp_path / "r.fq")
    write(lengths, path)
    gsize, depth = E.settings(sum(lengths), 1 << 20)
    info, inp, outs = check(lib, path, str(tmp_path / "out"), gsize, count, depth, 2)
    assert info["reads_per_subset"] == 0 and inp[:2] == (n, sum(lengths)) and outs == [(0, 0, 0)] * count
    assert all(os.path.getsize(tmp_path / "out" / f"sample_{i + 1:02}.fastq") == 0 for i in range(count))


# ---- bad records -----------------------------------------------------------------------------------------------------------------
def check_refused(lib, tmp_path, recs, rec, why):
    path = str(tmp_path / "r.fq")
    data = b"".join(recs)
    open(path, "wb").write(data)
    with pytest.raises(O.FastqError) as oe:
        O.parse_fastq(data)
    assert str(oe.value) == f"record {rec}: {E.REASON[why]}"
    out = tmp_path / "out"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.subsample(path, str(out), "1", lib=lib)
    assert e.value.code == -6 and e.value.message == f"Error reading FASTQ file: record {rec}: {E.REASON[why]}"
    assert out.is_dir() and os.listdir(out) == []


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("why", [E.NO_AT, E.NO_PLUS, E.TRUNCATED, E.UNEQUAL])
def test_bad_record_in_a_later_window(lib, tmp_path, window, why):
    w, j = 400, 37 if why != E.TRUNCATED else 52
    recs = E.with_bad(E.record_bytes(E.reads_of([30 + i for i in range(60)])), [(j, why)])
    where = E.windows_of([len(r) for r in recs], w)
    assert where[j] >= 1
    window(w)
    check_refused(lib, tmp_path, recs, j + 1, why)


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("at,why", [(0, E.UNEQUAL), (1, E.NO_PLUS)])
def test_bad_record_after_the_window_doubled(lib, tmp_path, window, at, why):
    """A record longer than the window makes it double; the long record itself, or the one after it, is bad."""
    w, j = 400, 20
    recs = E.record_bytes(E.reads_of([30] * 20 + [2000] + [30] * 10))
    assert len(recs[j]) > w and E.windows_of([len(r) for r in recs[:j]], w)[-1] >= 1
    recs = E.with_bad(recs, [(j + at, why)])
    window(w)
    check_refused(lib, tmp_path, recs, j + at + 1, why)


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("w", [1500, None])
def test_earliest_bad_record_wins(lib, tmp_path, window, w):
    """Three bad records in one window, the later ones with lower reason codes: the earliest is reported with its own reason."""
    bad = [(30, E.UNEQUAL), (32, E.NO_PLUS), (35, E.NO_AT)]
    recs = E.with_bad(E.record_bytes(E.reads_of([30 + i for i in range(80)])), bad)
    if w:
        where = E.windows_of([len(r) for r in recs], w)
        assert where[30] == where[32] == where[35] >= 1
    window(w)
    check_refused(lib, tmp_path, recs, 31, E.UNEQUAL)


@pytest.mark.gpu
def test_gpu_bad_records_across_blocks(gpu, tmp_path, window):
    n = 1 << 20
    recs = E.record_bytes(E.reads_of([12 + i % 7 for i in range(n)]))
    bad = [(700_000, E.UNEQUAL)] + [(700_000 + 25_000 * k, E.NO_PLUS if k % 2 else E.NO_AT) for k in range(1, 14)]
    check_refused(gpu, tmp_path, E.with_bad(recs, bad), 700_001, E.UNEQUAL)


# ---- gzip and windows -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("w", [300, 4096, 1 << 20, 3 << 20])
def test_gz_in_many_windows(lib, tmp_path, window, w):
    path = str(tmp_path / "r.fq.gz")
    data, claim = E.gz_many_windows(path, w)
    assert claim["cut_inside_line"] and claim["long_record"] > w and claim["size"] > 4 * w
    window(w)
    info, inp, _ = check(lib, path, str(tmp_path / "out"), "100", 4, 1.0, 4)
    assert info["windows"] > 1 and info["bytes_scanned"] == claim["size"] == len(data) and inp[0] == claim["records"]


@pytest.mark.parametrize("lib", builds(), indirect=True)
@pytest.mark.parametrize("w", [None, 700])
def test_sample_one_byte_longer_than_the_input(lib, tmp_path, window, w):
    """Every read in every sample and no final newline: a sample is the input plus that newline, win_bytes + 1 in one window."""
    path = str(tmp_path / "r.fq")
    gsize, depth, data = E.one_byte_case(path)
    window(w)
    info, inp, _ = check(lib, path, str(tmp_path / "out"), gsize, 4, depth, 3)
    assert info["reads_per_subset"] == inp[0] == 30 and (info["windows"] == 1) == (w is None)
    for i in range(4):
        assert open(tmp_path / "out" / f"sample_{i + 1:02}.fastq", "rb").read() == data + b"\n"


# ---- contention and scale on the GPU --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_one_length_in_every_row(gpu, tmp_path):
    """2^20 + 77 reads of one length at count 64: every row's atomics land on one level-1 and one level-2 cell."""
    n, L, count = (1 << 20) + 77, 24, 64
    path = str(tmp_path / "r.fq")
    write([L] * n, path)
    gsize, depth = E.settings(n * L, 64)
    info, inp, outs = check(gpu, path, str(tmp_path / "out"), gsize, count, depth, 5)
    rps = info["reads_per_subset"]
    assert rps == round(n / 16) and inp == (n, n * L, L) and outs == [(rps, rps * L, L)] * count


@pytest.mark.gpu
@pytest.mark.parametrize("shape,count,seed,row", [("bucket0_end", 65, 11, 64), ("run_past", 65, 12, 63), ("bucket10", 2, 13, None)])
def test_gpu_n50_edges_at_scale(gpu, tmp_path, shape, count, seed, row):
    check_n50_case(gpu, tmp_path, shape, 1 << 20, count, seed, row, x=64, short=True)
