"""`autocycler dotplot` (dotplot.rs): the product's image against the CPU oracle (tests/dotplot_oracle.py), pixel for pixel, on seeded
inputs; the reference's unit-test data (tests/golden/dotplot_kats.json); the literal and vectorised oracle forms against each other;
the three input types, the errors and the PNG file.  The CPU tests run the product's code through the host-emulation library (the dot
kernels' bodies, serially); the tests marked gpu run the CUDA build on the H100."""
import gzip
import hashlib
import json
import os
import random
import struct
import subprocess
import zlib

import numpy as np
import pytest

import dotplot_oracle as O
from autocycler_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "dotplot_kats.json")))
GOLDENS = json.load(open(os.path.join(ROOT, "tests", "golden", "dotplot_goldens.json")))
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")


@pytest.fixture(scope="session")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


@pytest.fixture(scope="session")
def gpu():
    return api.load_library()


def rnd(rng, n, alphabet="ACGT"):
    return "".join(rng.choice(alphabet) for _ in range(n))


def rc(s):
    return O.reverse_complement(s.encode()).decode()


def mutate(rng, s, rate):
    return "".join(rng.choice("ACGT") if rng.random() < rate else c for c in s)


def make_case(name):
    """-> (seqs [(filename, name, bases)], res, kmer)"""
    rng = random.Random(name)
    if name.startswith("k"):                           # k = 10, 11, 32, 51, 100 (W = 1..4): repeats, inversions, palindromes at even k
        k = int(name[1:])
        g = rnd(rng, 3000)
        pal = "AATT" * 40 + "ACGT" * 30 + "GGATCC" * 10
        return ([("asm_1.fasta", "c1", g[:1200] + rc(g[1200:2000]) + g[2000:] + pal),
                 ("asm_2.fasta", "c1", mutate(rng, g, 0.01)),
                 ("asm_2.fasta", "c2", rc(g[500:1800]) + g[100:400] * 3)], 500, k)
    if name == "odd_bytes":                            # N, IUPAC letters and '.', lowercase, sequences shorter than k
        g = rnd(rng, 1500)
        return ([("a", "x", g[:600] + "NNNNNNNNNNNN" + g[600:1200] + "RYKM" + g[1200:]),
                 ("a", "y", rc(g[:700]) + "N" * 40 + g[700:] + "...." + g[:200].lower()),
                 ("b", "x", "ACGTN.RY" * 30 + rnd(rng, 300, "ACGTN") + "N" * 50),
                 ("b", "short", "ACGTACG"), ("c", "tiny", "N")], 501, 11)
    if name == "one_sequence":
        g = rnd(rng, 4000)
        return ([("", "only", g + rc(g[1000:1600]) + g[2000:2600])], 500, 21)
    if name.startswith("many_"):                       # 2 .. 60 sequences, and enough to shrink the gaps until boxes touch
        n = int(name[5:])
        g = rnd(rng, 1200)
        seqs = []
        for i in range(n):
            a = rng.randrange(0, 1000)
            piece = g[a:a + rng.randrange(30, 200)]
            seqs.append((f"f{i % 3}", f"s{i}", piece if i % 2 else rc(piece)))
        return (seqs, 500 if n < 100 else 503, 10)
    if name == "ties":                                 # bp/pixel below 1, and exact .5 ties (bp/pixel 2.0)
        g = rnd(rng, 300)
        seqs = [("", "a", g), ("", "b", rc(g))]
        return (seqs, 777, 10)
    if name == "ties_half":
        res, k = 500, 12                               # one sequence: 458 pixels; 916 windows give 2.0 bp/pixel, so every odd j is a .5 tie
        g = rnd(rng, 916 + k - 1)
        return ([("", "a", g)], res, k)
    if name == "tandem":
        unit = rnd(rng, 37)
        return ([("t", "a", unit * 60), ("t", "b", rc(unit) * 45 + rnd(rng, 200)), ("t", "c", "AC" * 500)], 640, 10)
    if name == "identical":
        g = rnd(rng, 2500)
        return ([("x", "a", g), ("y", "a", g), ("z", "a", g)], 500, 32)
    if name == "homopolymer":                          # one group of 10^4 windows
        return ([("h", "a", "A" * 5000 + rnd(rng, 500) + "T" * 5000), ("h", "b", "A" * 200)], 600, 10)
    raise KeyError(name)


CASES = ["k10", "k11", "k32", "k51", "k100", "odd_bytes", "one_sequence", "many_2", "many_7", "many_60", "many_130", "ties", "ties_half",
         "tandem", "identical"]
SLOW = ["homopolymer"]


def test_kats_kmer_positions():
    for case in KATS["kmer_positions"]:
        seq = case["seq"].encode()
        forward, reverse = O.get_all_kmer_positions(case["k"], seq, O.reverse_complement(seq))
        assert {k.decode(): v for k, v in forward.items()} == case["forward"]
        # the reference compares the reverse map's position lists as its test lists them (both orders occur)
        assert {k.decode(): sorted(v) for k, v in reverse.items()} == {k: sorted(v) for k, v in case["reverse"].items()}


def test_kats_between_seq_gap():
    for case in KATS["between_seq_gap"]:
        assert abs(O.between_seq_gap(case["gap"], case["max_total_gap"], case["seq_count"]) - case["expected"]) < 1e-8


def test_kats_product(emu):
    """The KAT's k-mers through the product: 4-mers are below the CLI's range, so the same sequence at k = 10 with its repeats"""
    seq = KATS["kmer_positions"][0]["seq"]
    seqs = [("", "a", seq * 3), ("", "b", rc(seq) * 2)]
    img, _ = api.dotplot_rgb(seqs, 500, 10, font="", lib=emu)
    assert np.array_equal(img, O.dotplot_literal(seqs, 500, 10))


@pytest.mark.parametrize("name", CASES)
def test_oracle_forms_agree(name):
    seqs, res, k = make_case(name)
    assert np.array_equal(O.dotplot_literal(seqs, res, k), O.dotplot_vectorised(seqs, res, k))


def _check(lib, name, font=""):
    seqs, res, k = make_case(name)
    img, info = api.dotplot_rgb(seqs, res, k, font=font, lib=lib)
    want = O.dotplot_vectorised(seqs, res, k, font=font or None)
    assert img.shape == (res, res, 3)
    diff = np.argwhere((img != want).any(axis=2))
    assert len(diff) == 0, f"{len(diff)} pixels differ, first at (y, x) = {diff[0].tolist()}"
    windows = sum(max(len(s) - k + 1, 0) for _, _, s in seqs)
    assert info["windows"] == windows
    assert info["text_height"] == O.layout(O._prepare(seqs), res, k, O.load_font(font or None))[3]
    return info


@pytest.mark.parametrize("name", CASES + SLOW)
def test_cases_emu(emu, name):
    info = _check(emu, name)
    if name == "odd_bytes":
        assert info["host_windows"] > 0
    if name == "homopolymer":
        assert info["dots"] > 10 ** 8


def test_layout_branches():
    seqs, res, k = make_case("many_130")
    starts, ends, _, _ = O.layout(seqs, res, k)
    assert min(starts[i + 1] - ends[i] for i in range(len(seqs) - 1)) <= 1   # the shrunk gap: outlines of neighbouring boxes touch
    seqs, res, k = make_case("ties_half")
    _, _, bpp, _ = O.layout(seqs, res, k)
    assert bpp == 2.0
    seqs, res, k = make_case("ties")
    assert O.layout(seqs, res, k)[2] < 1.0


# ---- inputs, errors and the PNG -----------------------------------------------------------------------------------------------

def read_png(path):
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, w, h = 8, b"", None, None
    while pos < len(data):
        n, typ = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert zlib.crc32(typ + body) == struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0]
        if typ == b"IHDR":
            w, h, depth, colour, _, _, interlace = struct.unpack(">IIBBBBB", body)
            assert (depth, colour, interlace) == (8, 2, 0)
        elif typ == b"IDAT":
            idat += body
        pos += 12 + n
    raw = zlib.decompress(idat)
    stride = w * 3 + 1
    rows = [raw[y * stride:(y + 1) * stride] for y in range(h)]
    assert all(r[0] == 0 for r in rows)                # the encoder writes filter type 0 only
    return np.frombuffer(b"".join(r[1:] for r in rows), dtype=np.uint8).reshape(h, w, 3)


def write_fasta(path, recs, gz=False):
    text = "".join(f">{n} some description\n{s}\n" for n, s in recs)
    if gz:
        with gzip.open(path, "wt") as f:
            f.write(text)
    else:
        open(path, "w").write(text)


def test_inputs_emu(emu, tmp_path):
    seqs, res, k = make_case("k32")
    d = tmp_path / "asm"
    d.mkdir()
    write_fasta(d / "asm_1.fasta", [(n, s) for f, n, s in seqs if f == "asm_1.fasta"])
    write_fasta(d / "asm_2.fasta.gz", [(n, s) for f, n, s in seqs if f == "asm_2.fasta"], gz=True)
    out = tmp_path / "dir.png"
    info = api.dotplot(str(d), str(out), res, k, font="", lib=emu)
    want = O.dotplot_vectorised([(f if f == "asm_1.fasta" else "asm_2.fasta.gz", n, s) for f, n, s in seqs], res, k)
    got = read_png(str(out))
    assert np.array_equal(got, want)
    assert info["windows"] == sum(len(s) - k + 1 for _, _, s in seqs)
    try:
        from PIL import Image
        assert np.array_equal(np.asarray(Image.open(str(out)).convert("RGB")), want)
    except ImportError:
        pass
    # one FASTA file (gzipped): no filename in the labels
    fa = tmp_path / "all.fa.gz"
    write_fasta(fa, [(f"{f}_{n}", s) for f, n, s in seqs], gz=True)
    api.dotplot(str(fa), str(tmp_path / "fa.png"), res, k, font="", lib=emu)
    assert np.array_equal(read_png(str(tmp_path / "fa.png")), O.dotplot_vectorised([("", f"{f}_{n}", s) for f, n, s in seqs], res, k))


def test_gfa_input_emu(emu, tmp_path):
    import oracle_lib
    rng = random.Random(7)
    g = rnd(rng, 3000)
    d = tmp_path / "asm"
    d.mkdir()
    # file and record order differ from the sorted (filename, name) order the GFA path uses
    write_fasta(d / "b.fasta", [("zeta", mutate(rng, g, 0.01)), ("alpha", rc(g[:900]))])
    write_fasta(d / "a.fasta", [("m", g)])
    gfa, _, _ = oracle_lib.compress_dir(str(d), 31)
    (tmp_path / "input_assemblies.gfa").write_text(gfa)
    want_seqs = []
    for fname in ("a.fasta", "b.fasta"):
        text = open(d / fname).read().split(">")[1:]
        for r in text:
            head, body = r.split("\n", 1)
            want_seqs.append((fname, head.split()[0], body.replace("\n", "")))
    want_seqs.sort()
    api.dotplot(str(tmp_path / "input_assemblies.gfa"), str(tmp_path / "g.png"), 500, 32, font="", lib=emu)
    assert np.array_equal(read_png(str(tmp_path / "g.png")), O.dotplot_vectorised(want_seqs, 500, 32))


def test_png_writer_emu(emu, tmp_path):
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, size=(37, 53, 3), dtype=np.uint8)
    api.png_write(str(tmp_path / "r.png"), img, lib=emu)
    assert np.array_equal(read_png(str(tmp_path / "r.png")), img)


def test_errors_emu(emu, tmp_path):
    seqs = [("", "a", "ACGT" * 10)]
    for res, k, msg in ((499, 32, "--res cannot be less than 500"), (10001, 32, "--res cannot be greater than 10000"),
                        (2000, 9, "--kmer cannot be less than 10"), (2000, 101, "--kmer cannot be greater than 100")):
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.dotplot_rgb(seqs, res, k, font="", lib=emu)
        assert e.value.code == -6 and e.value.message == msg
        with pytest.raises(api.AutocyclerGpuError) as e:
            api.dotplot(str(tmp_path), str(tmp_path / "x.png"), res, k, lib=emu)
        assert e.value.message == msg
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.dotplot(str(tmp_path / "missing"), str(tmp_path / "x.png"), lib=emu)
    assert e.value.code == -6 and e.value.message == "--input is neither a file nor a directory"
    (tmp_path / "junk.txt").write_text("\n\nhello\n")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.dotplot(str(tmp_path / "junk.txt"), str(tmp_path / "x.png"), lib=emu)
    assert e.value.message == "--input is neither GFA or FASTA"
    (tmp_path / "empty.gfa").write_text("H\tVN:Z:1.0\tKM:i:51\n")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.dotplot(str(tmp_path / "empty.gfa"), str(tmp_path / "x.png"), lib=emu)
    assert e.value.message == "no sequences were loaded"
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.dotplot_rgb([("f", "a", "ACGT" * 10), ("f", "a", "TTTT" * 10)], 500, 10, font="", lib=emu)
    assert e.value.code == -6 and "two sequences are named f a" in e.value.message
    (tmp_path / "dup").mkdir()
    write_fasta(tmp_path / "dup" / "x.fasta", [("a", "ACGT" * 10)])
    write_fasta(tmp_path / "dup" / "y.fasta", [("a", "ACGT" * 10)])
    api.dotplot(str(tmp_path / "dup"), str(tmp_path / "x.png"), 500, 10, font="", lib=emu)   # the same name in two files is two boxes


# ---- the CUDA build ----------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES + SLOW)
def test_cases_gpu(gpu, name):
    info = _check(gpu, name)
    assert info["kernel_ms"] > 0


@pytest.mark.gpu
def test_inputs_gpu(gpu, tmp_path):
    test_inputs_emu(gpu, tmp_path)


@pytest.mark.gpu
def test_errors_gpu(gpu, tmp_path):
    test_errors_emu(gpu, tmp_path)


@pytest.mark.gpu
def test_workload_a_golden_gpu(gpu):
    import bench_dotplot
    res, k = bench_dotplot.SETTINGS["a"]
    img, info = api.dotplot_rgb(bench_dotplot.sequences("a"), res, k, font="", lib=gpu)
    assert hashlib.sha256(img.tobytes()).hexdigest() == GOLDENS[bench_dotplot.NAMES["a"]]["rgb_sha256"]


@pytest.mark.gpu
def test_cli_gpu(tmp_path):
    font = write_test_font(tmp_path / "t.ttf")
    seqs, res, k = make_case("k11")
    fa = tmp_path / "x.fasta"
    write_fasta(fa, [(f"{f}_{n}", s) for f, n, s in seqs])
    r = subprocess.run([AUTOCYCLER, "dotplot", "-i", str(fa), "-o", str(tmp_path / "x.png"), "--res", str(res), "--kmer", str(k), "--font", font],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert np.array_equal(read_png(str(tmp_path / "x.png")), O.dotplot_vectorised([("", f"{f}_{n}", s) for f, n, s in seqs], res, k, font=font))
    d = tmp_path / "asm"
    d.mkdir()
    write_fasta(d / "a.fasta", [(n, s) for _, n, s in seqs[1:]])         # c1 and c2: names are unique within a file
    r = subprocess.run([AUTOCYCLER, "dotplot", "-i", str(d), "-o", str(tmp_path / "d.png"), "--res", "600", "--font", font], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert np.array_equal(read_png(str(tmp_path / "d.png")), O.dotplot_vectorised([("a.fasta", n, s) for _, n, s in seqs[1:]], 600, 32, font=font))


@pytest.mark.gpu
def test_labels_gpu(gpu, tmp_path):
    test_labels_emu(gpu, tmp_path)


# ---- labels: a TrueType font built here with struct -----------------------------------------------------------------------------

def _glyph(contours, short=False):
    """a simple glyph: contours of (x, y, on_curve); short: 1-byte deltas where they fit, and repeated flags"""
    pts = [p for c in contours for p in c]
    xs, ys = [p[0] for p in pts], [p[1] for p in pts]
    out = struct.pack(">hhhhh", len(contours), min(xs), min(ys), max(xs), max(ys))
    end, ends = -1, []
    for c in contours:
        end += len(c)
        ends.append(end)
    out += struct.pack(f">{len(ends)}H", *ends) + struct.pack(">H", 0)
    flags, xb, yb, px, py = [], b"", b"", 0, 0
    for x, y, on in pts:
        f = 1 if on else 0
        for v, prev, sbit, same, axis in ((x, px, 2, 16, "x"), (y, py, 4, 32, "y")):
            dv = v - prev
            if short and dv == 0:
                f |= same
            elif short and -255 <= dv <= 255:
                f |= sbit | (same if dv > 0 else 0)
                b = struct.pack(">B", abs(dv))
                xb, yb = (xb + b, yb) if axis == "x" else (xb, yb + b)
            else:
                b = struct.pack(">h", dv)
                xb, yb = (xb + b, yb) if axis == "x" else (xb, yb + b)
        flags.append(f)
        px, py = x, y
    fb, i = b"", 0
    while i < len(flags):                     # runs of equal flags use the repeat bit
        j = i
        while j + 1 < len(flags) and flags[j + 1] == flags[i] and j - i < 254:
            j += 1
        if short and j > i:
            fb += struct.pack(">BB", flags[i] | 8, j - i)
        else:
            fb += struct.pack(">B", flags[i]) * (j - i + 1)
        i = j + 1
    out += fb + xb + yb
    return out + b"\0" * (len(out) % 2)


def build_test_font():
    glyphs = [
        _glyph([[(50, 0, 1), (450, 0, 1), (450, 700, 1), (50, 700, 1)], [(100, 50, 1), (100, 650, 1), (400, 650, 1), (400, 50, 1)]]),   # .notdef
        b"",                                                                                   # space: no outline
        _glyph([[(40, -150, 1), (560, -150, 1), (560, 620, 1), (40, 620, 1)],                  # a box with a hole (lines)
                [(140, -50, 1), (140, 520, 1), (460, 520, 1), (460, -50, 1)]]),
        _glyph([[(275, 0, 0), (520, 20, 0), (500, 360, 1), (470, 700, 0), (275, 720, 0), (60, 700, 0), (40, 360, 1), (70, 10, 0)]]),   # quadratic, starts off the curve
        struct.pack(">hhhhh", -1, 0, 0, 400, 600) + struct.pack(">HHhh", 0x0001, 2, 0, 0),    # composite: advances, no ink
        _glyph([[(10, 0, 1), (300, 0, 1), (590, 0, 1), (590, 5, 1), (300, 760, 0), (10, 5, 1)], [(200, 100, 1), (300, 400, 1), (400, 100, 1)]], short=True),
    ]
    advances = [500, 300, 600, 550, 400, 620]
    glyf, loca = b"", [0]
    for g in glyphs:
        glyf += g
        loca.append(len(glyf))
    segs = [(ord(" "), ord(" "), [1]), (ord("."), ord("9"), [2] + [0] + [3] * 10), (ord("A"), ord("Z"), [5] * 26),
            (ord("_"), ord("_"), [4]), (ord("a"), ord("z"), [2] * 13 + [3] * 13)]
    n = len(segs) + 1
    ends = [e for _, e, _ in segs] + [0xFFFF]
    starts = [st for st, _, _ in segs] + [0xFFFF]
    arrays, ro = [], []
    for i, (_, _, ids) in enumerate(segs):
        ro.append(2 * (n - i) + 2 * sum(len(a) for a in arrays))
        arrays.append(ids)
    ro.append(0)
    body = struct.pack(">HHHH", 2 * n, 0, 0, 0) + struct.pack(f">{n}H", *ends) + b"\0\0" + struct.pack(f">{n}H", *starts)
    body += struct.pack(f">{n}h", *([0] * len(segs) + [1])) + struct.pack(f">{n}H", *ro)
    body += b"".join(struct.pack(f">{len(a)}H", *a) for a in arrays)
    sub = struct.pack(">HHH", 4, 6 + len(body), 0) + body
    cmap = struct.pack(">HHHHI", 0, 1, 3, 1, 12) + sub
    tables = {
        b"cmap": cmap,
        b"glyf": glyf,
        b"head": struct.pack(">IIIIHH", 0x10000, 0, 0, 0x5F0F3CF5, 0, 1000) + b"\0" * 16 + struct.pack(">hhhhHHhhh", 0, -200, 600, 800, 0, 8, 2, 0, 0),
        b"hhea": struct.pack(">Ihhh", 0x10000, 800, -200, 0) + b"\0" * 22 + struct.pack(">hH", 0, len(glyphs)),
        b"hmtx": b"".join(struct.pack(">Hh", a, 0) for a in advances),
        b"loca": struct.pack(f">{len(loca)}H", *[o // 2 for o in loca]),
        b"maxp": struct.pack(">IH", 0x5000, len(glyphs)),
    }
    off = 12 + 16 * len(tables)
    head, data = struct.pack(">IHHHH", 0x10000, len(tables), 0, 0, 0), b""
    for tag in sorted(tables):
        t = tables[tag] + b"\0" * (-len(tables[tag]) % 4)
        head += tag + struct.pack(">III", 0, off + len(data), len(tables[tag]))
        data += t
    return head + data


def write_test_font(path):
    path.write_bytes(build_test_font())
    return str(path)


def label_cases():
    rng = random.Random("labels")
    g = rnd(rng, 2500)
    short = [("asm_1.fasta", "c1", g), ("asm_2.fasta", "c1", rc(g[300:2000]))]
    long_names = [(f"assembly_number_{i}_with_a_LONG_filename_0123456789.fasta", f"contig {i} x_y.z", g[i * 200:i * 200 + 300 + 150 * i])
                  for i in range(7)]
    odd = [("Ünïcode.fa", "weird_€_name", g[:900]), ("", "A", g[400:1400]), ("b.fa", "", g[100:300])]
    medium = [(f"sample_{i}_assembly.fasta", f"contig_{i}_circular", g[i * 100:i * 100 + 1500]) for i in range(3)]
    return [("short", short, 500, 32), ("medium", medium, 700, 21), ("long", long_names, 777, 11), ("odd", odd, 640, 10), ("many", make_case("many_60")[0], 500, 10)]


@pytest.mark.parametrize("case", [c[0] for c in label_cases()])
def test_label_oracle_forms_agree(tmp_path, case):
    font = write_test_font(tmp_path / "t.ttf")
    _, seqs, res, k = next(c for c in label_cases() if c[0] == case)
    assert np.array_equal(O.dotplot_literal(seqs, res, k, font=font), O.dotplot_vectorised(seqs, res, k, font=font))


def test_labels_emu(emu, tmp_path):
    font = write_test_font(tmp_path / "t.ttf")
    for name, seqs, res, k in label_cases():
        img, info = api.dotplot_rgb(seqs, res, k, font=font, lib=emu)
        want = O.dotplot_vectorised(seqs, res, k, font=font)
        diff = np.argwhere((img != want).any(axis=2))
        assert len(diff) == 0, f"{name}: {len(diff)} pixels differ, first at (y, x) = {diff[0].tolist()}"
        max_font = max(int(O.rust_round(0.025 * res)), 1)
        if name == "long":
            assert info["text_height"] < max_font        # long names shrink the font, and with it the top-left gap
        plain, plain_info = api.dotplot_rgb(seqs, res, k, font="", lib=emu)
        assert plain_info["text_height"] == max_font
        starts = O.layout(O._prepare(seqs), res, k)[0]
        top = plain[:starts[0] - 1]                     # above the boxes: labels only
        assert (top == 255).all()                       # no font: no label ink
        grey = want[:O.layout(O._prepare(seqs), res, k, O.load_font(font))[0][0] - 1]
        assert (grey < 255).any() or info["text_height"] < 2   # with the font: label ink above the boxes (unless shrunk to nothing)
        if name == "short":                             # labels that fit at the largest size: the layout is the same with and without
            assert info["text_height"] == plain_info["text_height"]
            box = np.argwhere((plain != 255).any(axis=2)).min(axis=0)
            assert (box == np.argwhere((want[box[0]:, box[1]:] != 255).any(axis=2)).min(axis=0) + box).all()
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.dotplot_rgb(label_cases()[0][1], 500, 32, font=str(tmp_path / "missing.ttf"), lib=emu)
    assert e.value.code == -6 and "cannot read the font file" in e.value.message
    (tmp_path / "bad.ttf").write_bytes(b"not a font")
    with pytest.raises(api.AutocyclerGpuError) as e:
        api.dotplot_rgb(label_cases()[0][1], 500, 32, font=str(tmp_path / "bad.ttf"), lib=emu)
    assert e.value.code == -6


def test_cli_errors(tmp_path):
    """The CLI's argument parsing, messages and exit codes.  It links the CUDA library; these paths stop before any device work, so
    they run without a GPU (drawing an image needs one: test_cli_gpu)."""
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc")], check=True)
    fa = tmp_path / "x.fasta"
    write_fasta(fa, [("a", "ACGT" * 20)])
    (tmp_path / "junk.txt").write_text("hello\n")
    for args, msg in ((["-i", str(fa), "--kmer", "5"], "Error: --kmer cannot be less than 10"),
                      (["-i", str(fa), "--kmer", "101"], "Error: --kmer cannot be greater than 100"),
                      (["-i", str(fa), "--res", "499"], "Error: --res cannot be less than 500"),
                      (["-i", str(fa), "--res", "10001"], "Error: --res cannot be greater than 10000"),
                      (["-i", str(tmp_path / "nope")], "Error: --input is neither a file nor a directory"),
                      (["-i", str(tmp_path / "junk.txt")], "Error: --input is neither GFA or FASTA"),
                      (["-i", str(fa), "--font", str(tmp_path / "none.ttf")], "Error: cannot read the font file")):
        r = subprocess.run([AUTOCYCLER, "dotplot", *args, "-o", str(tmp_path / "y.png")], capture_output=True, text=True)
        assert r.returncode == 1 and msg in r.stderr, (args, r.stderr)
    r = subprocess.run([AUTOCYCLER, "dotplot", "-i", str(fa)], capture_output=True, text=True)
    assert r.returncode == 2
    r = subprocess.run([AUTOCYCLER, "dotplot", "-i", str(fa), "-o", "x.png", "--res", "abc"], capture_output=True, text=True)
    assert r.returncode == 2 and "invalid value" in r.stderr
