"""Generators for test_kernel_shapes.py: inputs shaped for the kernels' multi-round, multi-tile and racing branches (the trim overlap
sweep, the bridge distance sweep, the UPGMA CTA and the k-mer table build), and the exact expectations built from the oracles."""
import ctypes
import math
import os
import random

import numpy as np

import trim_oracle as T
from autocycler_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SHARED_OPTIN = 227 * 1024           # cudaDevAttrMaxSharedMemoryPerBlockOptin on an H100 (the emulation build's constant)
CUDA_ATTR_SHARED_OPTIN = 97              # cudaDevAttrMaxSharedMemoryPerBlockOptin


def device_shared_optin():
    """The opt-in shared memory per block of device 0, read from the CUDA runtime itself."""
    rt = None
    for name in ("libcudart.so.12", "libcudart.so", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = ctypes.CDLL(name)
            break
        except OSError:
            continue
    assert rt is not None, "no CUDA runtime library to ask"
    dev, v = ctypes.c_int(), ctypes.c_int()
    assert rt.cudaGetDevice(ctypes.byref(dev)) == 0
    assert rt.cudaDeviceGetAttribute(ctypes.byref(v), CUDA_ATTR_SHARED_OPTIN, dev) == 0
    return v.value


def overlap_shared_k_max(optin):         # align.cu overlap_shared_k_max: three f64 diagonals of k + 1 cells, 64 B of static shared
    return (optin - 64) // 24 - 1


def bridge_shared_n_max(optin):          # align.cu bridge_shared_n_max: three u32 diagonals of n + 1 cells
    return optin // 12 - 1


# ---- trim ---------------------------------------------------------------------------------------------------------------------------

TRIM_WINDOWS = [31, 32, 33, 1023, 1024, 1025, 1056, 2047, 2049, 4097]
TRIM_WEIGHTS = ("equal", "mixed", "big")
TRIM_MIN_IDENTITY = {"equal": 0.75, "mixed": 2 / 3, "big": 0.5}      # equal: every fourth unit of the planted copy substituted -> 3/4 exactly


def trim_weights(kind, n_units, seed):
    rng = random.Random(seed)
    if kind == "equal":
        return {u: 7 for u in range(1, n_units + 1)}
    if kind == "mixed":
        return {u: rng.choice([1, 2, 3, 5, 10, 10]) for u in range(1, n_units + 1)}
    return {u: rng.choice([2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, rng.randint(1, 10)]) for u in range(1, n_units + 1)}


def trim_path(seed, k, mode, kind, n_units):
    """A path of exactly k units (the whole path is the window) with a planted overlap for `mode`: a start-end copy or a hairpin, of up
    to k / 3 units, changed without changing its length (equal weights: every fourth unit; otherwise random substitutions and one
    deletion balanced by one insertion).  Small alphabets add chance matches and ties all over the matrix; with two or three units
    many tracebacks meet a tie of up and left away from the planted copy, where the order of the gaps decides the trim."""
    rng = random.Random(seed)
    alphabet = rng.choice([2, 3, 40, n_units])

    def unit():
        return rng.choice([1, -1]) * rng.randint(1, alphabet)

    def fresh():
        return rng.choice([1, -1]) * rng.randint(1, n_units)

    def change(p):
        p = list(p)
        if kind == "equal":
            for x in range(1, len(p), 4):
                p[x] = fresh()
            return p
        for x in range(len(p)):
            if rng.random() < 0.1:
                p[x] = fresh()
        if len(p) > 2:
            del p[rng.randrange(len(p))]
            p.insert(rng.randrange(len(p) + 1), fresh())
        return p
    if k < 3 or rng.random() < 0.15:
        return [unit() for _ in range(k)]
    ov = max(1, min(k // 3, rng.choice([k // 3, k // 8, rng.randint(1, 64)])))
    core = [unit() for _ in range(k - ov)]
    if mode == "start_end":
        return core + change(core[:ov])
    if mode == "hairpin_end":
        return core + change(T.reverse_path(core[-ov:]))
    return change(T.reverse_path(core[:ov])) + core


def trim_call(mode, kind, k_shared, seed):
    """-> (paths, weights, min_identity, max_unitigs): one path per window, K and K + 1 among them (shared memory and HBM in one call)."""
    windows = TRIM_WINDOWS + [k_shared, k_shared + 1]
    n_units = 2 * max(windows) + 50
    paths = [trim_path(seed * 1000 + x, k, mode, kind, n_units) for x, k in enumerate(windows)]
    assert [len(p) for p in paths] == windows
    return paths, trim_weights(kind, n_units, seed), TRIM_MIN_IDENTITY[kind], max(windows) + 1


# ---- bridges ------------------------------------------------------------------------------------------------------------------------

BRIDGE_N = [255, 256, 257, 511, 512, 513]


def bridge_weights(big, n_units, seed):
    """small: every DP sum stays below 2^32 (FAST_DP holds); big: the wrapping set of test_resolve's _random_groups(big_weights=True)."""
    rng = random.Random(seed)
    if big:
        return {u: rng.choice([2 ** 31, 2 ** 31 - 1, rng.randint(2 ** 30, 2 ** 31), rng.randint(1, 100)]) for u in range(1, n_units + 1)}
    return {u: rng.choice([1, 10, 10, 10, rng.randint(1, 5000)]) for u in range(1, n_units + 1)}


def bridge_group(seed, n, m, n_units):
    """3-6 paths whose shortest non-empty path has n units: a base of n units, a variant of m units (m - n insertions and a few
    substitutions), a substituted copy of the base, duplicates and an empty path."""
    rng = random.Random(seed)
    alphabet = rng.choice([30, n_units])

    def unit():
        return rng.choice([1, -1]) * rng.randint(1, alphabet)
    base = [unit() for _ in range(n)]
    long = list(base)
    for _ in range(m - n):
        long.insert(rng.randrange(len(long) + 1), unit())
    for _ in range(rng.randint(0, 3)):
        long[rng.randrange(len(long))] = unit()
    sub = list(base)
    for _ in range(rng.randint(1, 4)):
        sub[rng.randrange(n)] = unit()
    paths = [base, long, sub, []]
    for _ in range(rng.randint(0, 2)):
        paths.append(list(rng.choice(paths)))
    rng.shuffle(paths)
    return paths


def bridge_groups(seed, n_units):
    out = []
    for x, n in enumerate(BRIDGE_N):
        for m in (n, n + 1, 2 * n + 3):
            out.append(bridge_group(seed * 100 + 3 * x + len(out), n, m, n_units))
    return out


def bridge_boundary_group(n_shared, seed):
    """Paths of N and N + 1 units (N = the last shared-memory size): two jobs of N rows, one of N + 1 rows, and the empty path's three."""
    rng = random.Random(seed)
    n_units = n_shared + 60
    a = [rng.choice([1, -1]) * u for u in range(1, n_shared + 1)]
    b, c = list(a), list(a)
    b.insert(rng.randrange(n_shared), n_shared + 1)
    c.insert(rng.randrange(n_shared), n_shared + 2)
    for _ in range(5):
        c[rng.randrange(len(c))] = rng.randint(n_shared + 3, n_units)
    w = {u: rng.randint(1, 1000) for u in range(1, n_units + 1)}
    return [a, b, list(a), c, []], w


def expected_jobs(groups, n_shared):
    """(shared, HBM) jobs: one per unordered pair of distinct paths of a group, on shared memory when its shorter path fits."""
    shared = hbm = 0
    for g in groups:
        d = []
        for p in g:
            if p not in d:
                d.append(p)
        for x in range(len(d)):
            for y in range(x + 1, len(d)):
                if min(len(d[x]), len(d[y])) <= n_shared:
                    shared += 1
                else:
                    hbm += 1
    return shared, hbm


# ---- UPGMA --------------------------------------------------------------------------------------------------------------------------

UPGMA_N = [1, 2, 3, 31, 32, 33, 1023, 1024, 1025, 2049]
UPGMA_KINDS = ("equal", "small_int", "real", "inf", "signed_zero")


def _symmetric(m):
    iu = np.triu_indices(len(m), 1)
    m[(iu[1], iu[0])] = m[iu]
    np.fill_diagonal(m, 0.0)
    return m


def upgma_matrix(kind, n, seed):
    """-> (matrix, ids).  equal: every merge an exact tie decided by (a, b); small_int: many ties, exact sums; inf: a few +inf entries;
    signed_zero: -0.0 and 0.0 entries side by side.  Every other matrix has ids that are not contiguous."""
    rng = np.random.default_rng(seed)
    if kind == "equal":
        m = np.full((n, n), 0.375)
    elif kind in ("small_int", "signed_zero"):
        m = rng.integers(0, 6 if kind == "small_int" else 3, (n, n)).astype(np.float64)
    else:
        m = rng.random((n, n))
    m = _symmetric(m)
    if kind == "inf":
        for _ in range(max(1, n // 64)):
            i, j = rng.integers(0, n, 2)
            if i != j:
                m[i, j] = m[j, i] = np.inf
    if kind == "signed_zero":
        iu = np.triu_indices(n, 1)
        neg = (m[iu] == 0.0) & (rng.random(len(iu[0])) < 0.5)
        m[(iu[0][neg], iu[1][neg])] = -0.0
        m[(iu[1][neg], iu[0][neg])] = -0.0
    ids = sorted(rng.choice(np.arange(1, 3 * n + 1), n, replace=False).tolist()) if seed % 2 else list(range(1, n + 1))
    return m, ids


def upgma_rescan_matrix(n, rows, seed):
    """The first merge (a, b = n - 1) leaves the rows 0..rows-1, whose minimum pointed at b, to be scanned again: more than a warp's worth."""
    rng = np.random.default_rng(seed)
    m = _symmetric(2.0 + rng.random((n, n)))
    b, a = n - 1, n // 2
    m[:rows, b] = m[b, :rows] = 1.5
    m[a, b] = m[b, a] = 0.5
    return m, list(range(1, n + 1))


def upgma_expected(m, ids):
    """cluster_oracle.upgma, up to the first merge at +inf.  From there every live pair is at +inf (a sum with an infinite term stays
    infinite) and the (distance, a, b) order merges the two live clusters of least index each time, as in any other tie."""
    import cluster_oracle as O
    want = O.upgma(m, ids)
    p = next((x for x, mg in enumerate(want) if mg[3] == math.inf), len(want))
    label = list(ids)
    live = list(range(len(ids)))
    index = {v: x for x, v in enumerate(ids)}
    out = list(want[:p])
    for node, left, right, _ in out:
        a, b = index[left], index[right]
        label[a] = node
        index[node] = a
        live.remove(b)
    nxt = out[-1][0] if out else max(ids, default=0)
    while len(live) > 1:
        a, b = live[0], live[1]
        nxt += 1
        out.append((nxt, label[a], label[b], math.inf))
        label[a] = nxt
        live.remove(b)
    return out


def merge_bits(merges):
    return [(a, b, c, float(d).hex()) for a, b, c, d in merges]


# ---- the k-mer build ------------------------------------------------------------------------------------------------------------------

KMER_KS = [21, 31, 51, 63, 65, 127, 129, 255]          # W = 1, 1, 2, 2, 3, 4, 5, 8
SORT_TILE, SORT_WAYS = 2048, 8                         # pipeline.cu AC_SORT_TILE (CUDA build), AC_SORT_WAYS


def _bases(rng, n):
    return np.frombuffer(bytes(rng.choice(b"ACGT") for _ in range(n)), dtype=np.uint8).copy()


def _homopolymer(rng, n):
    return np.full(n, ord(rng.choice("ACGT")), dtype=np.uint8)


def _tandem(rng, n, period):
    unit = _bases(rng, period)
    return np.resize(unit, n)


def _inverted(rng, n):
    seg = _bases(rng, n)
    return [seg, _bases(rng, rng.randint(0, 40)), synth.revcomp(seg)]


def _insert(rng, g, pieces):
    for p in pieces:
        at = rng.randrange(len(g))
        g = np.concatenate([g[:at], p, g[at:]])
    return g


# (name, assemblies, replicon lengths, edits, (sub, ins, dele) or None for identical copies of one assembly)
KMER_CASES = [
    ("homopolymer_runs", 3, [120_000], [("homo", 2_000, 20_000, 6)], (5e-4, 2.5e-4, 2.5e-4)),
    ("homopolymer_runs_many_assemblies", 8, [60_000], [("homo", 2_000, 8_000, 4)], (5e-4, 2.5e-4, 2.5e-4)),
    ("homopolymer_two_replicons", 4, [90_000, 50_000], [("homo", 5_000, 20_000, 3)], (1e-4, 0, 0)),
    ("tandem_period_2", 4, [100_000], [("tandem2", 2_000, 20_000, 4)], (5e-4, 2.5e-4, 2.5e-4)),
    ("tandem_period_3", 4, [100_000], [("tandem3", 2_000, 20_000, 4)], (5e-4, 2.5e-4, 2.5e-4)),
    ("tandem_period_4", 4, [100_000], [("tandem4", 2_000, 20_000, 4)], (5e-4, 2.5e-4, 2.5e-4)),
    ("tandem_mixed_periods", 6, [80_000], [("tandem2", 2_000, 6_000, 2), ("tandem3", 2_000, 6_000, 2), ("tandem4", 2_000, 6_000, 2)], (5e-4, 0, 0)),
    ("identical_16", 16, [60_000], [], None),
    ("identical_16_homopolymer", 16, [50_000], [("homo", 3_000, 6_000, 2)], None),
    ("identical_16_tandem", 16, [50_000], [("tandem3", 2_000, 4_000, 2)], None),
    ("inverted_repeats", 4, [150_000], [("inv", 2_000, 10_000, 6)], (5e-4, 2.5e-4, 2.5e-4)),
    ("inverted_and_tandem", 5, [100_000], [("inv", 1_000, 5_000, 4), ("tandem2", 2_000, 10_000, 2)], (5e-4, 2.5e-4, 2.5e-4)),
    ("homopolymer_and_inverted", 3, [200_000], [("homo", 2_000, 15_000, 4), ("inv", 3_000, 8_000, 3)], (5e-4, 2.5e-4, 2.5e-4)),
    ("divergent_3k_unitigs", 6, [150_000], [], (3e-3, 1e-3, 1e-3)),
    ("divergent_two_merge_passes", 16, [220_000], [], (2e-3, 1e-3, 1e-3)),
    ("divergent_plasmids", 8, [120_000, 40_000, 10_000], [("homo", 2_000, 4_000, 1)], (2e-3, 5e-4, 5e-4)),
    ("tandem_long_runs", 3, [200_000], [("tandem2", 15_000, 20_000, 2), ("tandem4", 15_000, 20_000, 2)], (2e-4, 1e-4, 1e-4)),
    ("homopolymer_all_bases", 4, [100_000], [("homo", 2_000, 4_000, 8)], (5e-4, 2.5e-4, 2.5e-4)),
    ("mixed_contention", 12, [60_000], [("homo", 2_000, 5_000, 2), ("tandem3", 2_000, 5_000, 1), ("inv", 1_000, 3_000, 2)], (1e-3, 5e-4, 5e-4)),
    ("identical_16_inverted", 16, [50_000], [("inv", 2_000, 5_000, 2)], None),
]


def kmer_case(index):
    """-> (name, k, files) of case `index`: a synthetic replicon set (synth.make_genome) with the edits planted, then one assembly per
    file (synth.derive_assembly: rotation, strand, substitutions and indels), or 16 copies of one assembly."""
    name, n_asm, lengths, edits, rates = KMER_CASES[index]
    k = KMER_KS[index % len(KMER_KS)]
    rng = random.Random(index)
    grng = synth.SplitMix64(7_000 + index)
    replicons = []
    for L in lengths:
        g = synth.make_genome(grng, L)
        for kind, lo, hi, count in edits:
            pieces = []
            for _ in range(count):
                n = rng.randint(lo, min(hi, L // 4))
                if kind == "homo":
                    pieces.append(_homopolymer(rng, n))
                elif kind.startswith("tandem"):
                    pieces.append(_tandem(rng, n, int(kind[-1])))
                else:
                    pieces.append(np.concatenate(_inverted(rng, n)))
            g = _insert(rng, g, pieces)
        replicons.append(g)
    files = []
    for a in range(n_asm):
        arng = synth.SplitMix64((index * 1_000_003 + 7919 * (a + 1)) & 0xFFFFFFFFFFFFFFFF)
        if rates is None:
            contigs = files[0][1] if files else None
            if contigs is None:
                contigs = [(f"contig_{i + 1}", bytes(c).decode()) for i, c in enumerate(synth.derive_assembly(arng, replicons, 5e-4, 2.5e-4, 2.5e-4))]
            files.append((f"asm_{a:02d}.fasta", list(contigs)))
            continue
        contigs = synth.derive_assembly(arng, replicons, *rates)
        files.append((f"asm_{a:02d}.fasta", [(f"contig_{i + 1}", bytes(c).decode()) for i, c in enumerate(contigs)]))
    return name, k, files


def sort_shape(n):
    """(tiles, merge passes) of sort_indices over n records on the GPU."""
    tiles = (n + SORT_TILE - 1) // SORT_TILE
    passes, width = 0, SORT_TILE
    while width < n:
        passes += 1
        width *= SORT_WAYS
    return tiles, passes


CHILD = """
import sys
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
from autocycler_b200 import api
lib = api.load_library(%(lib)r)
d, k, want = sys.argv[1], int(sys.argv[2]), open(sys.argv[3]).read()
kg, seqs, count = api.load_sequences(d, k, lib=lib)
for r in range(3):                          # one handle, three builds: the bytes must not depend on who wins a race
    sys.stderr.write("BUILD\\n"); sys.stderr.flush()
    kg.upload()
    g = api.UnitigGraph.compress(kg)
    assert bytes(g.gfa_view()).decode() == want, "build %%d: GFA differs from the oracle" %% r
    print("CAPACITY", g.timings().table_capacity, g.timings().table_used, flush=True)
print("CHECKED", flush=True)
"""
