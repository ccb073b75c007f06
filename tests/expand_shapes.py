"""Generators for test_expand_shapes.py: assemblies whose graphs drive the device repeat expansion (pipeline.cu LevelsCoopBody,
SimplifyCoopBody, ApplyLevelBody) into the shapes only the GPU runs — full grids, compares across 32-byte chunks, first-pass
relocations, multi-pass cascades — and the census that shows each case plants what it says, read from the graph before simplify."""
import collections
import ctypes
import re

import numpy as np

import oracle_lib as o

H100_SMS = 132                   # cudaDevAttrMultiProcessorCount on an H100 SXM (the arithmetic of the emulation build)
CUDA_ATTR_SM_COUNT = 16          # cudaDevAttrMultiProcessorCount
SIMPLIFY_PER_BLOCK = 64          # pipeline.cu: ac_launch_coop("simplify", ..., n_cands, 64)
LEVELS_PER_BLOCK = 4096          # pipeline.cu: ac_launch_coop("levels", ..., n_cands, 4096)
COOP_THREADS = 256               # backend.h: every cooperative CTA has 256 threads
SEQ_SLACK = 32                   # pipeline.h AC_SEQ_SLACK: spare arena bytes on both sides of a unitig
CHUNK = 32                       # warp_first_mismatch compares one byte per lane, 32 bytes a step
SORT_TILE = 2048                 # pipeline.cu AC_SORT_TILE (CUDA build)
LARGE_K = 127                    # from here on a case must fill the simplify grid


def device_sm_count():
    """The multiprocessor count of device 0, read from the CUDA runtime itself."""
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
    assert rt.cudaDeviceGetAttribute(ctypes.byref(v), CUDA_ATTR_SM_COUNT, dev) == 0
    return v.value


def full_grid(sms):
    """Candidates beyond which the simplify launch holds one CTA per SM (min(ceil(n / 64), SMs) CTAs)."""
    return SIMPLIFY_PER_BLOCK * sms


def looping_grid(sms):
    """Candidates beyond which a thread of the full simplify grid takes more than one candidate per level."""
    return COOP_THREADS * sms


# ---- the generators -------------------------------------------------------------------------------------------------------------------

_COMP = str.maketrans("ACGT", "TGCA")
TANDEM_UNITS = ("ACGTTGCAT", "GATTACAGCA", "TTGACCAGTCA", "CAG", "AT")     # few units, so equal leftovers recur across sites


def rc(s):
    return s[::-1].translate(_COMP)


def _bases(rng, n):
    return "".join(np.array(list("ACGT"))[rng.integers(0, 4, n)])


def _other(rng, b, avoid=""):
    return str(rng.choice([x for x in "ACGT" if x != b and x not in avoid]))


def _site(rng, kind, k, genome, p):
    """-> (ref length at p, alleles): the variant planted at genome position p.  Insertion kinds replace nothing (ref length 0)."""
    ref = genome[p]
    if kind == "snp":
        return 1, [ref, _other(rng, ref)]
    if kind == "pair":                          # two substitutions 33-40 bases apart: one compare meets both, a chunk or more apart
        d = int(rng.integers(33, 41))
        seg = genome[p:p + d + 1]
        return d + 1, [seg, _other(rng, seg[0]) + seg[1:d] + _other(rng, seg[d])]
    if kind == "multi":                         # 3 or 4 alleles of one base: 3 or 4 sources on both sides
        alts = [x for x in "ACGT" if x != ref]
        rng.shuffle(alts)
        return 1, [ref] + alts[:int(rng.integers(2, 4))]
    if kind == "indel":
        n = int(rng.integers(1, 21))
        if rng.random() < 0.5:
            return 1, [ref, ref + _bases(rng, n)]
        return n, [genome[p:p + n], ""]
    if kind == "homo":                          # homopolymer length: the common sequence runs through the run, capped pass after pass
        b = _other(rng, genome[p - 1], genome[p])
        h = int(rng.integers(3, 13))
        return 0, [b * (h + x) for x in range(int(rng.integers(2, 4)))]
    if kind == "tandem":                        # copy number of a tandem unit
        unit = TANDEM_UNITS[int(rng.integers(0, len(TANDEM_UNITS)))]
        c = int(rng.integers(2, 5))
        return 0, [unit * (c + x) for x in range(int(rng.integers(2, 4)))]
    if kind == "inv":                           # an inversion between inverted repeats: X U X' against X U' X', U = P M P'
        x = _bases(rng, k + 20)
        pp = _bases(rng, int(rng.integers(20, 41)))
        u = pp + _bases(rng, int(rng.integers(5, 21))) + rc(pp)
        return 0, [x + u + rc(x), x + rc(u) + rc(x)]
    raise ValueError(kind)


def _assemble(rng, kind_weights, k, n_sites, n_asm, gap, end_gap=None):
    """-> ([site kinds], [assembly sequence]) for one replicon of n_sites sites 2k + 1 + [0, gap) bases apart, the first and last
    `end_gap` bases from the contig's ends when it is given."""
    kinds = list(kind_weights)
    w = np.array([kind_weights[x] for x in kinds], dtype=float)
    genome = _bases(rng, n_sites * (2 * k + gap + 60) + 4 * k)
    pieces, prev = [[] for _ in range(n_asm)], 0
    p = 2 * k if end_gap is None else end_gap
    kinds_used = []
    for s in range(n_sites):
        kind = kinds[int(rng.choice(len(kinds), p=w / w.sum()))]
        r, alleles = _site(rng, kind, k, genome, p)
        order = rng.permutation(n_asm)
        for a in range(n_asm):
            pieces[a].append(genome[prev:p] + alleles[order[a] % len(alleles)])
        kinds_used.append(kind)
        prev = p + r
        p = prev + 2 * k + 1 + int(rng.integers(0, gap))
    end = prev + (2 * k if end_gap is None else end_gap)
    return kinds_used, ["".join(x) + genome[prev:end] for x in pieces]


# (name, k, {site kind: weight}, sites per replicon, replicons, assemblies, spacing jitter, sites at the contig ends)
CASES = [
    ("snp_k63", 63, {"snp": 1}, 2600, 1, 3, 20, False),
    ("snp_k65", 65, {"snp": 1}, 2600, 1, 3, 20, False),
    ("snp_k67_looping", 67, {"snp": 1}, 17_500, 1, 2, 20, False),
    ("snp_k127", 127, {"snp": 1}, 4400, 1, 2, 20, False),
    ("snp_pair_k129", 129, {"snp": 1, "pair": 1}, 4400, 1, 2, 20, False),
    ("snp_k131", 131, {"snp": 1}, 4400, 1, 2, 20, False),
    ("snp_pair_k255", 255, {"snp": 1, "pair": 1}, 4400, 1, 2, 10, False),
    ("snp_k501", 501, {"snp": 1}, 4400, 1, 2, 6, False),
    ("cascade_k65", 65, {"indel": 2, "multi": 2, "homo": 3, "tandem": 3}, 1500, 1, 5, 20, False),
    ("cascade_k129", 129, {"indel": 2, "multi": 2, "homo": 3, "tandem": 3}, 4400, 1, 4, 20, False),
    ("inverted_k65", 65, {"inv": 1, "snp": 1}, 600, 1, 3, 20, False),
    ("contig_ends_k99", 99, {"snp": 2, "indel": 1, "homo": 1}, 3, 24, 4, 20, True),
]
NAMES = [c[0] for c in CASES]
MULTI_PASS = ("cascade_k65", "cascade_k129")


def case(index):
    """-> (name, k, files, {site kind: count}): one file per assembly, one linear contig per replicon (odd assemblies on the other
    strand), every allele of a site in at least one assembly."""
    name, k, kinds, n_sites, n_rep, n_asm, gap, ends = CASES[index]
    rng = np.random.default_rng(9_000 + index)
    files = [(f"asm_{a:02d}.fasta", []) for a in range(n_asm)]
    planted = collections.Counter()
    for r in range(n_rep):
        used, seqs = _assemble(rng, kinds, k, n_sites, n_asm, gap, 1 + r % (k // 2 - 1) if ends else None)
        planted.update(used)
        for a, s in enumerate(seqs):
            files[a][1].append((f"contig_{r + 1}", rc(s) if a % 2 else s))
    return name, k, files, dict(planted)


# ---- the census ----------------------------------------------------------------------------------------------------------------------

def parse_gfa(text):
    """-> ({number: forward sequence}, [[(number, strand)] per path])"""
    seqs, paths = {}, []
    for ln in text.splitlines():
        f = ln.split("\t")
        if f[0] == "S":
            seqs[int(f[1])] = f[2]
        elif f[0] == "P":
            paths.append([(int(x[:-1]), x[-1] == "+") for x in f[2].split(",")])
    return seqs, paths


def _strand_seq(seqs, number, fwd):
    return seqs[number] if fwd else rc(seqs[number])


def _common(a, b, limit):
    m = 0
    while m < limit and a[m] == b[m]:
        m += 1
    return m


def candidates(gfa):
    """The exclusive input and output sets of the graph (oracle gfa_exclusive) with two or more members, each with what the first pass
    sees: common length, the index of every mismatch of each source against the first, the zero-length cap, the start-of-path cap.
    Fixed starts and ends are not left out: they only ever remove candidates."""
    seqs, paths = parse_gfa(gfa)
    fpos, rpos = collections.defaultdict(list), collections.defaultdict(list)
    for path in paths:                                    # unitig positions as the graph stores them: the offset of each occurrence
        total = sum(len(seqs[n]) for n, _ in path)
        off = 0
        for n, fwd in path:
            (fpos if fwd else rpos)[n].append(off)
            (rpos if fwd else fpos)[n].append(total - off - len(seqs[n]))
            off += len(seqs[n])
    out = []
    for number, (ins, outs) in o.gfa_exclusive(gfa).items():
        for side, spec in ((0, ins), (1, outs)):
            src = [(int(x[:-1]), x[-1] == "+") for x in spec.split(",")] if spec else []
            if len(src) < 2:
                continue
            view = [_strand_seq(seqs, n, f) for n, f in src]
            if side == 0:
                view = [v[::-1] for v in view]            # the common END, read backwards
            min_len = min(len(v) for v in view)
            common, mism = min_len, []
            for v in view[1:]:
                lim = min(len(v), len(view[0]))
                common = min(common, _common(v, view[0], lim))
                mism.append([i for i in range(lim) if v[i] != view[0][i]])
            dup = len({n for n, _ in src}) != len(src)
            zero_cap = (min_len - 1) // (2 if dup else 1)
            ps = (fpos if side == 0 else rpos)[number]
            start_cap = (min(ps) - 1 if min(ps) > 0 else 0) if ps else None
            out.append(dict(number=number, side=side, src=src, spec=spec, gn=len(src), common=common, min_len=min_len, mism=mism, dup=dup,
                            zero_cap=zero_cap, start_cap=start_cap))
    return out


def first_pass_c(c):
    """The bases the candidate moves when it is the first to touch its sources (they are as built)."""
    n = c["common"]
    if n > 0:
        n = min(n, c["zero_cap"])
    if n > 0 and c["start_cap"] is not None:
        n = min(n, c["start_cap"])
    return n


LAUNCH = re.compile(r"\[device\] expand_repeats launch: (\d+) passes \((\d+) so far\), (\d+) levels, (\d+) candidates")
LEVEL = re.compile(r"\[device\] pass (\d+) level (\d+): (\d+) due at its start")


def launches(stderr):
    """-> [(passes, passes so far, levels, candidates)] of the AC_HOST_PROFILE launch lines."""
    return [tuple(map(int, m)) for m in LAUNCH.findall(stderr)]


def level_lines(stderr):
    """-> {pass: {level: due}} of the emulation build's per-level lines (levels stepped over print nothing)."""
    out = collections.defaultdict(dict)
    for p, lv, due in LEVEL.findall(stderr):
        out[int(p)][int(lv)] = int(due)
    return out


def tie_groups(gfa):
    """The final GFA's unitigs in number order, grouped by (length, sequence): -> [(length, first index, last index)] of every group of
    two or more.  Within such a group the device renumbering falls through to depth and then position."""
    seqs, _ = parse_gfa(gfa)
    order = sorted(seqs)
    assert order == list(range(1, len(order) + 1))
    groups = collections.defaultdict(list)
    for x, n in enumerate(order):
        groups[seqs[n]].append(x)
    return [(len(s), min(xs), max(xs)) for s, xs in groups.items() if len(xs) > 1]


CHILD = """
import sys
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
from autocycler_b200 import api
lib = api.load_library(%(lib)r)
d, k, mode = sys.argv[1], int(sys.argv[2]), sys.argv[3]
kg, seqs, count = api.load_sequences(d, k, lib=lib)
if mode == "census":                        # the plain build's graph before simplify
    kg.upload()
    open(d + "/before.gfa", "wb").write(bytes(api.UnitigGraph.from_kmer_graph(kg).gfa_bytes()))
if mode in ("census", "fused"):             # one fused build (its AC_HOST_PROFILE lines go to stderr)
    kg.upload()
    open(d + "/fused.gfa", "wb").write(bytes(api.UnitigGraph.compress(kg).gfa_view()))
if mode == "repeat":                        # two fused builds on this handle, one on a fresh handle
    for r in range(2):
        kg.upload()
        open(d + "/fused_%%d.gfa" %% r, "wb").write(bytes(api.UnitigGraph.compress(kg).gfa_view()))
    kg2, _, _ = api.load_sequences(d, k, lib=lib)
    kg2.upload()
    open(d + "/fused_2.gfa", "wb").write(bytes(api.UnitigGraph.compress(kg2).gfa_view()))
print("DONE", flush=True)
"""
