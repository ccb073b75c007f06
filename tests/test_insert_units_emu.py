"""The k-mer table insert takes 64 windows per warp, two per lane (windows g0 + l and g0 + 32 + l of a unit aligned to 64 coordinates).
These cases put sequence starts and ends, dotted windows, shard cuts and repeated k-mers at every place inside such a unit, on the
host-emulation build, and every one must give the oracle's bytes: contigs shorter than a unit and of 63, 64 and 65 windows, ends that end
repair leaves dotted, a tandem repeat of period 32 (the windows g and g + 32, one lane's pair, hold the same k-mer), and sharded builds
over 2 and 3 emulated ranks whose first sequences start inside a unit."""
import os
import random
import subprocess
import sys
import tempfile

import pytest

import cases
import oracle_lib as o
from parity_common import check_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")
KS = [9, 31, 33, 51, 63, 91, 131]          # W = 1, 1, 2, 2, 2, 3, 5


def unit_case(seed, k):
    """Several files of short contigs (a contig of L bases has L windows), period-32 repeats, fragments of one genome with random ends
    (unrepaired: their dotted windows stay) and the genome itself on either strand."""
    rng = random.Random(seed)
    genome = cases.rand_seq(rng, rng.randint(3 * k, 3 * k + 200))
    short = [63, 64, 65] if k <= 63 else [k, k + 1, k + 63]
    files = []
    for f in range(rng.randint(2, 4)):
        recs = []
        for c in range(rng.randint(2, 5)):
            kind = rng.randrange(4)
            if kind == 0:
                s = cases.rand_seq(rng, rng.choice(short + [rng.randint(k, max(k, 63))]))
            elif kind == 1:
                unit = cases.rand_seq(rng, 32)
                s = cases.rand_seq(rng, rng.randint(0, 40)) + unit * (k // 32 + rng.randint(2, 4)) + cases.rand_seq(rng, rng.randint(0, 40))
            elif kind == 2:
                a = rng.randrange(len(genome) - k)
                s = cases.rand_seq(rng, rng.randint(1, k)) + genome[a:a + rng.randint(k, len(genome) - a)] + cases.rand_seq(rng, rng.randint(1, k))
            else:
                s = genome if rng.random() < 0.5 else cases.rc(genome)
            recs.append((f"c{c + 1}", s if len(s) >= k else s + cases.rand_seq(rng, k - len(s))))
        files.append((f"asm_{f:02d}.fasta", recs))
    return files


def _oracle_sequences(files, k):
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        try:
            return o.load_sequences(d, k)[1]
        except o.OracleError:
            return []


def _shard_starts(seqs, world):
    """Coordinate of each rank's first window: the padded forward strands are laid end to end, and rank r owns sequences
    [n r / world, n (r + 1) / world)."""
    starts, at = [], 0
    for t in seqs:
        starts.append(at)
        at += len(t[4])
    return [starts[len(seqs) * r // world] for r in range(1, world) if len(seqs) * r // world < len(seqs)]


def test_the_cases_hold_what_they_are_for():
    """The cases put sequence starts, and so shard cuts, in both halves of a unit, and hold dotted windows."""
    for k in KS:
        offsets, dotted = set(), 0
        for seed in range(12):
            seqs = _oracle_sequences(unit_case(1000 * k + seed, k), k)
            dotted += any(t[4].startswith(".") or t[4].endswith(".") for t in seqs)
            for world in (2, 3):
                offsets.update(g % 64 for g in _shard_starts(seqs, world))
        assert any(0 < x < 32 for x in offsets) and any(32 < x < 64 for x in offsets), (k, sorted(offsets))
        assert dotted >= 3, (k, dotted)


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    from autocycler_b200 import api
    return api.load_library(EMU)


@pytest.mark.parametrize("k", KS)
def test_windows_across_units(emu, k):
    for seed in range(12):
        check_case(emu, unit_case(1000 * k + seed, k), k)


WORKER = r'''
import os, sys
sys.path.insert(0, os.path.join({root!r}, "tests")); sys.path.insert(0, {root!r})
import torch.distributed as dist
import cases, oracle_lib as o, test_insert_units_emu as t
from autocycler_b200 import api, dist as acdist
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + os.environ["MASTER_PORT"], rank=rank, world_size=world)
lib = api.load_library(t.EMU)
ok = True
for k in t.KS:
    for seed in range(6):
        d = os.path.join({tmp!r}, f"k{{k}}_{{seed}}")
        if rank == 0:
            cases.write_case(t.unit_case(1000 * k + seed, k), d)
        dist.barrier()
        try:
            count, oseqs = o.load_sequences(d, k)
        except o.OracleError:
            continue
        seqs = [api.Sequence(*x[:1], x[4], x[1], x[2], x[3]) for x in oseqs]
        want = o.compress_seqs(oseqs, count, k)[0] if rank == 0 else None
        lo, hi = acdist.shard_bounds(len(seqs), rank, world)
        kg = api.KmerGraph(k, lib=lib)
        kg.add_sequences(seqs, count)
        g = acdist.from_kmer_graph_distributed(kg, lo, hi, "cpu")
        if rank == 0:
            api.simplify_structure(g)
            if g.gfa_bytes().decode() != want:
                ok = False
                print("MISMATCH k", k, "seed", seed, flush=True)
        kg.upload()
        g = acdist.compress_distributed(kg, lo, hi, "cpu")
        if rank == 0 and bytes(g.gfa_view()).decode() != want:
            ok = False
            print("MISMATCH (fused) k", k, "seed", seed, flush=True)
dist.barrier()
if rank == 0:
    print("RESULT", "OK" if ok else "FAIL", flush=True)
dist.destroy_process_group()
'''


@pytest.mark.parametrize("world", [2, 3])
def test_shard_cuts_inside_units(tmp_path, world):
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, tmp=str(tmp_path)))
    port = str(31500 + (os.getpid() % 2000) + world)
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=port, AC_EMU_POISON="1")
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(outs)
    assert "RESULT OK" in outs[0], outs[0]
