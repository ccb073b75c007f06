"""The N>1 path on CPU: world_size-2 (and 3) torch.distributed `gloo` groups driving the host-emulation build of the
device stages (tests/emu), compared byte-for-byte with the oracle.  The same code path runs over NCCL in bench.py."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys
sys.path.insert(0, os.path.join({root!r}, "tests")); sys.path.insert(0, {root!r})
import torch, torch.distributed as dist
import cases, oracle_lib as o
from autocycler_b200 import api, dist as acdist, synth
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + os.environ["MASTER_PORT"], rank=rank, world_size=world)
lib = api.load_library(os.path.join({root!r}, "tests", "emu", "libautocycler_emu.so"))
ok = True
todo = []
for seed, k in [(1, 9), (2, 31), (3, 51), (717, 9), (44, 5), (45, 65), (46, 91)]:
    todo.append((cases.random_case(seed * 100 + k, k), k))
big = synth.make_assemblies("x", n_assemblies=5, replicon_lengths=[40_000, 3_000], seed=77)
todo.append(([(fn, [(h, s.tobytes().decode()) for h, s in recs]) for fn, recs in big], 51))
import table_routes                  # a small file and a large walk the size estimate cannot see: the small file's rank overflows while merging
for big_first in (False, True):
    todo.append((table_routes.walk_case(77, 0.0, big_first=big_first), 51))
for ci, (files, k) in enumerate(todo):
    d = os.path.join({tmp!r}, f"case{{ci}}")
    if rank == 0:
        cases.write_case(files, d)
    dist.barrier()
    try:
        count, oseqs = o.load_sequences(d, k)
    except o.OracleError:
        continue
    seqs = [api.Sequence(*t[:1], t[4], t[1], t[2], t[3]) for t in oseqs]
    kg = api.KmerGraph(k, lib=lib)
    kg.add_sequences(seqs, count)
    lo, hi = acdist.shard_bounds(len(seqs), rank, world)
    if hi == lo:            # more ranks than sequences: give the empty ranks nothing to do but still take part
        lo, hi = 0, 0
    g = acdist.from_kmer_graph_distributed(kg, lo, hi, "cpu")
    want = o.compress_seqs(oseqs, count, k)[0] if rank == 0 else None
    if rank == 0:
        api.simplify_structure(g)
        got = g.gfa_bytes().decode()
        if got != want:
            ok = False
            print("MISMATCH case", ci, "k", k, flush=True)
    kg.upload()
    g = acdist.compress_distributed(kg, lo, hi, "cpu")          # the fused form: expansion, renumbering and text on rank 0's device
    if rank == 0 and bytes(g.gfa_view()).decode() != want:
        ok = False
        print("MISMATCH (fused) case", ci, "k", k, flush=True)
    cuts = [acdist.shard_bounds(len(seqs), r, world) for r in range(world)]
    kg = api.KmerGraph(k, lib=lib)                                   # a fresh handle: its strand buffer holds nothing yet
    kg.add_sequences(seqs, count, upload=False)
    if any(b == a for a, b in cuts):
        kg.upload()
    else:                                                            # every rank uploads its own strands only; broadcasts bring the rest
        acdist.upload_sharded(kg, [c[0] for c in cuts] + [len(seqs)], "cpu")
    g2, lines = acdist.compress_distributed_split(kg, lo, hi, "cpu")   # the same with every rank printing the P lines of its own sequences
    parts = [None] * world
    dist.all_gather_object(parts, bytes(lines.view()))
    if rank == 0 and (bytes(g2.gfa_view()) + b"".join(parts)).decode() != want:
        ok = False
        print("MISMATCH (split path lines) case", ci, "k", k, flush=True)
dist.barrier()
if rank == 0:
    print("RESULT", "OK" if ok else "FAIL", flush=True)
dist.destroy_process_group()
'''


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_build_matches_oracle(tmp_path, world):
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, tmp=str(tmp_path)))
    port = str(29500 + (os.getpid() % 2000) + world)
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=port,
                   AC_EMU_POISON="1")        # every device buffer a kernel writes is filled with a pattern before each table build: leftovers of the previous build on the handle cannot help
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(outs)
    assert "RESULT OK" in outs[0], outs[0]
