#!/usr/bin/env python
"""bench_trim.py — DP cells/s through `autocycler trim`'s overlap alignments (ac_trim), one JSON line.

The workload is what `autocycler cluster` writes as 1_untrimmed.gfa for a one-cluster genome: the config's compress GFA through
merge_linear_paths (cluster.rs:794-806).  cfg2 (the default) has 8 paths of about 72,000 unitigs, so every alignment uses the full
window; `--max-unitigs 12000` puts the windows above what a CTA's shared memory holds, so the DP diagonals live in HBM (the kernel's
other side).  Every run is gated on the trim oracle's committed SHA-256 (tests/golden/trim_goldens.json, make_trim_goldens.py).

  python bench_trim.py [--workload cfg2] [--max-unitigs 5000] [--steps K] [--warmup W] [--no-cpu-baseline]

Writes nothing into the tree: the synthetic assemblies go to a temporary directory.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True            # the tree may be read-only
from bench import WORKLOADS, gpu_identity  # noqa: E402

TRIM_METRIC = "DP cells/sec through trim's overlap alignments (ac_trim)"


def run_trim(args):
    """trim.rs:43-51 (ac_trim) on what `autocycler cluster` writes as 1_untrimmed.gfa for a one-cluster genome — the
    workload's compress GFA through merge_linear_paths (cluster.rs:794-806).  The timed call is ac_trim on a freshly loaded graph
    (loading is untimed); the alignment kernels are also timed alone with CUDA events.  DP cells = the sum of k^2 over the alignments,
    k = min(--max-unitigs, path length).  Parity: SHA-256 of the trim oracle's 2_trimmed.gfa (tests/golden/trim_goldens.json)."""
    import hashlib
    import tempfile
    import torch
    from autocycler_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the GPU path has no CPU fallback")
    workload = args.workload
    golden_key = f"{workload}_k{args.k}_trim_mu{args.max_unitigs}"
    try:
        golden = json.load(open(os.path.join(ROOT, "tests", "golden", "trim_goldens.json")))[golden_key]
    except Exception:
        golden = {}
    with tempfile.TemporaryDirectory() as d:
        synth.write_assemblies(synth.make_assemblies(workload), d)
        kg, _, _ = api.load_sequences(d, args.k)
        kg.upload()
        g = api.UnitigGraph.compress(kg)
        api.merge_linear_paths(g, seqs=[1])
        untrimmed = bytes(g.gfa_bytes())
    lib = g._h.lib
    paths = [len(g.get_unitig_path_for_sequence_i32(i)) for i in range(g.counts().n_sequences)]
    del g, kg
    graph, _ = api.UnitigGraph.from_gfa_lines(untrimmed)
    times, kernel_ms, out = [], [], None
    for i in range(args.warmup + args.steps):
        graph._h.check(lib.ac_load_gfa(graph._h.ptr, untrimmed, len(untrimmed)))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        graph.trim(0.75, args.max_unitigs, 5.0)        # returns after the device work it needs (its results are read back)
        dt = time.perf_counter() - t0
        if i >= args.warmup:
            times.append(dt)
            kernel_ms.append(graph.timings().trim_kernel)
    out = bytes(graph.gfa_bytes())
    stats = graph.trim_stats()
    sha = hashlib.sha256(out).hexdigest()
    ms = sorted(times)[len(times) // 2] * 1e3
    kms = sorted(kernel_ms)[len(kernel_ms) // 2]
    card = gpu_identity(torch.cuda.current_device())
    # overlap_shared_k_max (align.cu): three f64 diagonals of k + 1 entries per CTA, beside 64 bytes of static shared memory
    shared_k = (torch.cuda.get_device_properties(torch.cuda.current_device()).shared_memory_per_block_optin - 64) // 24 - 1
    line = {
        "impl": "b200", "command": "trim", "metric": TRIM_METRIC, "value": round(stats["dp_cells"] / (ms / 1e3), 1), "unit": "cells/s",
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms, 3), "higher_is_better": True,
        "kernel_ms": round(kms, 3), "kernel_cells_per_s": round(stats["dp_cells"] / (kms / 1e3), 1) if kms > 0 else None,
        "gpu": card,
        "config": {"workload": f"{WORKLOADS[workload]}, k={args.k}: compress GFA -> merge_linear_paths -> trim (--min_identity 0.75 --max_unitigs "
                               f"{args.max_unitigs} --mad 5)", "sequences": len(paths), "path_lengths": paths,
                   "windows": sorted({min(args.max_unitigs, n) for n in paths}), "alignments": stats["alignments"], "dp_cells": stats["dp_cells"],
                   "max_window": stats["max_window"], "shared_memory_window": stats["max_window"] <= shared_k},
        "parity": {"sha256": sha, "golden": golden.get("sha256"), "golden_key": golden_key,
                   "untrimmed_ok": hashlib.sha256(untrimmed).hexdigest() == golden.get("untrimmed_sha256"), "ok": sha == golden.get("sha256")},
    }
    if not args.no_cpu_baseline:
        # the trim oracle (tests/trim_oracle.py: the reference's full-matrix DP, rows vectorised with numpy) on one core; the reference
        # itself runs the per-sequence alignments in parallel over its -t threads (rayon, trim.rs:122,148)
        os.environ.setdefault("OMP_NUM_THREADS", "1")
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import trim_oracle
        t0 = time.perf_counter()
        ref_gfa, _ = trim_oracle.trim_gfa(untrimmed.decode(), 0.75, args.max_unitigs, 5.0)
        dt = time.perf_counter() - t0
        line["cpu_baseline"] = {"value": round(stats["dp_cells"] / dt, 1), "unit": "cells/s", "seconds": round(dt, 2), "cores": 1, "host_cores": os.cpu_count(),
                                "kind": "oracle", "same_output": ref_gfa.encode() == out,
                                "note": "trim oracle on one core; the reference parallelises this stage over its -t threads (rayon)"}
        line["vs_baseline"] = round((dt * 1e3) / ms, 2)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workload", default="cfg2", choices=sorted(WORKLOADS))
    ap.add_argument("--k", type=int, default=51)
    ap.add_argument("--max-unitigs", type=int, default=5000, help="trim's --max_unitigs (windows above about 9,680 keep the DP diagonals in HBM)")
    ap.add_argument("--no-cpu-baseline", action="store_true", help="skip the trim oracle's one-core run")
    run_trim(ap.parse_args())


if __name__ == "__main__":
    main()
