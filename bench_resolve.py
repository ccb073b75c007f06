#!/usr/bin/env python
"""bench_resolve.py — `autocycler resolve` (ac_resolve) on two workloads, one JSON line each.

  (a) dense   cfg2's compress GFA -> merge_linear_paths -> trim: anchors every few unitigs, many bridges with tiny distance jobs.
  (b) sparse  one 120 kbp replicon in 12 assemblies whose 60 kbp stretch [40 k, 100 k) carries a 2e-2 substitution rate of its own in
              every assembly: a 51-mer free of errors in all 12 copies is rare there (0.98^612 ~ 4e-6 per position), so anchors vanish
              over the stretch and its bridge carries thousands of unitigs and ~12 distinct paths (composed from synth's functions with a
              fixed seed).

Each line reports the median ac_resolve time after warm-up, the distance kernels' time (CUDA events), jobs, cells and cells/s, which
storage form the jobs ran in (shared memory or HBM scratch), parity against the resolve oracle's SHA-256 (tests/golden/resolve_goldens.json,
make_resolve_goldens.py), the oracle's one-core time where given (--cpu-baseline), and the card with its power limit read in the same run.

  python bench_resolve.py [--workload a|b|all] [--steps K] [--warmup W] [--cpu-baseline]

Writes nothing into the tree: the synthetic assemblies go to a temporary directory.
"""
import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True            # the tree may be read-only

NAMES = {"a": "a_dense_cfg2", "b": "b_sparse_stretch"}


def sparse_assemblies():
    """Workload (b): 12 linear copies of a 120 kbp replicon at synth's default error rates, each with its own 2e-2 substitutions over
    [40 k, 100 k)."""
    import numpy as np
    from autocycler_b200 import synth
    grng = synth.SplitMix64(0xB0E5)
    genome = synth.make_genome(grng, 120_000, repeats=False)
    out = []
    for a in range(12):
        rng = synth.SplitMix64(0xB0E5 * 1_000_003 + 7919 * (a + 1))
        s = np.concatenate([synth.mutate(rng, genome[:40_000]), synth.mutate(rng, genome[40_000:100_000], sub=2e-2), synth.mutate(rng, genome[100_000:])])
        out.append((f"asm_{a:02d}.fasta", [(f"contig_1 length={len(s)}", s)]))
    return out


def assemblies(key):
    from autocycler_b200 import synth
    return synth.make_assemblies("cfg2") if key == "a" else sparse_assemblies()


def trimmed_gfa_gpu(key, d):
    """compress -> merge_linear_paths (what cluster writes for a one-cluster genome) -> trim, on the GPU: the text of 2_trimmed.gfa."""
    from autocycler_b200 import api, synth
    asm_dir = os.path.join(d, key)
    synth.write_assemblies(assemblies(key), asm_dir)
    kg, _, _ = api.load_sequences(asm_dir, 51)
    kg.upload()
    g = api.UnitigGraph.compress(kg)
    api.merge_linear_paths(g, seqs=[1])
    untrimmed = bytes(g.gfa_bytes())
    del g, kg
    g2, _ = api.UnitigGraph.from_gfa_lines(untrimmed)
    g2.trim()
    return bytes(g2.gfa_bytes()).decode()


def workloads(d, keys=("a", "b")):
    return {NAMES[k]: trimmed_gfa_gpu(k, d) for k in keys}


def power_limit_w():
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def run(args):
    import torch
    from autocycler_b200 import api
    if not torch.cuda.is_available():
        raise SystemExit("bench_resolve.py: no CUDA device; the GPU path has no CPU fallback")
    try:
        goldens = json.load(open(os.path.join(ROOT, "tests", "golden", "resolve_goldens.json")))
    except Exception:
        goldens = {}
    keys = ("a", "b") if args.workload == "all" else (args.workload,)
    card = torch.cuda.get_device_name(torch.cuda.current_device())
    with tempfile.TemporaryDirectory() as d:
        texts = workloads(d, keys)
    for key in keys:
        name = NAMES[key]
        text = texts[name]
        g, _ = api.UnitigGraph.from_gfa_lines(text.encode())
        times, kms = [], []
        for i in range(args.warmup + args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            g.resolve()                                # returns after the device work it needs (the distances are read back)
            dt = time.perf_counter() - t0
            if i >= args.warmup:
                times.append(dt)
                kms.append(g.resolve_stats()["kernel_ms"])
        st = g.resolve_stats()
        sha = {w: hashlib.sha256(g.resolve_text(w).encode()).hexdigest() for w in ("bridged", "merged", "final")}
        ms = sorted(times)[len(times) // 2] * 1e3
        km = sorted(kms)[len(kms) // 2]
        gold = goldens.get(name, {})
        line = {
            "impl": "b200", "command": "resolve", "workload": name, "gpu": card, "power_limit_w": power_limit_w(),
            "steps": args.steps, "warmup": args.warmup, "resolve_ms": round(ms, 3), "kernel_ms": round(km, 3),
            "jobs": st["jobs"], "cells": st["cells"], "cells_per_s": round(st["cells"] / (km / 1e3), 1) if km > 0 else None,
            "storage": {"shared_jobs": st["shared_jobs"], "hbm_jobs": st["hbm_jobs"]},
            "anchors": st["anchors"], "unique_bridges": st["unique_bridges"], "conflicting_bridges": st["conflicting_bridges"],
            "culled_bridges": st["culled_bridges"], "longest_path": st["longest_path"],
            "parity": {"ok": bool(gold) and sha == gold.get("sha256"), "golden_present": bool(gold),
                       "trimmed_ok": hashlib.sha256(text.encode()).hexdigest() == gold.get("trimmed_sha256")},
            "oracle_one_core_s": gold.get("oracle_seconds", "not measured"),
        }
        if args.cpu_baseline:
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            import resolve_oracle
            resolve_oracle.FAST_DP = True
            t0 = time.perf_counter()
            resolve_oracle.resolve_gfa(text)
            line["oracle_one_core_s"] = round(time.perf_counter() - t0, 2)
        print(json.dumps(line), flush=True)
        del g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workload", default="all", choices=["a", "b", "all"])
    ap.add_argument("--cpu-baseline", action="store_true", help="time the resolve oracle on one core in this run")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
