"""Benchmark of `autocycler cluster` (one JSON line, like bench_trim.py).  Default: ac_cluster on cfg3's compress graph (12 assemblies x
6 replicons), gated on the SHA-256 bundle of tests/golden/cluster_goldens.json, with the distance and UPGMA kernels' times (CUDA events),
the host time of the per-cluster graphs and the whole call.  --upgma-n N: the UPGMA kernel alone on a seeded N x N matrix, checked
against the CPU oracle, whose one-core time is the baseline (--no-oracle skips it)."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:
        return f"unknown ({type(e).__name__})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--upgma-n", type=int, default=0)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import numpy as np
    from autocycler_b200 import api, synth
    name, power = card()
    out = {"gpu": name, "power_limit": power}
    if a.upgma_n:
        n = a.upgma_n
        rng = np.random.default_rng(n)
        m = rng.random((n, n))
        m = np.maximum(m, m.T)
        np.fill_diagonal(m, 0.0)
        ids = list(range(1, n + 1))
        h = api._Handle(api.load_library(), 51)
        times = []
        for s in range(a.warmup + a.steps):
            merges, ms = api.upgma(m, ids, handle=h)
            if s >= a.warmup:
                times.append(ms)
        out.update(metric="upgma", n=n, upgma_kernel_ms=min(times), upgma_kernel_ms_all=times)
        if not a.no_oracle:
            import cluster_oracle
            t0 = time.perf_counter()
            want = cluster_oracle.upgma(m, ids)
            out.update(oracle_ms=(time.perf_counter() - t0) * 1e3, matches_oracle=merges == want)
        print(json.dumps(out))
        return
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "cluster_goldens.json")))["cfg3_k51_cutoff0.2"]
    with tempfile.TemporaryDirectory() as d:
        synth.write_assemblies(synth.make_assemblies("cfg3"), os.path.join(d, "asm"))
        api.compress(os.path.join(d, "asm"), os.path.join(d, "ac"))
        gfa = open(os.path.join(d, "ac", "input_assemblies.gfa"), "rb").read()
    runs = []
    for s in range(a.warmup + a.steps):
        g, seqs = api.UnitigGraph.from_gfa_lines(gfa)
        t0 = time.perf_counter()
        g.cluster()
        wall = (time.perf_counter() - t0) * 1e3
        st = g.cluster_stats()
        if s >= a.warmup:
            runs.append(dict(st, wall_ms=wall))
    got = {"pairwise_distances.phylip": g.cluster_text("phylip"), "clustering.newick": g.cluster_text("newick"),
           "clustering.tsv": g.cluster_text("tsv"), "clustering.yaml": g.cluster_text("yaml")}
    for k in want:
        if "/" in k:
            got[k] = g.cluster_text("gfa" if k.endswith(".gfa") else "untrimmed_yaml", int(k.split("/")[1][8:]))
    ok = {k: hashlib.sha256(v.encode()).hexdigest() for k, v in got.items()} == want
    out.update(metric="ac_cluster_cfg3", golden_ok=ok, sequences=runs[-1]["sequences"], pass_clusters=runs[-1]["pass_clusters"],
               fail_clusters=runs[-1]["fail_clusters"], wall_ms=[r["wall_ms"] for r in runs], distance_kernel_ms=[r["distance_ms"] for r in runs],
               upgma_kernel_ms=[r["upgma_ms"] for r in runs], cluster_gfa_host_ms=[r["cluster_gfa_ms"] for r in runs])
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
