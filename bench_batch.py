#!/usr/bin/env python
"""bench_batch.py — trim and resolve of every QC-pass cluster: one CLI process per directory against one batched call.

Workload: cfg3 (12 assemblies x 6 replicons, seeded) through compress -> cluster, by the product, into a temporary directory.  Two arms,
each run on its own fresh copy of the QC-pass cluster directories:
  loop   `autocycler trim -c DIR` for every directory, then `autocycler resolve -c DIR` for every directory (the pipelines' shell loop)
  batch  `autocycler trim -c DIR...` once, then `autocycler resolve -c DIR...` once
The arms alternate over --reps repetitions, and every timed repetition must leave the same bytes in every output file as the other
arm; the first repetition of each arm is a warm-up.  One JSON line reports the median wall time per arm and command, the batched
calls' launches, jobs, DP cells, kernel ms and planned device buffer bytes (from ac_trim_dirs / ac_resolve_dirs on a further copy),
and the card with its power limit, read in the same run.

  python bench_batch.py [--reps 5]

Writes nothing into the tree.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True            # the tree may be read-only
AUTOCYCLER = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
OUTPUTS = ("2_trimmed.gfa", "2_trimmed.yaml", "3_bridged.gfa", "4_merged.gfa", "5_final.gfa")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                        os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]], capture_output=True, text=True, timeout=30)
    name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(limit)


def fresh(src, dst):
    shutil.copytree(src, dst)
    return sorted(os.path.join(dst, d) for d in os.listdir(dst))


def cli(*args):
    r = subprocess.run([AUTOCYCLER, *args], capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit(f"autocycler {' '.join(args[:1])} failed:\n{r.stderr}")


def run_arm(arm, dirs):
    """-> {command: wall seconds}"""
    times = {}
    for command in ("trim", "resolve"):
        t0 = time.perf_counter()
        if arm == "loop":
            for d in dirs:
                cli(command, "-c", d)
        else:
            cli(command, "-c", *dirs)
        times[command] = time.perf_counter() - t0
    return times


def outputs(dirs):
    return [[open(os.path.join(d, n), "rb").read() for n in OUTPUTS] for d in dirs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from autocycler_b200 import api, synth
    name, limit = card()
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_assemblies(synth.make_assemblies("cfg3"), os.path.join(tmp, "asm"))
        api.compress(os.path.join(tmp, "asm"), os.path.join(tmp, "ac"))
        api.cluster(os.path.join(tmp, "ac"))
        src = os.path.join(tmp, "ac", "clustering", "qc_pass")
        walls = {"loop": {"trim": [], "resolve": []}, "batch": {"trim": [], "resolve": []}}
        for rep in range(args.reps + 1):
            got = {}
            for arm in (("loop", "batch") if rep % 2 == 0 else ("batch", "loop")):
                dirs = fresh(src, os.path.join(tmp, f"{arm}{rep}"))
                t = run_arm(arm, dirs)
                got[arm] = outputs(dirs)
                if rep > 0:
                    for command in t:
                        walls[arm][command].append(t[command])
            if got["loop"] != got["batch"]:
                raise SystemExit(f"repetition {rep}: the batched outputs differ from the loop's")
        dirs = fresh(src, os.path.join(tmp, "info"))
        trim = api.trim_dirs(dirs)
        resolve = api.resolve_dirs(dirs)
        n = len(dirs)
    med = {arm: {c: statistics.median(v) for c, v in walls[arm].items()} for arm in walls}
    print(json.dumps({
        "impl": "b200", "bench": "batch", "workload": "cfg3_qc_pass", "clusters": n, "reps": args.reps, "gpu": name, "power_limit_w": limit,
        "loop_s": {c: round(v, 4) for c, v in med["loop"].items()}, "batch_s": {c: round(v, 4) for c, v in med["batch"].items()},
        "loop_total_s": round(sum(med["loop"].values()), 4), "batch_total_s": round(sum(med["batch"].values()), 4),
        "trim": trim, "resolve": resolve, "outputs_equal": True,
    }))


if __name__ == "__main__":
    main()
