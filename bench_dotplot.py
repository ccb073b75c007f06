"""Benchmark of `autocycler dotplot` on the GPU: one JSON line per workload.

  (a) cfg2   8 assemblies of a 4.64 Mbp chromosome at the reference's defaults (k = 32, res 2000): one lookup per window dominates.
  (b) k10    8 assemblies of a 1 Mbp replicon at k = 10: 10-mers recur by chance, so the groups are large and the dots dominate.

Each line: the median ac_dotplot_rgb time after warm-up and its kernels' time (CUDA events), windows, dots and dots/s, the PNG
encoding time on its own, parity of the image's SHA-256 against tests/golden/dotplot_goldens.json (made by the vectorised CPU oracle,
tests/golden/make_dotplot_goldens.py), and the card with its power limit read in the same run.  The images are drawn without labels
(font ""), so that they do not depend on the fonts a machine has.  kernel_ms spans the dot kernels from the first to the last and
includes two blocking reads of a count by the host.  The reference's one-core time is not
measured here.
usage: python bench_dotplot.py [--steps 5] [--warmup 2] [--workload a|b|all]"""
import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from autocycler_b200 import synth  # noqa: E402

NAMES = {"a": "a_cfg2_k32", "b": "b_1mbp_k10"}
SETTINGS = {"a": (2000, 32), "b": (2000, 10)}


def sequences(key):
    """-> [(filename, contig name, bytes)] in the order a directory of these assemblies loads (file order, then record order)"""
    if key == "a":
        asm = synth.make_assemblies("cfg2")
    else:
        asm = synth.make_assemblies("dotplot_k10", n_assemblies=8, replicon_lengths=[1_000_000], seed=20261016)
    return [(fname, header.split()[0], bytes(arr)) for fname, recs in asm for header, arr in recs]


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
        raise SystemExit("bench_dotplot.py: no CUDA device; the GPU path has no CPU fallback")
    try:
        goldens = json.load(open(os.path.join(ROOT, "tests", "golden", "dotplot_goldens.json")))
    except Exception:
        goldens = {}
    keys = ("a", "b") if args.workload == "all" else (args.workload,)
    card = torch.cuda.get_device_name(torch.cuda.current_device())
    for key in keys:
        name = NAMES[key]
        res, kmer = SETTINGS[key]
        seqs = sequences(key)
        times, kms = [], []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            img, info = api.dotplot_rgb(seqs, res, kmer, font="")  # returns once the image is back on the host; no labels
            dt = time.perf_counter() - t0
            if i >= args.warmup:
                times.append(dt)
                kms.append(info["kernel_ms"])
        with tempfile.TemporaryDirectory() as d:
            png_times = []
            for _ in range(3):
                t0 = time.perf_counter()
                api.png_write(os.path.join(d, "dotplot.png"), img)
                png_times.append(time.perf_counter() - t0)
            png_bytes = os.path.getsize(os.path.join(d, "dotplot.png"))
        ms = sorted(times)[len(times) // 2] * 1e3
        km = sorted(kms)[len(kms) // 2]
        gold = goldens.get(name, {})
        sha = hashlib.sha256(img.tobytes()).hexdigest()
        line = {
            "impl": "b200", "command": "dotplot", "workload": name, "gpu": card, "power_limit_w": power_limit_w(),
            "res": res, "kmer": kmer, "sequences": len(seqs), "steps": args.steps, "warmup": args.warmup,
            "dotplot_rgb_ms": round(ms, 3), "kernel_ms": round(km, 3),
            "windows": info["windows"], "groups": info["groups"], "dots": info["dots"], "host_windows": info["host_windows"],
            "dots_per_s": round(info["dots"] / (km / 1e3), 1) if km > 0 else None,
            "png_encode_ms": round(sorted(png_times)[1] * 1e3, 3), "png_bytes": png_bytes,
            "parity": {"ok": bool(gold) and sha == gold.get("rgb_sha256"), "golden_present": bool(gold)},
            "reference_one_core_s": "not measured",
        }
        print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workload", default="all", choices=["a", "b", "all"])
    run(ap.parse_args())


if __name__ == "__main__":
    main()
