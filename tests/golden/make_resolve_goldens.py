"""Writes tests/golden/resolve_goldens.json: the SHA-256 of the resolve oracle's 3_bridged.gfa, 4_merged.gfa and 5_final.gfa on the
benchmark workloads of bench_resolve.py, whose 2_trimmed.gfa is made by the CPU oracles (compress, merge_linear_paths, trim), and the
resolve oracle's one-core time.  CPU only.
usage: python tests/golden/make_resolve_goldens.py [a] [b]"""
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench_resolve  # noqa: E402
import oracle_lib  # noqa: E402
import resolve_oracle  # noqa: E402
import trim_oracle  # noqa: E402
from autocycler_b200 import synth  # noqa: E402


def trimmed_gfa_oracle(key):
    with tempfile.TemporaryDirectory() as d:
        synth.write_assemblies(bench_resolve.assemblies(key), d)
        gfa, _, _ = oracle_lib.compress_dir(d, 51)
    untrimmed = oracle_lib.gfa_merge_linear_paths(gfa, use_paths=True, renumber=False)
    return trim_oracle.trim_gfa(untrimmed)[0]


def main():
    keys = sys.argv[1:] or ["a", "b"]
    path = os.path.join(HERE, "resolve_goldens.json")
    out = json.load(open(path)) if os.path.exists(path) else {}
    resolve_oracle.FAST_DP = True
    for key in keys:
        trimmed = trimmed_gfa_oracle(key)
        t0 = time.perf_counter()
        info = {}
        texts = resolve_oracle.resolve_gfa(trimmed, info)
        dt = time.perf_counter() - t0
        out[bench_resolve.NAMES[key]] = {"trimmed_sha256": hashlib.sha256(trimmed.encode()).hexdigest(),
                                         "sha256": {w: hashlib.sha256(t.encode()).hexdigest() for w, t in zip(("bridged", "merged", "final"), texts)},
                                         "oracle_seconds": round(dt, 2), "oracle": info}
        print(bench_resolve.NAMES[key], out[bench_resolve.NAMES[key]], flush=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
