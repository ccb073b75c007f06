"""Writes tests/golden/qv_goldens.json: for bench_qv.py's workloads a (1 GB of reads against 12 assemblies of 5 Mbp) and c (a
chromosome and a 3-copy plasmid, with a variant), the SHA-256 of every file `autocycler qv` writes, as the oracle (tests/qv_oracle.py)
computes them, in the same working directory layout, with the oracle's one-core time.  Workload b (gzipped) shares a's.
usage: python tests/golden/make_qv_goldens.py [--workloads a,c]"""
import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import qv_oracle as O  # noqa: E402
import bench_qv as B  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="a,c")
    args = ap.parse_args()
    path = os.path.join(HERE, "qv_goldens.json")
    out = json.load(open(path)) if os.path.exists(path) else {}
    here = os.getcwd()
    for name in args.workloads.split(","):
        with tempfile.TemporaryDirectory() as tmp:
            os.chdir(tmp)
            try:
                reads, asm = B.write_input(name, tmp)
                t0 = time.perf_counter()
                r = O.run(reads, asm, B.K)
                out[f"oracle_seconds_{name}"] = round(time.perf_counter() - t0, 1)
            finally:
                os.chdir(here)
        out[name] = {"k": B.K, "valley": r["valley"], "min_count": r["t"], "solid_kmers": r["S"],
                     "sha256": {n: hashlib.sha256(d).hexdigest() for n, d in sorted(r["files"].items())}}
        print(json.dumps({name: out[name]}), flush=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
