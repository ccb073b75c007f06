"""Writes tests/golden/depth_goldens.json: for bench_depth.py's workloads a (5 Mbp at 100x, the genome as the assembly) and c (a
chromosome and a 3-copy plasmid), the SHA-256 of the output FASTA, each contig's unique k-mers and depth, as the oracle
(tests/depth_oracle.py) computes them, with the oracle's one-core time.  Workload b (gzipped) shares a's.
usage: python tests/golden/make_depth_goldens.py"""
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import depth_oracle as O  # noqa: E402
import bench_depth as B  # noqa: E402


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in ("a", "c"):
            asm, reads = B.write_input(name, tmp)
            t0 = time.perf_counter()
            r = O.run(asm, reads, B.K)
            out[f"oracle_seconds_{name}"] = round(time.perf_counter() - t0, 1)
            out[name] = {"k": B.K, "fasta_sha256": hashlib.sha256(r["fasta"]).hexdigest(), "unique": r["unique"], "depths": r["depths"]}
    print(json.dumps(out), flush=True)
    with open(os.path.join(HERE, "depth_goldens.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
