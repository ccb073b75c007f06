"""Writes tests/golden/genome_size_goldens.json: for bench_genome_size.py's workload a (5 Mbp at 100x with 1% errors, k = 21), the
SHA-256 of the k-mer histogram (AC_GENOME_SIZE_BINS little-endian u64 bins), W and the rule's outputs, as the oracle
(tests/genome_size_oracle.py) computes them, with the oracle's one-core time.  Workloads b (gzipped) and c (four partitions) share it.
usage: python tests/golden/make_genome_size_goldens.py"""
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import genome_size_oracle as O  # noqa: E402
import bench_genome_size as B  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as tmp:
        path = B.write_input("a", tmp)
        t0 = time.perf_counter()
        hist, W = O.histogram(path, B.K)
        est = O.estimate(hist, W)
        seconds = round(time.perf_counter() - t0, 1)
    out = {"oracle_seconds_a": seconds,
           "a": {"k": B.K, "histogram_sha256": B.histogram_sha256(hist), "windows": W, **est}}
    print(json.dumps(out), flush=True)
    with open(os.path.join(HERE, "genome_size_goldens.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
