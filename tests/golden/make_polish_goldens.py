"""Writes tests/golden/polish_goldens.json: for bench_polish.py's workloads a (1,000 planted errors) and c (bench_qv.py's QV 27 variant),
both against about 1 GB of reads of a 5 Mbp genome, the SHA-256 of every file `autocycler polish` writes, as the oracle
(tests/polish_oracle.py) computes them, with the summary's counts and the oracle's one-core time.  Workload b (gzipped reads) shares a's.
usage: python tests/golden/make_polish_goldens.py"""
import hashlib
import json
import os
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import genome_size_oracle as G  # noqa: E402
import polish_oracle as O  # noqa: E402
import qv_oracle as Q  # noqa: E402
import bench_polish as B  # noqa: E402


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        counts = None
        for name in ("a", "c"):
            d = os.path.join(tmp, name)
            os.makedirs(d)
            reads, asm = B.write_input(name, d)
            t0 = time.perf_counter()
            if counts is None:                               # a and c share their reads
                uk, uc, W = Q.read_counts(reads, B.K)
                counts = (O.Counts(uk, uc), np.bincount(np.minimum(uc, G.H - 1), minlength=G.H).astype(np.int64), W)
            r = O.run(reads, asm, B.K, counts=counts)
            summary = dict(zip(*(line.split("\t") for line in r["files"]["summary.tsv"].decode().splitlines())))
            out[name] = {"k": B.K, "read_windows": int(r["W"]), "valley": r["valley"], "min_count": r["t"], "summary": summary,
                         "oracle_seconds": round(time.perf_counter() - t0, 1),
                         "sha256": {n: hashlib.sha256(x).hexdigest() for n, x in sorted(r["files"].items())}}
            print(json.dumps({name: out[name]}), flush=True)
    with open(os.path.join(HERE, "polish_goldens.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
