"""Writes tests/golden/unassembled_goldens.json: for bench_unassembled.py's workload a (about 1 GB of reads of a 5 Mbp chromosome and two
plasmids against the chromosome alone), the SHA-256 of every file `autocycler unassembled` writes, as the oracle
(tests/unassembled_oracle.py) computes them, with W and the oracle's one-core time.  Workloads b (gzipped) and c (four partitions) share it.
usage: python tests/golden/make_unassembled_goldens.py"""
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import unassembled_oracle as O  # noqa: E402
import bench_unassembled as B  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as tmp:
        reads, asm = B.write_input("a", tmp)
        t0 = time.perf_counter()
        r = O.run(reads, asm, B.K)
        seconds = round(time.perf_counter() - t0, 1)
    out = {"oracle_seconds_a": seconds,
           "a": {"k": B.K, "read_windows": int(r["W"]), "valley": r["valley"], "min_count": r["t"], "selected_reads": len(r["selected"]),
                 "absent_kmers": r["absent_kmers"], "sha256": {n: hashlib.sha256(d).hexdigest() for n, d in sorted(r["files"].items())}}}
    print(json.dumps(out), flush=True)
    with open(os.path.join(HERE, "unassembled_goldens.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
