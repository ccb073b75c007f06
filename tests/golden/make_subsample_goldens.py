"""Writes tests/golden/subsample_goldens.json: the SHA-256 of every output of bench_subsample.py's workloads as the oracle
(tests/subsample_oracle.py) computes them, with the oracle's one-core time.  Workload b is a's reads gzipped, so it shares a's hashes.
usage: python tests/golden/make_subsample_goldens.py"""
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import subsample_oracle as O  # noqa: E402
import bench_subsample as B  # noqa: E402


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in ("a", "c"):
            path = B.write_input(name, tmp)
            t0 = time.perf_counter()
            files = O.subsample(path, B.WORKLOADS[name]["genome_size"], 4, 25.0, 0)
            out[f"oracle_seconds_{name}"] = round(time.perf_counter() - t0, 1)
            out[name] = {f: hashlib.sha256(files[f]).hexdigest() for f in sorted(files)}
            os.remove(path)
            print(name, out[f"oracle_seconds_{name}"], files["subsample.yaml"].decode(), flush=True)
    with open(os.path.join(HERE, "subsample_goldens.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
