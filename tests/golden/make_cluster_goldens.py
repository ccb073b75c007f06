"""Writes tests/golden/cluster_goldens.json: the SHA-256 of every file `autocycler cluster` writes under clustering/ for cfg3
(12 assemblies x 6 replicons, k = 51, cutoff 0.2), compressed and clustered by the CPU oracles (oracle_lib, tests/cluster_oracle.py)."""
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import cluster_oracle  # noqa: E402
import oracle_lib  # noqa: E402
from autocycler_b200 import synth  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as d:
        synth.write_assemblies(synth.make_assemblies("cfg3"), d)
        gfa, _, _ = oracle_lib.compress_dir(d, 51)
    files = cluster_oracle.cluster(gfa, 0.2)
    out = {"cfg3_k51_cutoff0.2": {k: hashlib.sha256(v.encode()).hexdigest() for k, v in sorted(files.items())}}
    with open(os.path.join(HERE, "cluster_goldens.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
