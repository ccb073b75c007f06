"""Writes tests/golden/dotplot_goldens.json: the SHA-256 of the RGB buffer (res x res x 3, row-major) that the vectorised dotplot oracle
(tests/dotplot_oracle.py) draws, without labels, for the benchmark workloads of bench_dotplot.py, with the dot count.  CPU only.
usage: python tests/golden/make_dotplot_goldens.py [a] [b]"""
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench_dotplot  # noqa: E402
import dotplot_oracle  # noqa: E402


def main():
    keys = sys.argv[1:] or ["a", "b"]
    path = os.path.join(HERE, "dotplot_goldens.json")
    out = json.load(open(path)) if os.path.exists(path) else {}
    for key in keys:
        name = bench_dotplot.NAMES[key]
        res, kmer = bench_dotplot.SETTINGS[key]
        seqs = bench_dotplot.sequences(key)
        t0 = time.perf_counter()
        img = dotplot_oracle.dotplot_vectorised(seqs, res, kmer)
        out[name] = {"res": res, "kmer": kmer, "rgb_sha256": hashlib.sha256(img.tobytes()).hexdigest(),
                     "oracle_seconds": round(time.perf_counter() - t0, 1)}
        print(name, out[name], flush=True)
        json.dump(out, open(path, "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
