"""Writes tests/golden/variants_goldens.json: for bench_variants.py's workload a (about 1.2 GB of reads of a 5 Mbp genome and of a copy with
2,500 planted variants, against the genome), the SHA-256 of every file `autocycler variants` writes, as the oracle
(tests/variants_oracle.py) computes them, with the summary's counts and the oracle's one-core time.  Workload b (gzipped reads) shares a's.
usage: python tests/golden/make_variants_goldens.py"""
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import variants_oracle as O  # noqa: E402
import bench_variants as B  # noqa: E402


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        reads, asm, want = B.write_input("a", tmp)
        t0 = time.perf_counter()
        r = O.run(reads, asm, B.K, max_indel=B.MAX_INDEL)
        summary = dict(zip(*(line.split("\t") for line in r["files"]["summary.tsv"].decode().splitlines())))
        got = {(x["pos"], x["REF"], x["ALT"]) for x in r["rows"]}
        out["a"] = {"k": B.K, "max_indel": B.MAX_INDEL, "read_windows": int(r["W"]), "valley": r["valley"], "min_count": r["t"],
                    "summary": summary, "planted": len(want), "recovered": len(got & want), "extra_rows": len(got - want),
                    "oracle_seconds": round(time.perf_counter() - t0, 1),
                    "sha256": {n: hashlib.sha256(x).hexdigest() for n, x in sorted(r["files"].items())}}
        print(json.dumps(out), flush=True)
    with open(os.path.join(HERE, "variants_goldens.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
