"""Writes tests/golden/subsample_kats.json: the data of the reference's unit tests for `subsample` (test_parse_genome_size and
test_subsample_indices in subsample.rs), so that the oracle and the product can be checked against them without the reference's
sources in this tree.
usage: python tests/golden/extract_subsample_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/)"""
import ast
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main(ref):
    src = open(os.path.join(ref, "src", "subsample.rs")).read()
    body = src[src.index("mod tests"):]
    sizes = [[s, int(v)] for s, v in re.findall(r'assert_eq!\(parse_genome_size\("([^"]*)"\), (\d+)\);', body)]
    refused = re.findall(r'parse_genome_size\("([^"]*)"\);\s*\}\)\.is_err\(\)', body)
    order = ast.literal_eval(re.search(r"let read_order = vec!(\[[^\]]*\]);", body).group(1))
    indices = [{"count": int(c), "reads_per_subset": int(r), "i": int(i), "expected": sorted(ast.literal_eval(e))}
               for c, r, i, e in re.findall(r"assert_eq!\(subsample_indices\((\d+), (\d+), &read_order, (\d+)\), HashSet::from\((\[[^\]]*\])\)\);", body)]
    out = {"source": "Autocycler v0.6.1 src/subsample.rs, mod tests",
           "parse_genome_size": sizes, "parse_genome_size_refused": refused,
           "subsample_indices": {"read_order": order, "cases": indices}}
    with open(os.path.join(HERE, "subsample_kats.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(f"{len(sizes)} sizes, {len(refused)} refusals, {len(indices)} index cases")


if __name__ == "__main__":
    main(sys.argv[1])
