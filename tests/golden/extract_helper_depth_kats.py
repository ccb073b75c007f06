"""Writes tests/golden/helper_depth_kats.json: the data of the reference's unit tests for the helper's depth filter (test_depth_from_header
and test_depth_filter in helper.rs), so that the product can be checked against them without the reference's sources in this tree.
test_depth_filter's steps run one after another on the same file: each has its bounds (null: not given) and the records the file holds
afterwards (null: the file is gone).
usage: python tests/golden/extract_helper_depth_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/)"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def bound(text):
    text = text.strip()
    return None if text == "&None" else float(re.fullmatch(r"&Some\(([-0-9.]+)\)", text).group(1))


def main(ref):
    src = open(os.path.join(ref, "src", "helper.rs")).read()
    body = src[src.index("mod tests"):]
    headers = []
    for h, v in re.findall(r'assert_eq!\(depth_from_header\("([^"]*)"\), (Some\([-0-9.]+\)|None)\);', body):
        headers.append([h, None if v == "None" else float(v[5:-1])])
    test = body[body.index("fn test_depth_filter()"):]
    test = test[:test.index("#[test]")]
    lines = re.search(r'make_test_file\(&fasta, "(.*?)"\);', test, re.S).group(1)
    fasta = "".join(re.findall(r"(>[^\\]*\\n[^\\]*\\n)", lines)).replace("\\n", "\n")
    steps = []
    for m in re.finditer(r"depth_filter\(&out_prefix, (&None|&Some\([-0-9.]+\)), (&None|&Some\([-0-9.]+\))\);\s*(assert_eq!\(load_fasta\(&fasta\)\.len\(\), (\d+)\);|assert!\(panic::catch_unwind)", test):
        steps.append({"min_abs": bound(m.group(1)), "min_rel": bound(m.group(2)), "records": None if m.group(4) is None else int(m.group(4))})
    out = {"source": "Autocycler v0.6.1 src/helper.rs, mod tests", "depth_from_header": headers,
           "depth_filter": {"fasta": fasta, "steps": steps}}
    with open(os.path.join(HERE, "helper_depth_kats.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(f"{len(headers)} headers, {len(steps)} filter steps")


if __name__ == "__main__":
    main(sys.argv[1])
