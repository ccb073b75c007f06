"""Writes tests/golden/trim_kats.json: the data of the reference's trim.rs unit tests (paths, weights, settings and the expected
results of overlap_alignment, trim_path_start_end, trim_path_hairpin_end / _start), so that the oracle and the product can be checked
against them without the reference's sources in this tree.
usage: python tests/golden/extract_trim_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/trim.rs)"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def ints(text):
    return [int(x) for x in re.findall(r"-?\d+", text)]


def weights_of(text):
    return {int(a): int(b) for a, b in re.findall(r"(\d+)\s*=>\s*(\d+)", text)}


def piece(text):
    vals = dict(re.findall(r"(\w+):\s*(-?\w+)", text))
    conv = lambda v: 0 if v == "GAP" else -1 if v == "NONE" else int(v)
    return [conv(vals["a_unitig"]), conv(vals["a_index"]), conv(vals["b_unitig"]), conv(vals["b_index"])]


def extract(src):
    tests = src[src.index("mod tests"):]
    cases = []
    for name, body in re.findall(r"#\[test\]\s*fn (\w+)\(\) \{(.*?)\n    \}\n", tests, re.S):
        if not (name.startswith("test_trim_path") or name == "test_overlap_alignment"):
            continue
        weights, path, pending, pieces = None, None, None, None
        for stmt in (s.strip() for s in re.sub(r"//[^\n]*", "", body).split(";")):
            stmt = " ".join(stmt.split())
            if stmt.startswith("let weights"):
                weights = weights_of(stmt)
            elif stmt.startswith("let path"):
                path = ints(stmt[stmt.index("vec!"):])
            elif stmt.startswith("let alignment = overlap_alignment"):
                args = stmt[stmt.index("("):]
                nums = re.findall(r"&weights, ([\d.]+), (\d+), (true|false)", args)[0]
                pending = dict(kind="overlap_alignment", path=path, min_identity=float(nums[0]), max_unitigs=int(nums[1]), skip_diagonal=nums[2] == "true")
            elif stmt.startswith("let expected_alignment"):
                pieces = [piece(p) for p in re.findall(r"AlignmentPiece \{[^}]*\}", stmt)]
            elif stmt.startswith("let trimmed_path = trim_path_"):
                fn = re.search(r"trim_path_(\w+)\(", stmt).group(1)
                mi, mu = re.findall(r"&weights, ([\d.]+), (\d+)\)", stmt)[0]
                if "&trimmed_path.unwrap()" in stmt:      # a second trim on the first one's result
                    pending = dict(pending, kind=pending["kind"] + "_then_" + fn)
                else:
                    pending = dict(kind=fn, path=path, min_identity=float(mi), max_unitigs=int(mu))
            elif stmt.startswith("assert"):
                if "is_none()" in stmt or "is_empty()" in stmt:
                    expected = None
                elif "expected_alignment" in stmt:
                    expected = pieces
                elif "trimmed_path.unwrap()" in stmt:
                    expected = ints(stmt[stmt.index("vec!"):])
                else:
                    continue
                cases.append(dict(test=name, weights={str(a): b for a, b in sorted(weights.items())}, expected=expected, **pending))
    return cases


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    src = open(os.path.join(sys.argv[1], "src", "trim.rs")).read()
    cases = extract(src)
    json.dump({"source": "Autocycler v0.6.1 src/trim.rs, mod tests", "cases": cases}, open(os.path.join(HERE, "trim_kats.json"), "w"), indent=None)
    print(len(cases), "cases")
