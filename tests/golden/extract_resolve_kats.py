"""Writes tests/golden/resolve_kats.json: the data of the reference's resolve.rs unit tests (anchor-to-anchor segments, their grouping,
bridge fields, ambiguity flags, best paths and global_alignment_distance values), so that the oracle and the product can be checked
against them without the reference's sources in this tree.
usage: python tests/golden/extract_resolve_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/resolve.rs)"""
import ast
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def literal(text):
    """A Rust vec!/hashmap! literal as Python data (tuple keys become "a,b" strings for JSON)."""
    t = text.replace("vec![", "[").replace("hashmap!{", "{").replace("=>", ":").replace("HashSet::from(", "(")
    return ast.literal_eval(t)


def extract(src):
    tests = src[src.index("mod tests"):]
    cases = []
    for name, body in re.findall(r"#\[test\]\s*fn (\w+)\(\) \{(.*?)\n    \}\n", tests, re.S):
        env, bridges = {}, {}
        for stmt in (" ".join(s.split()) for s in re.sub(r"//[^\n]*", "", body).split(";")):
            m = re.match(r"let mut bridges = vec!\[(.*)\]$", stmt)
            if m:
                env["bridges"] = [bridges[x.strip()] for x in m.group(1).split(",")]
                continue
            m = re.match(r"let (?:mut )?(\w+)(?:: [\w<>]+)? = (.*)$", stmt)
            if m and m.group(2).startswith(("vec!", "hashmap!", "HashSet::from")):
                env[m.group(1)] = literal(m.group(2))
                continue
            m = re.match(r"let (\w+) = Bridge::new\((-?\d+), (-?\d+), (.*), &unitig_lengths\)$", stmt)
            if m:
                paths = env[m.group(4)] if m.group(4) in env else literal(m.group(4))
                bridges[m.group(1)] = {"start": int(m.group(2)), "end": int(m.group(3)), "paths": paths}
                continue
            w = {str(k): v for k, v in env.get("unitig_lengths", {}).items()}
            m = re.match(r"assert_eq!\(bridge\.best_path, (.*)\)$", stmt)
            if m:
                cases.append({"test": name, "kind": "best_path", "weights": w, "start": bridges["bridge"]["start"], "end": bridges["bridge"]["end"],
                              "paths": bridges["bridge"]["paths"], "expected": literal(m.group(1))})
                continue
            m = re.match(r"assert_eq!\(bridge\.(rev_start|rev_end|depth)\(\), (-?\d+)\)$", stmt)
            if m:
                cases.append({"test": name, "kind": "bridge_" + m.group(1), "weights": w, "start": bridges["bridge"]["start"],
                              "end": bridges["bridge"]["end"], "paths": bridges["bridge"]["paths"], "expected": int(m.group(2))})
                continue
            m = re.match(r"assert!\((!?)bridges\[(\d+)\]\.conflicting\)$", stmt)
            if m:
                if not cases or cases[-1]["test"] != name:
                    cases.append({"test": name, "kind": "ambiguity", "weights": w, "bridges": env["bridges"], "expected": []})
                assert int(m.group(2)) == len(cases[-1]["expected"])
                cases[-1]["expected"].append(m.group(1) != "!")
                continue
            m = re.match(r"assert_eq!\(global_alignment_distance\((\w+)\.as_slice\(\), (\w+)\.as_slice\(\), &unitig_lengths\), (\d+)\)$", stmt)
            if m:
                cases.append({"test": name, "kind": "distance", "weights": w, "a": env[m.group(1)], "b": env[m.group(2)], "expected": int(m.group(3))})
                continue
            m = re.match(r"assert_eq!\(anchor_to_anchor_paths, (.*)\)$", stmt)
            if m:
                cases.append({"test": name, "kind": "anchor_to_anchor", "sequence_paths": env["sequence_paths"], "anchor_set": sorted(env["anchor_set"]),
                              "expected": literal(m.group(1))})
                continue
            m = re.match(r"assert_eq!\(grouped_paths, (.*)\)$", stmt)
            if m:
                cases.append({"test": name, "kind": "group", "paths": env["anchor_to_anchor_paths"],
                              "expected": [[list(k), v] for k, v in literal(m.group(1)).items()]})
                continue
            if stmt.startswith(("assert", "let")) and "determine_ambiguity" not in stmt and "get_anchor" not in stmt and "group_paths" not in stmt:
                raise SystemExit(f"{name}: statement not understood: {stmt}")
    return cases


def main():
    src = open(os.path.join(sys.argv[1], "src", "resolve.rs")).read()
    cases = extract(src)
    tests = sorted({c["test"] for c in cases})
    assert len(tests) == 11, tests
    with open(os.path.join(HERE, "resolve_kats.json"), "w") as f:
        json.dump({"source": "Autocycler v0.6.1 src/resolve.rs unit tests", "cases": cases}, f, indent=1)
        f.write("\n")
    print(f"{len(cases)} cases from {len(tests)} tests")


if __name__ == "__main__":
    main()
