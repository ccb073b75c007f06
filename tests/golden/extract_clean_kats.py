"""Writes tests/golden/clean_kats.json: the data of the reference's unit tests for `clean`, `gfa2fasta` and `table` (the graph edits of
unitig_graph.rs, parse_tig_numbers, the gfa2fasta texts, table's file selection, field names and value formatting, and
format_float_sigfigs), so that the oracle and the product can be checked against them without the reference's sources in this tree.
usage: python tests/golden/extract_clean_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/)"""
import ast
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def tests_of(src):
    body = src[src.index("mod tests"):]
    return {name: [" ".join(s.split()) for s in re.sub(r"//[^\n]*", "", text).split(";")]
            for name, text in re.findall(r"#\[test\]\s*fn (\w+)\(\) \{(.*?)\n    \}\n", body, re.S)}


def rust_literal(text):
    t = text.replace("vec![", "[").replace("HashSet::from(", "(").replace("Vec::<u32>::new()", "[]")
    return ast.literal_eval(t)


def graph_steps(stmts):
    """The statements of a graph test as steps: load, remove, duplicate, low_depth, merge and the asserted values."""
    steps = []
    for s in stmts:
        if not s:
            continue
        m = re.match(r"let \(mut graph, _\) = UnitigGraph::from_gfa_lines\(&get_test_gfa_(\d+)\(\)\)$", s)
        if m:
            steps.append(["load", int(m.group(1))])
            continue
        m = re.match(r"assert_eq!\(graph\.connected_components\(\), (.*)\)$", s)
        if m:
            steps.append(["components", rust_literal(m.group(1))])
            continue
        m = re.match(r"graph\.remove_unitigs_by_number\(HashSet::from\((\[.*\])\)\)$", s)
        if m:
            steps.append(["remove", rust_literal(m.group(1))])
            continue
        m = re.match(r"graph\.duplicate_unitig_by_number\(&(\d+)\)$", s)
        if m:
            steps.append(["duplicate", int(m.group(1))])
            continue
        m = re.match(r"graph\.remove_low_depth_unitigs\(([\d.]+)\)$", s)
        if m:
            steps.append(["low_depth", float(m.group(1))])
            continue
        if s == "merge_linear_paths(&mut graph, &vec![])":
            steps.append(["merge"])
            continue
        m = re.match(r"assert_eq!\(graph\.(unitigs\.len|total_length|link_count)\(\), (.*)\)$", s)
        if m:
            steps.append([{"unitigs.len": "unitigs", "total_length": "length", "link_count": "links"}[m.group(1)], rust_literal(m.group(2))])
            continue
        raise SystemExit(f"statement not understood: {s}")
    return steps


def main():
    src = os.path.join(sys.argv[1], "src")
    read = lambda f: open(os.path.join(src, f)).read()
    out = {"source": "Autocycler v0.6.1 src/ unit tests (unitig_graph.rs, clean.rs, gfa2fasta.rs, table.rs, misc.rs, metrics.rs)"}

    ug = tests_of(read("unitig_graph.rs"))
    out["graph_edits"] = {t: graph_steps(ug[t]) for t in ("test_remove_unitigs_by_number", "test_duplicate_unitig_by_number", "test_remove_low_depth_unitigs")}

    pt = " ".join(tests_of(read("clean.rs"))["test_parse_tig_numbers"])
    parse = {"error": [ast.literal_eval(x) for x in re.findall(r'parse_tig_numbers\(Some\(("[^"]*")\.to_string\(\)\)\)\s*;?\s*\}\)\.is_err\(\)', pt)],
             "ok": [[None if a == "None" else ast.literal_eval(b), rust_literal(c)]
                    for a, b, c in re.findall(r'assert_eq!\(parse_tig_numbers\((None|Some\(("[^"]*")\.to_string\(\)\))\), (vec!\[[^\]]*\]|Vec::<u32>::new\(\))\)', pt)]}
    assert len(parse["error"]) == 3 and len(parse["ok"]) == 4, parse
    out["parse_tig_numbers"] = parse

    g2f = []
    for name, stmts in tests_of(read("gfa2fasta.rs")).items():
        text = " ".join(stmts)
        n = int(re.search(r"get_test_gfa_(\d+)\(\)", text).group(1))
        body = re.search(r'assert_eq!\(contents, (".*")\)', text).group(1)
        fasta = "".join(ast.literal_eval(p) for p in re.findall(r'"(?:[^"\\]|\\.)*"', body.replace("\\ ", "")))
        g2f.append({"test": name, "fixture": n, "fasta": fasta})
    out["gfa2fasta"] = g2f

    tb = tests_of(read("table.rs"))
    def paths(s):
        return [p for p in re.findall(r'PathBuf::from\("([^"]*)"\)', s)]
    one = " ".join(tb["test_get_one_copy_yaml"])
    files = paths(re.search(r"let yaml_files = vec!\[(.*?)\]", one).group(1))
    cases = [[f, None if r == "None" else paths(r)[0]] for f, r in re.findall(r'get_one_copy_yaml\(&yaml_files, "([^"]+)"\), (None|Some\(PathBuf::from\("[^"]*"\)\))', one)]
    errors = re.findall(r'get_one_copy_yaml\(&yaml_files, "([^"]+)"\)\s*;?\s*\}\)\.is_err\(\)', one)
    out["one_copy"] = {"files": files, "found": cases, "error": errors}
    multi = " ".join(tb["test_get_multi_copy_yaml"])
    files = paths(re.search(r"let yaml_files = vec!\[(.*?)\]", multi).group(1))
    found = [[f, paths(r)] for f, r in re.findall(r'assert_eq!\(get_multi_copy_yaml\(&yaml_files, "([^"]+)"\),\s*(vec!\[.*?\]|empty_vec)\)', multi)]
    out["multi_copy"] = {"files": files, "found": found}
    pf = " ".join(tb["test_parse_fields"])
    out["parse_fields"] = {"ok": [[a, rust_literal(b)] for a, b in re.findall(r'assert_eq!\(parse_fields\("([^"]*)"\.to_string\(\)\),\s*(vec!\[.*?\])\)', pf)],
                           "error": re.findall(r'parse_fields\("([^"]*)"\.to_string\(\)\)\s*;?\s*\}\)\.is_err\(\)', pf)}
    fv = []
    for s in tb["test_format_value_simple"]:
        m = re.match(r'assert_eq!\(format_value\(&Value::(Number|String|Bool)\((.*)\), (\d+)\), "(.*)"\)$', s)
        if not m:
            continue
        kind, arg = m.group(1), m.group(2)
        if kind == "Number":
            x = re.match(r"serde_yaml::Number::from\((.*)\)", arg).group(1)
            value = float(x) if "." in x else int(x)
        elif kind == "String":
            value = ast.literal_eval(re.match(r'("[^"]*")\.to_string\(\)', arg).group(1))
        else:
            value = arg == "true"
        fv.append({"value": value, "sigfigs": int(m.group(3)), "expected": m.group(4)})
    out["format_value"] = fv
    seq = " ".join(tb["test_format_value_sequence"])
    out["format_sequence"] = {"value": [12, 1.2, "abc", True], "sigfigs": 2,
                              "expected": re.search(r'format_value\(&seq, 2\), "([^"]*)"', seq).group(1)}
    mp = " ".join(tb["test_format_value_mapping"])
    out["format_mapping"] = {"value": [[12, 1.2], ["abc", True]], "sigfigs": 2,
                             "expected": re.search(r'format_value\(&Value::Mapping\(map\), 2\), "([^"]*)"', mp).group(1)}
    assert "map.insert(v1, v2)" in mp and "map.insert(v3, v4)" in mp and "vec![v1, v2, v3, v4]" in seq

    ff = []
    for s in tests_of(read("misc.rs"))["test_format_float_sigfigs"]:
        m = re.match(r'assert_eq!\(format_float_sigfigs\((-?[\d.]+), (\d+)\), "([^"]*)"\)$', s)
        if m:
            ff.append([float(m.group(1)), int(m.group(2)), m.group(3)])
        elif s:
            raise SystemExit(f"format_float_sigfigs: statement not understood: {s}")
    out["format_float_sigfigs"] = ff

    names = {}
    for s in tests_of(read("metrics.rs"))["test_get_field_names"]:
        m = re.match(r"assert_eq!\((\w+)::get_field_names\(\), (vec!\[.*\])\)$", s)
        if m:
            names[m.group(1)] = rust_literal(m.group(2))
    assert len(names) == 6, names
    out["field_names"] = names

    assert len(g2f) == 7 and len(ff) > 50
    with open(os.path.join(HERE, "clean_kats.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(f"{len(g2f)} gfa2fasta texts, {len(ff)} format_float_sigfigs cases, {sum(len(v) for v in out['graph_edits'].values())} graph steps")


if __name__ == "__main__":
    main()
