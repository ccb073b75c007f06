"""Writes tests/golden/cluster_kats.json: the data of the reference's cluster.rs unit tests (cluster.rs:915-1273: UPGMA matrices and
Newick strings, the two test trees, and the inputs and expected results of the clustering, QC and parsing helpers), as a list of cases,
each a start state and a list of operations with their expected results, so that the oracle and the product can be checked against
them without the reference's sources in this tree.  test_tree_1 / test_tree_2 also become ultrametric distance matrices
(d(i, j) = twice the distance of the pair's lowest common ancestor), whose UPGMA tree the tests check is that tree.
usage: python tests/golden/extract_cluster_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/cluster.rs)"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SEQ = re.compile(r'Sequence::new_with_seq\((\d+), "[^"]*"\.to_string\(\), "([^"]*)"\.to_string\(\), "([^"]*)"\.to_string\(\), (\d+), \d+\)')


def ints(text):
    return [int(x) for x in re.findall(r"-?\d+", text)]


def lists(text):   # "vec![vec![1, 2], vec![3]]" / "vec![1, 2]" / "&[1, 2]"
    inner = re.findall(r"\[([^\[\]]*)\]", text)
    return [ints(x) for x in inner]


def parse_tree(body):
    nodes = {}
    for name, fields in re.findall(r"let (n\d+) = TreeNode \{([^}]*)\}", body):
        nodes[name] = fields
    root = re.search(r"\n\s*TreeNode \{([^}]*)\}\s*$", body.rstrip()).group(1)
    out = []
    for fields in list(nodes.values()) + [root]:
        f = dict(re.findall(r"(\w+): ([^,]+)", fields))
        if "left" in f:
            l = int(re.search(r"n(\d+)", f["left"]).group(1)); r = int(re.search(r"n(\d+)", f["right"]).group(1))
            out.append([int(f["id"]), ids_of(nodes, l), ids_of(nodes, r), float(f["distance"].strip())])
    return out


def ids_of(nodes, k):
    return int(re.search(r"id: (\d+)", nodes[f"n{k}"]).group(1))


def ultrametric(tree):
    left = {n: l for n, l, r, d in tree}
    right = {n: r for n, l, r, d in tree}
    dist = {n: d for n, l, r, d in tree}

    def tips(u):
        return [u] if u not in left else tips(left[u]) + tips(right[u])
    root = max(left)
    ids = sorted(tips(root))
    m = [[0.0] * len(ids) for _ in ids]
    for n in left:
        for a in tips(left[n]):
            for b in tips(right[n]):
                m[ids.index(a)][ids.index(b)] = m[ids.index(b)][ids.index(a)] = 2.0 * dist[n]
    return ids, m


def statements(body):
    body = re.sub(r"//[^\n]*", "", body)
    body = re.sub(r"assert!\(panic::catch_unwind\(\|\| \{\s*(.*?);\s*\}\)\.is_err\(\)\);", r"PANICS(\1);", body, flags=re.S)
    body = re.sub(r"for (\w+) in (\d+)\.\.=(\d+)\s*\{(.*?)\}",
                  lambda m: "".join(re.sub(rf"\b{m.group(1)}\b", str(i), m.group(4)) for i in range(int(m.group(2)), int(m.group(3)) + 1)),
                  body, flags=re.S)
    return [" ".join(s.split()) for s in body.split(";") if s.strip()]


def extract(src):
    tests = src[src.index("mod tests"):]
    trees = {name: parse_tree(body) for name, body in re.findall(r"fn (test_tree_\d)\(\) -> TreeNode \{(.*?)\n    \}\n", tests, re.S)}
    cases = []
    for name, body in re.findall(r"#\[test\]\s*fn (\w+)\(\) \{(.*?)\n    \}\n", tests, re.S):
        case = {"test": name, "ops": []}
        ops = case["ops"]
        for st in statements(body):
            panics = st.startswith("PANICS(")
            if st.startswith("let tree = "):
                t = re.search(r"(test_tree_\d)", st).group(1)
                ops.append(["tree", t])
            elif "let distances = HashMap::from_iter" in st:
                pairs = re.findall(r"\(\((\d+), (\d+)\), ([\d.]+)\)", st)
                ids = sorted({int(a) for a, _, _ in pairs})
                m = [[0.0] * len(ids) for _ in ids]
                for a, b, v in pairs:
                    m[ids.index(int(a))][ids.index(int(b))] = float(v)
                case["matrix"], case["ids"] = m, ids
            elif "Sequence::new_with_seq" in st and ("let sequences" in st or "let mut sequences" in st):
                ops.append(["sequences", [[int(i), fn, hd, int(ln)] for i, fn, hd, ln in SEQ.findall(st)]])
            elif re.match(r"let mut seq_\d+ = Sequence", st):
                i, fn, hd, ln = SEQ.search(st).groups()
                case.setdefault("sequences", []).append([int(i), fn, hd, int(ln)])
            elif re.match(r"seq_\d+\.cluster = \d+", st):
                k, c = ints(st)
                ops.append(["set_cluster", k - 1, c])
            elif re.match(r"sequences\[\d+\]\.cluster = \d+", st):
                k, c = ints(st)
                ops.append(["set_cluster", k, c])
            elif st.startswith("let sequences = vec![seq_"):
                pass
            elif "upgma(&distances" in st:
                ops.append(["upgma"])
            elif st.startswith("normalise_tree"):
                ops.append(["normalise"])
            elif "assert_almost_eq(root.distance" in st:
                ops.append(["root_distance", float(st.split(",")[1])])
            elif "assert_eq!(newick_string" in st:
                ops.append(["newick", re.search(r'"([^"]*)"', st).group(1)])
            elif "automatic_clustering" in st:
                ops.append(["automatic", float(re.search(r"automatic_clustering\(([\d.]+)\)", st).group(1)), lists(st)[-1]])
            elif "manual_clustering" in st:
                a = re.search(r"manual_clustering\(([\d.]+), &\[([^\]]*)\]\)", st)
                ops.append(["manual", float(a.group(1)), ints(a.group(2)), lists(st)[-1]])
            elif "has_manual_child" in st:
                ops.append(["has_manual_child", lists(st)[0], not st.startswith("assert!(!")])
            elif "check_consistency" in st:
                ops.append(["consistency", lists(st)[0], not panics])
            elif "check_complete_coverage" in st:
                ops.append(["coverage", lists(st)[0], not panics])
            elif "max_pairwise_distance" in st:
                a = re.search(r"max_pairwise_distance\((\d+)\), (-?[\d.]+)", st)
                ops.append(["max_pairwise_distance", int(a.group(1)), float(a.group(2))])
            elif "get_tips" in st:
                a = re.search(r"get_tips\((\d+)\), vec!\[([^\]]*)\]", st)
                ops.append(["get_tips", int(a.group(1)), ints(a.group(2))])
            elif "split_clusters" in st:
                arg, exp = st.split("]),", 1)
                ops.append(["split", lists(arg + "]")[0], lists(exp[exp.index("vec![") + 5:-2] if "vec![vec!" in exp else "")])
            elif "find_node" in st:
                a = ints(st)
                ops.append(["find_node", a[0], a[1] if "is_none" not in st else None])
            elif "parse_manual_clusters" in st:
                if panics:
                    ops.append(["parse_manual", re.search(r'Some\("(.*?)"\.to_string', st).group(1), None])
                elif "None" in st.split(")")[0]:
                    ops.append(["parse_manual", None, []])
                else:
                    a = re.search(r'Some\("(.*?)"\.to_string\(\)\)\), vec!\[([^\]]*)\]', st)
                    ops.append(["parse_manual", a.group(1), ints(a.group(2))])
            elif "cluster_assembly_count" in st:
                a = re.search(r"cluster_assembly_count\(&sequences, (\d+)\), (\d+)", st)
                ops.append(["cluster_assembly_count", int(a.group(1)), int(a.group(2))])
            elif "set_min_assemblies" in st:
                a = re.search(r"set_min_assemblies\((None|Some\((\d+)\)), &sequences\), (\d+)", st)
                ops.append(["set_min_assemblies", int(a.group(2)) if a.group(2) else None, int(a.group(3))])
            elif st == "sequences.pop()":
                ops.append(["pop"])
            elif st.startswith("sequences.truncate"):
                ops.append(["truncate", ints(st)[0]])
            elif st.startswith("reorder_clusters"):
                ops.append(["reorder"])
            elif re.match(r"assert_eq!\(sequences\[\d+\]\.cluster, \d+\)", st):
                k, c = ints(st)
                ops.append(["cluster_of", k, c])
            elif "get_assembly_count" in st:
                ops.append(["assembly_count", ints(st)[-1]])
            elif "get_max_cluster" in st:
                ops.append(["max_cluster", ints(st)[-1]])
            elif st.startswith(("let index", "let newick_string", "let mut root", "let root")):
                pass
            else:
                raise SystemExit(f"{name}: statement not understood: {st}")
        cases.append(case)
    out = {"source": "rrwick/Autocycler v0.6.1, src/cluster.rs:915-1273", "trees": {}, "cases": cases}
    for t, nodes in sorted(trees.items()):
        ids, m = ultrametric(nodes)
        out["trees"][t] = {"nodes": sorted(nodes), "ids": ids, "matrix": m}
    return out


def main():
    src = open(os.path.join(sys.argv[1], "src", "cluster.rs")).read()
    with open(os.path.join(HERE, "cluster_kats.json"), "w") as f:
        json.dump(extract(src), f, indent=None)
        f.write("\n")


if __name__ == "__main__":
    main()
