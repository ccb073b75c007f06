"""Writes tests/golden/dotplot_kats.json: the data of the reference's dotplot.rs unit tests (test_get_all_kmer_positions: a sequence,
k and the expected forward / reverse k-mer positions; test_between_seq_gap: arguments and expected values), so that the oracle and the
product can be checked against them without the reference's sources in this tree.
usage: python tests/golden/extract_dotplot_kats.py <reference checkout>   (an Autocycler v0.6.1 checkout: src/dotplot.rs)"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def extract(src):
    tests = src[src.index("mod tests"):]
    body = tests[tests.index("fn test_get_all_kmer_positions"):tests.index("fn test_between_seq_gap")]
    seq = re.search(r'let seq = b"([ACGT]+)"', body).group(1)
    k = int(re.search(r"get_all_kmer_positions\((\d+),", body).group(1))
    fwd_part = body[body.index("expected_forward"):body.index("expected_reverse")]
    rev_part = body[body.index("expected_reverse"):body.index("let kmers")]
    entry = r'map\.insert\(&b"([ACGT]+)"\[\.\.\], vec!\[([\d, ]*)\]\)'
    as_map = lambda part: {m: [int(x) for x in v.split(",") if x.strip()] for m, v in re.findall(entry, part)}
    gap = tests[tests.index("fn test_between_seq_gap"):]
    gaps = [{"gap": float(a), "max_total_gap": float(b), "seq_count": int(c), "expected": float(e)}
            for a, b, c, e in re.findall(r"between_seq_gap\(([\d.]+), ([\d.]+), (\d+)\), ([\d.]+)", gap)]
    return {"kmer_positions": [{"seq": seq, "k": k, "forward": as_map(fwd_part), "reverse": as_map(rev_part)}], "between_seq_gap": gaps}


def main():
    src = open(os.path.join(sys.argv[1], "src", "dotplot.rs")).read()
    out = extract(src)
    out["source"] = "Autocycler v0.6.1 src/dotplot.rs tests (test_get_all_kmer_positions, test_between_seq_gap)"
    json.dump(out, open(os.path.join(HERE, "dotplot_kats.json"), "w"), indent=1, sort_keys=True)
    print(len(out["kmer_positions"][0]["forward"]), "forward k-mers,", len(out["between_seq_gap"]), "gap cases")


if __name__ == "__main__":
    main()
