"""Shared body of the k-mer table route tests (test_table_routes_emu.py, test_table_routes_gpu.py).

A table build takes one of three routes (pipeline.cu local_w / insert_w): the size the sampling pass estimates, a retry at the safe size
when the insert passes the probe limit, and a repeat with 32-bit side counts when a loaded 20-bit count reaches 2^19.  Each case here
is run through check_case (every output against the oracle), then built once more with AC_HOST_PROFILE's per-attempt lines captured, and
the attempts must be the ones tests/table_sizing.py predicts."""
import os
import random
import re
import subprocess
import sys
import tempfile

import cases
import oracle_lib as o
import table_sizing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALARM = 1 << 19                 # AC_SLOT_COUNT_ALARM
ATTEMPT = re.compile(r"\[device\] k-mer table attempt (\d+): capacity (\d+), side counts (\d)")
KS = [11, 31, 51, 91, 255]      # W = 1, 1, 2, 3, 8
WALK = 200_000                 # bases of the walks: 3 x the 65,536 windows above which the table is sized from the estimate


def small(rng):
    return ("a.fasta", [("c1", cases.rand_seq(rng, 3000))])


def walk_case(seed, rate, big_first=False):
    """A small random file and a large walk (tests/cases.py sampled_walk) in a file of its own."""
    rng = random.Random(seed)
    big = ("b.fasta", [("w1", cases.sampled_walk(rng, WALK, rate))])
    files = [small(rng), big]
    if big_first:
        files = [("a.fasta", big[1]), ("b.fasta", files[0][1])]
    return files


def case_list(k):
    """-> [(name, files, max occurrences of one k-mer)] for one k."""
    out = [("unsampled_walk", walk_case(k, 0.0), None),
           ("biased_walk_overflow", walk_case(k + 1, 0.003), None),       # an estimate of ~1/2 of the distinct k-mers: the insert overflows
           ("biased_walk_high_load", walk_case(k + 2, 0.008), None)]      # an estimate that leaves a load of ~0.8: long probe chains, no retry
    for occ in (ALARM - 1, ALARM, (1 << 20) + 5):
        out.append((f"homopolymer_{occ}", cases.homopolymer_case(random.Random(k + occ), occ, k, base="A" if occ & 1 else "T"), occ))
    rng = random.Random(k + 3)
    both = [small(rng), ("b.fasta", [("w1", cases.sampled_walk(rng, WALK, 0.0))]), ("c.fasta", cases.homopolymer_case(rng, (1 << 20) + 100, k)[0][1])]
    out.append(("walk_and_homopolymer", both, (1 << 20) + 100))
    return out


def expected_attempts(pred, max_occ, exact_alarm):
    """The (capacity, side counts) of every attempt, from the predicted sizes.  At exactly 2^19 occurrences the alarm rises on the
    emulation (loads never lag there) and may or may not on the GPU: None there, for either."""
    att = [(pred["estimate_cap"], 0), (pred["safe"], 0)] if pred["retry"] else [(pred["capacity"], 0)]
    if max_occ is not None and max_occ >= ALARM:
        if max_occ == ALARM and not exact_alarm:
            return None
        att.append((pred["capacity"], 1))
    return att


CHILD = """
import sys, json
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
from autocycler_b200 import api
from parity_common import check_case
import cases
lib = api.load_library(%(lib)r)
d, k = sys.argv[1], int(sys.argv[2])
files = json.load(open(d + "/files.json"))
got = check_case(lib, files, k)
for _ in range(%(repeats)d):                 # the same handle again: one build per marker
    sys.stderr.write("BUILD\\n"); sys.stderr.flush()
    got["kg"].upload()
    g = api.UnitigGraph.compress(got["kg"])
    print("CAPACITY", g.timings().table_capacity, g.timings().table_used, flush=True)
    print("SHA", __import__("hashlib").sha256(bytes(g.gfa_view())).hexdigest(), flush=True)
print("CHECKED", flush=True)
"""


def run_case(lib_path, files, k, max_occ, exact_alarm, poison=False, repeats=1):
    """check_case in a child process (the profile switch is read there), then `repeats` more builds on the same handle, each of whose
    attempts must match the prediction, with one output for all of them."""
    import json
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        count, oseqs = o.load_sequences(d, k)
        gfa, yaml, st = o.compress_dir(d, k)
        pred = table_sizing.predict([s[4] for s in oseqs], k, st.n_kmers // 2)
        json.dump(files, open(os.path.join(d, "files.json"), "w"))
        code = CHILD % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": lib_path, "repeats": repeats}
        env = {**os.environ, "AC_HOST_PROFILE": "1"}
        env.pop("AC_COUNT_ALARM", None)
        if poison:
            env["AC_EMU_POISON"] = "1"
        r = subprocess.run([sys.executable, "-c", code, d, str(k)], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and "CHECKED" in r.stdout, r.stderr[-3000:]
    caps = [tuple(map(int, l.split()[1:])) for l in r.stdout.splitlines() if l.startswith("CAPACITY")]
    shas = {l.split()[1] for l in r.stdout.splitlines() if l.startswith("SHA")}
    assert len(caps) == repeats and len(shas) == 1, (caps, shas)
    want = expected_attempts(pred, max_occ, exact_alarm)
    for cap, used in caps:
        assert (cap, used) == (pred["capacity"], pred["distinct"]), (pred, cap, used)
    for block in r.stderr.split("BUILD\n")[1:]:
        att = [(int(a), int(c), int(b)) for a, c, b in ATTEMPT.findall(block)]
        assert [a for a, _, _ in att] == list(range(len(att))), att
        if want is None:          # exactly 2^19 on the GPU: the side counts or not, the same graph (check_case passed)
            assert [(c, b) for _, c, b in att] in ([(pred["capacity"], 0)], [(pred["capacity"], 0), (pred["capacity"], 1)]), att
        else:
            assert [(c, b) for _, c, b in att] == want, (att, want, pred)
    return pred
