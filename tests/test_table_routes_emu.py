"""The k-mer table's three routes (estimated size, retry at the safe size, 32-bit side counts) on the host-emulation build: the capacity
against tests/table_sizing.py's exact restatement of the sizing pass, the attempts each build makes, and every output against the oracle.
The sharded build must survive an estimate that its own k-mers fit and the union does not."""
import os
import random
import subprocess
import sys

import pytest

import cases
import oracle_lib as o
import table_routes
import table_sizing
from autocycler_b200 import api, synth
from parity_common import run_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")
KS = table_routes.KS


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(EMU)


def _capacity(lib, d, k):
    count, oseqs = o.load_sequences(d, k)
    expected, yaml, st = o.compress_dir(d, k)
    got = run_library(lib, d, k)
    assert got["gfa"] == expected
    return got["graph"].timings().table_capacity, table_sizing.predict([s[4] for s in oseqs], k, st.n_kmers // 2)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", [c[0] for c in table_routes.case_list(11)])
def test_every_route_at_every_key_width(emu, name, k):
    files, max_occ = next((f, m) for n, f, m in table_routes.case_list(k) if n == name)
    table_routes.run_case(EMU, files, k, max_occ, exact_alarm=True, poison=name == "walk_and_homopolymer")


def test_sizing_pass_on_config1(emu, tmp_path):
    d = str(tmp_path / "cfg1")
    synth.write_assemblies(synth.make_assemblies("cfg1"), d)
    cap, pred = _capacity(emu, d, 51)
    assert pred["estimate_cap"] is not None and not pred["retry"]
    assert cap == pred["capacity"]


@pytest.mark.parametrize("k", [31, 51, 91])
def test_sizing_pass_on_the_medium_input(emu, tmp_path, k):
    d = str(tmp_path / "m")
    synth.write_assemblies(synth.make_assemblies("m", n_assemblies=6, replicon_lengths=[400_000, 22_000, 8_000, 3_000], seed=99), d)
    cap, pred = _capacity(emu, d, k)
    assert pred["estimate_cap"] is not None and pred["capacity"] < pred["safe"]
    assert cap == pred["capacity"]


@pytest.mark.parametrize("n", [65536, 65537])
def test_sizing_pass_starts_above_65536_windows(emu, n):
    """An unsampled walk of exactly n windows: at 65,536 the table takes the safe size at once, at 65,537 the sizing pass runs, sees
    nothing and the insert overflows its estimate."""
    files = [("a.fasta", [("c1", cases.sampled_walk(random.Random(n), n))])]
    pred = table_routes.run_case(EMU, files, 51, None, exact_alarm=True)
    assert (pred["estimate_cap"] is None) == (n == 65536) and pred["retry"] == (n == 65537)


SHARDED = """
import sys
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
import tempfile, os
import oracle_lib as o, table_routes, cases
from autocycler_b200 import api
lib = api.load_library(%(lib)r)
n_devices = int(sys.argv[1])
for big_first in (False, True):
    files = table_routes.walk_case(77, 0.0, big_first=big_first)
    with tempfile.TemporaryDirectory() as d:
        cases.write_case(files, d)
        expected, yaml, st = o.compress_dir(d, 51)
        count, oseqs = o.load_sequences(d, 51)
        seqs = [api.Sequence(t[0], t[4], t[1], t[2], t[3]) for t in oseqs]
        kg = api.KmerGraph(51, lib=lib, devices=list(range(n_devices)))
        kg.add_sequences(seqs, count)
        g = api.UnitigGraph.compress(kg)
        assert bytes(g.gfa_view()).decode() == expected, big_first
        out = os.path.join(d, "out")
        api.compress(d, out, k_size=51, lib=lib, devices=list(range(n_devices)))
        assert open(os.path.join(out, "input_assemblies.gfa")).read() == expected
print("SAME AS THE ORACLE")
"""


def _sharded(n_devices, lib):
    code = SHARDED % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": lib}
    return subprocess.run([sys.executable, "-c", code, str(n_devices)], env={**os.environ, "AC_EMU_POISON": "1", "AC_HOST_PROFILE": "1"},
                          capture_output=True, text=True, timeout=1200)


@pytest.mark.parametrize("n_devices", [2, 3, 5])
def test_sharded_build_survives_a_low_estimate(emu, n_devices):
    """One small file and one large unsampled walk, the walk first and last: the rank holding only the small file keeps the table its
    own k-mers fit, and the walk's merged entries overflow it.  That rank builds its table again at the safe size and merges the same
    records again: the same bytes as the oracle (buffers poisoned before every build and every attempt)."""
    r = _sharded(n_devices, EMU)
    assert r.returncode == 0 and "SAME AS THE ORACLE" in r.stdout, r.stderr[-3000:]
    safe = table_sizing.predict(["." * 25 + s + "." * 25 for _, recs in table_routes.walk_case(77, 0.0) for _, s in recs], 51, 1)["safe"]
    assert f"k-mer table attempt 1: capacity {safe}, side counts 0" in r.stderr


SIDE = """
import sys
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
import random, tempfile
import oracle_lib as o, cases
from autocycler_b200 import api
lib = api.load_library(%(lib)r)
rng = random.Random(5)
run = lambda n: cases.rand_seq(rng, 200) + "G" + "A" * (n + 10) + "G" + cases.rand_seq(rng, 200)
files = [("a.fasta", [("c1", run(int(sys.argv[1])))]), ("b.fasta", [("c1", run(int(sys.argv[2])))])]
with tempfile.TemporaryDirectory() as d:
    cases.write_case(files, d)
    count, oseqs = o.load_sequences(d, 11)
seqs = [api.Sequence(t[0], t[4], t[1], t[2], t[3]) for t in oseqs]
kg = api.KmerGraph(11, lib=lib, devices=[0, 1])
kg.add_sequences(seqs, count)
try:
    api.UnitigGraph.compress(kg)
except api.AutocyclerGpuError as e:
    print("ERROR", e)
"""


@pytest.mark.parametrize("a,b", [(600, 600), (1200, 100)], ids=["only_the_sum_reaches_it", "one_rank_reaches_it"])
def test_sharded_side_counts_are_refused(emu, a, b):
    """A k-mer whose count reaches the alarm across the ranks is not supported by the sharded build (the count alarm lowered to 1000):
    the build says so instead of returning a graph with a wrong depth."""
    code = SIDE % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": EMU}
    r = subprocess.run([sys.executable, "-c", code, str(a), str(b)], env={**os.environ, "AC_COUNT_ALARM": "1000"}, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "ERROR" in r.stdout and "a k-mer occurs more than 524287 times across the ranks: not supported by the multi-GPU exchange" in r.stdout, r.stdout
