"""The k-mer table's three routes on the H100 at the real thresholds (no AC_COUNT_ALARM): the retry after an estimate the insert
overflows, and the side counts behind the 2^19 alarm, whose exactness rests on the argument in kmer_key.h (a loaded count lags the true
one by fewer adds than the GPU holds threads).  At 2^20 + 5 occurrences and more, parity with the oracle proves that the alarm rose: a
20-bit count would have wrapped into the fingerprint and the depth would be wrong.  Run on an H100 with `pytest -m gpu`."""
import json
import os

import pytest

import oracle_lib as o
import table_routes
import table_sizing
from autocycler_b200 import api, synth
from parity_common import run_library

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "autocycler_b200", "libautocycler_gpu.so")


@pytest.fixture(scope="module")
def lib():
    lib = api.load_library()
    assert b"sm_90a" in lib.ac_version()
    return lib


@pytest.mark.parametrize("k", table_routes.KS)
@pytest.mark.parametrize("name", [c[0] for c in table_routes.case_list(11)])
def test_every_route_at_every_key_width(lib, name, k):
    """Each case through check_case, then three more builds on the same handle: the same bytes each time, and the attempts predicted."""
    files, max_occ = next((f, m) for n, f, m in table_routes.case_list(k) if n == name)
    table_routes.run_case(LIB, files, k, max_occ, exact_alarm=False, repeats=3)


def test_homopolymer_of_2_2_million_occurrences(lib):
    import random
    import cases
    files = cases.homopolymer_case(random.Random(22), 2_200_000, 51)
    table_routes.run_case(LIB, files, 51, 2_200_000, exact_alarm=False)


def test_sizing_pass_on_config2(lib, tmp_path):
    """cfg2's table capacity (55.7 M slots at the safe size) is what the sizing pass's exact restatement predicts."""
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))["cfg2_k51"]
    d = str(tmp_path / "cfg2")
    synth.write_assemblies(synth.make_assemblies("cfg2"), d)
    count, oseqs = o.load_sequences(d, 51)
    pred = table_sizing.predict([s[4] for s in oseqs], 51, g["n_kmers"] // 2)
    got = run_library(lib, d, 51)
    assert got["before"].n_kmers == g["n_kmers"]
    assert pred["estimate_cap"] is not None and pred["capacity"] < pred["safe"]
    assert got["graph"].timings().table_capacity == pred["capacity"]
