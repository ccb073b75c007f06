"""BASELINE.json configs[1] (8 x 4.64 Mbp, k=51) at full size through the host-emulation build: the code paths that only large
graphs take (sample-sort renumber, conflict levels on several threads, device-made work list, parallel GFA writer) against the
committed SHA-256 of the oracle's GFA.  About half a minute per run."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CODE = """
import sys, hashlib
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
from autocycler_b200 import api, synth
from parity_common import run_library
d = sys.argv[1]
synth.write_assemblies(synth.make_assemblies("cfg2"), d)
lib = api.load_library(%(lib)r)
if sys.argv[2] == "fused":           # ac_compress: simplify_structure and the GFA text by the device bodies
    kg, seqs, count = api.load_sequences(d, 51, lib=lib)
    kg.upload()
    g = api.UnitigGraph.compress(kg)
    gfa, before, after = bytes(g.gfa_view()), g.counts(), g.counts()
else:
    got = run_library(lib, d, 51)
    g, gfa, before, after = got["graph"], got["gfa"].encode(), got["before"], got["after"]
print("SHA", hashlib.sha256(gfa).hexdigest(), before.n_kmers, after.n_unitigs, after.n_links, g.timings().table_capacity)
"""


@pytest.mark.parametrize("mode,env", [("plain", {}), ("fused", {}), ("plain", {"AC_EXPAND_SERIAL": "1", "AC_HOST_CANDIDATES": "1"})],
                         ids=["default", "device_simplify_and_gfa", "serial_host"])
def test_config2_golden_under_emulation(tmp_path, mode, env):
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))["cfg2_k51"]
    code = CODE % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")}
    r = subprocess.run([sys.executable, "-c", code, str(tmp_path / "cfg2"), mode], env={**os.environ, **env}, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("SHA")][0].split()
    assert line[1] == g["sha256"]
    assert (int(line[3]), int(line[4])) == (g["unitigs_after"], g["links_after"])
    assert int(line[2]) == g["n_kmers"]
    if mode == "plain" and not env:          # the size the sizing pass's exact restatement predicts (tests/table_sizing.py)
        import oracle_lib as o
        import table_sizing
        count, oseqs = o.load_sequences(str(tmp_path / "cfg2"), 51)
        pred = table_sizing.predict([s[4] for s in oseqs], 51, g["n_kmers"] // 2)
        assert pred["capacity"] < pred["safe"] and int(line[5]) == pred["capacity"]


MULTI_CODE = """
import sys, hashlib, tempfile, os
sys.path.insert(0, %(tests)r); sys.path.insert(0, %(root)r)
from autocycler_b200 import api, synth
lib = api.load_library(%(lib)r)
with tempfile.TemporaryDirectory() as d:
    synth.write_assemblies(synth.make_assemblies("cfg5", n_assemblies=16), d)
    out = os.path.join(d, "out")
    api.compress(d, out, k_size=51, lib=lib, devices=[0, 1])
    print("SHA", hashlib.sha256(open(os.path.join(out, "input_assemblies.gfa"), "rb").read()).hexdigest())
"""


def test_config5_first_16_on_two_emulated_devices():
    """The N = 2 workload of bench.py --gpus 2 (the first 16 assemblies of BASELINE config 5, 80 Mbp) through the sharded build at full
    size — two emulated devices in one process, `autocycler compress --devices 0,1` — against the oracle's committed SHA-256; device
    buffers poisoned before every table build.  About half a minute."""
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))["cfg5_k51_n16"]
    code = MULTI_CODE % {"tests": os.path.join(ROOT, "tests"), "root": ROOT, "lib": os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so")}
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, "AC_EMU_POISON": "1"}, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-2000:]
    assert [l for l in r.stdout.splitlines() if l.startswith("SHA")][0].split()[1] == g["sha256"]
