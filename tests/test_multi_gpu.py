"""The N > 1 path on real GPUs, inside the `-m gpu` suite: spawns one process per GPU (torchrun, NCCL) when the box shows at least two
devices and checks the sharded build against the oracle (tests/multi_gpu_check.py).  On a one-GPU box the test is skipped; the host
logic of the same path is covered on CPU by tests/test_multi_rank_gloo.py."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _devices():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_build_matches_the_oracle(world):
    n = _devices()
    if n < world:
        pytest.skip(f"{n} CUDA device(s) visible, {world} needed")
    env = dict(os.environ)
    if world > 2:
        env["AC_MULTI_CHECK_QUICK"] = "1"      # cfg2 at full size once (world 2) is enough
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(29650 + world), os.path.join(ROOT, "tests", "multi_gpu_check.py")],
                       capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0 and "MULTI_GPU_CHECK OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


@pytest.mark.parametrize("n_devices", [2, 4, 8])
def test_several_devices_in_one_process(tmp_path, n_devices):
    """ac_config.n_devices: ONE process drives the GPUs, the peers' k-mer buckets and occurrences are read in place over NVLink (peer
    access), `autocycler compress --devices` shards by file — against the oracle on a medium input and, at 2 devices, cfg2's golden."""
    import hashlib
    import json
    n = _devices()
    if n < n_devices:
        pytest.skip(f"{n} CUDA device(s) visible, {n_devices} needed")
    sys.path.insert(0, ROOT)
    import oracle_lib as o
    from autocycler_b200 import api, synth
    devices = list(range(n_devices))
    d = str(tmp_path / "in")
    synth.write_assemblies(synth.make_assemblies("m", n_assemblies=6, replicon_lengths=[400_000, 22_000, 8_000, 3_000], seed=99), d)
    expected, yaml, st = o.compress_dir(d, 51)
    out = str(tmp_path / "out")
    api.compress(d, out, k_size=51, devices=devices)
    assert open(os.path.join(out, "input_assemblies.gfa")).read() == expected
    assert open(os.path.join(out, "input_assemblies.yaml")).read() == yaml
    exe = os.path.join(ROOT, "autocycler_b200", "bin", "autocycler")
    out2 = str(tmp_path / "out2")
    r = subprocess.run([exe, "compress", "-i", d, "-a", out2, "--devices", ",".join(map(str, devices))], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert open(os.path.join(out2, "input_assemblies.gfa")).read() == expected
    if n_devices == 2:
        g = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))["cfg2_k51"]
        d2 = str(tmp_path / "cfg2"); synth.write_assemblies(synth.make_assemblies("cfg2"), d2)
        kg, seqs, count = api.load_sequences(d2, 51)
        kg2 = api.KmerGraph(51, devices=devices)
        kg2.add_sequences(seqs, count)
        graph = api.UnitigGraph.compress(kg2)
        assert hashlib.sha256(bytes(graph.gfa_view())).hexdigest() == g["sha256"]


@pytest.mark.parametrize("n_devices", [2, 3])
@pytest.mark.parametrize("big_first", [False, True])
def test_several_devices_survive_a_low_estimate(tmp_path, n_devices, big_first):
    """Imbalanced shards: a small file and a large walk the size estimate cannot see.  The rank holding only the small file overflows
    its table while merging, builds it again at the safe size and merges the same records again: the oracle's bytes."""
    n = _devices()
    if n < n_devices:
        pytest.skip(f"{n} CUDA device(s) visible, {n_devices} needed")
    sys.path.insert(0, ROOT)
    import cases
    import oracle_lib as o
    import table_routes
    from autocycler_b200 import api
    d = str(tmp_path / "in")
    cases.write_case(table_routes.walk_case(77, 0.0, big_first=big_first), d)
    expected, yaml, st = o.compress_dir(d, 51)
    out = str(tmp_path / "out")
    api.compress(d, out, k_size=51, devices=list(range(n_devices)))
    assert open(os.path.join(out, "input_assemblies.gfa")).read() == expected
