"""Generates tests/golden/trim_goldens.json: SHA-256 of the trim oracle's 2_trimmed.gfa (tests/trim_oracle.py) for
bench_trim.py and the GPU tests.  The input is what `autocycler cluster` writes as 1_untrimmed.gfa for a one-cluster genome: the config's compress
GFA (C++ oracle) through merge_linear_paths.  Settings are the trim defaults (--min_identity 0.75 --mad 5.0) at each --max_unitigs.
Run in the build container:  python tests/golden/make_trim_goldens.py cfg2 5000 12000   (about three minutes on one core)"""
import hashlib
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import oracle_lib as o  # noqa: E402
import trim_oracle  # noqa: E402
from autocycler_b200 import synth  # noqa: E402

path = os.path.join(HERE, "trim_goldens.json")
name, windows = sys.argv[1], [int(x) for x in sys.argv[2:]] or [5000]
with tempfile.TemporaryDirectory() as d:
    synth.write_assemblies(synth.make_assemblies(name), d)
    gfa, _, _ = o.compress_dir(d, 51, threads=8)
untrimmed = o.gfa_merge_linear_paths(gfa, use_paths=True, renumber=False)
for mu in windows:
    t = time.time()
    stats = {}
    trimmed, yaml = trim_oracle.trim_gfa(untrimmed, 0.75, mu, 5.0, stats=stats)
    entry = dict(sha256=hashlib.sha256(trimmed.encode()).hexdigest(), gfa_bytes=len(trimmed), yaml=yaml,
                 untrimmed_sha256=hashlib.sha256(untrimmed.encode()).hexdigest(), oracle_seconds=round(time.time() - t, 1))
    print(mu, entry, flush=True)
    goldens = json.load(open(path)) if os.path.exists(path) else {}
    goldens[f"{name}_k51_trim_mu{mu}"] = entry
    json.dump(goldens, open(path, "w"), indent=1, sort_keys=True)
