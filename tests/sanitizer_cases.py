"""Driver of tests/run_sanitizers.sh: parity cases through a sanitizer build of the emulation library.
usage: python tests/sanitizer_cases.py <library.so> <seeds per k>"""
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import cases  # noqa: E402
import subsample_edges  # noqa: E402
import subsample_oracle  # noqa: E402
from autocycler_b200 import api  # noqa: E402
from parity_common import check_case  # noqa: E402

lib = api.load_library(sys.argv[1])
n = 0
for k in (3, 5, 9, 31, 51, 65, 91, 127):
    for seed in range(int(sys.argv[2])):
        check_case(lib, cases.random_case(9000 * k + seed, k), k)
        n += 1
print("cases", n, "OK")

# subsample with every read in every sample and no final newline: each sample's bytes of a window are that window's records as read
# plus one, the size gather() gives its output buffers; one window, then many
with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, "r.fq")
    gsize, depth, data = subsample_edges.one_byte_case(path)
    for w in (None, "700"):
        os.environ.pop("AC_SUBSAMPLE_WINDOW", None)
        if w:
            os.environ["AC_SUBSAMPLE_WINDOW"] = w
        out = os.path.join(d, f"out_{w}")
        info = api.subsample(path, out, gsize, 4, depth, 3, lib=lib)
        for f, want in subsample_oracle.subsample(path, gsize, 4, depth, 3).items():
            assert open(os.path.join(out, f), "rb").read() == want, (w, f)
        assert info["reads_per_subset"] == 30 and (info["windows"] == 1) == (w is None)
        assert open(os.path.join(out, "sample_01.fastq"), "rb").read() == data + b"\n"
    os.environ.pop("AC_SUBSAMPLE_WINDOW", None)
print("subsample one-byte growth OK")
