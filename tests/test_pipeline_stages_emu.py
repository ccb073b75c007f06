"""The compress pipeline's stage order, through the C ABI on the host-emulation build (tests/emu): a multi-GPU stage called before
the stage it needs is AC_EINVAL with a message that names the missing stage, and the handle stays usable."""
import ctypes as C
import os
import subprocess

import pytest

from autocycler_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -1
K = 9


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "autocycler_b200", "csrc"), "emu"], check=True)
    return api.load_library(os.path.join(ROOT, "tests", "emu", "libautocycler_emu.so"))


def _uploaded(emu):
    seqs = [api.Sequence.new_with_seq(1, "ACGTTGCATGCCATAGGACTTAGCAGGTACCATGAC", "a.fasta", "a1", 36, K // 2),
            api.Sequence.new_with_seq(2, "TTGCATGCCATAGGACTTAGCAGGTACCATGACGGA", "b.fasta", "b1", 36, K // 2)]
    kg = api.KmerGraph(K, lib=emu)
    kg.add_sequences(seqs, 2)
    return kg


def _expect(h, rc, message):
    assert rc == EINVAL
    assert h.lib.ac_last_error(h.ptr).decode() == message


@pytest.mark.parametrize("call, message", [
    ("ac_runs_local", "build_local must precede runs_local"),
    ("ac_entries_count", "build_local must precede the entry export"),
    ("ac_build_finish", "runs_local must precede finish"),
    ("ac_path_lines_render", "runs_local must precede render_path_lines"),
])
def test_after_upload(emu, call, message):
    h = _uploaded(emu)._h
    n = C.c_uint64(0)
    rc = {"ac_runs_local": lambda: emu.ac_runs_local(h.ptr, C.byref(n)),
          "ac_entries_count": lambda: emu.ac_entries_count(h.ptr, C.byref(n)),
          "ac_build_finish": lambda: emu.ac_build_finish(h.ptr),
          "ac_path_lines_render": lambda: emu.ac_path_lines_render(h.ptr, None, 0)}[call]()
    _expect(h, rc, message)
    h.check(emu.ac_build(h.ptr))          # nothing of the refused call is left behind


def test_runs_export_after_build_local(emu):
    h = _uploaded(emu)._h
    h.check(emu.ac_build_local(h.ptr, 0, 2, 0))
    dst = (C.c_uint8 * 4096)()
    _expect(h, emu.ac_runs_export(h.ptr, dst, 256), "runs_local must precede export_runs")


def test_path_tokens_export_after_compress(emu):
    h = _uploaded(emu)._h
    h.check(emu.ac_compress(h.ptr))
    dst = (C.c_uint32 * 1024)()
    counts = (C.c_uint64 * 1)(0)
    _expect(h, emu.ac_path_tokens_export(h.ptr, dst, 1024, counts, 1), "export_path_tokens follows a finish with split path lines")
