"""Memory-safety check of the CUDA sources on the host SIMT emulator built with AddressSanitizer (tests/emu,
build_emu.build(asan=True)): "device" buffers are exact-size heap blocks and the unused tail of the dynamic shared memory
window is poisoned, so any out-of-bounds global or shared access of a kernel aborts with the source line -- the CPU-side
stand-in for compute-sanitizer's memcheck.  Runs in a subprocess (ASan must be preloaded into the interpreter)."""
import os
import platform
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")

SCRIPT = """
import sys
sys.path.insert(0, %r)
import dada2_b200.api as api
api._LIBPATH = %r; api._LIB = None
import tests.test_gpu_parity as T
T.test_pair_corpus_kernels_match_reference()
for name in %r:
    T.test_e2e_matches_reference_golden(name, None)
T.test_error_paths()
print('ASAN RUN OK')
"""


def _preload():
    """libasan plus libstdc++ (the interpreter does not link libstdc++; without it ASan cannot intercept __cxa_throw)."""
    for cxx in (os.environ.get("CXX", "g++"), "/usr/bin/g++"):
        try:
            libs = [subprocess.run([cxx, "-print-file-name=" + n], capture_output=True, text=True).stdout.strip()
                    for n in ("libasan.so", "libstdc++.so.6")]
        except OSError:
            continue
        if all(os.path.isabs(f) and os.path.exists(f) for f in libs):
            return " ".join(os.path.realpath(f) for f in libs)
    return None


@pytest.mark.parametrize("flags", [{}, {"DADA2B_FALLBACK": "1", "DADA2B_TAIL_SMEM_CLUSTERS": "0"}], ids=["default", "fallback_kernels"])
def test_kernels_are_memory_clean_under_asan(flags):
    asan = _preload()
    if asan is None:
        pytest.skip("libasan not found")
    import build_emu
    lib = build_emu.build(asan=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", **flags)
    names = ["syn500_usequals0", "syn600_band0"] if os.environ.get("DADA2B_EMU_FULL") else ["syn500_usequals0"]
    out = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, lib, names)], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert "AddressSanitizer" not in out.stderr, out.stderr[-4000:]
    assert out.returncode == 0 and "ASAN RUN OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]


SCRIPT_F = """
import sys
sys.path.insert(0, %r)
import dada2_b200.api as api
api._LIBPATH = %r; api._LIB = None
from tests import bimera_cases as B, merge_cases as M, derep_cases as D
B.check_pairs(B.product_pair_fn, shifts=[16, -1], limit=40)
B.check_pairs_vs_oracle(B.product_pair_fn, shifts=(16, 50), npairs=12)
B.check_table("t40_one_sample", B.product_table_fn, [0, 1])
B.check_is_bimera("t40_one_sample", B.product_denovo_fn)
M.check(M.product_fn, opt_ids=[0, 2, 3, 4], limit=25, maxlen=160)
D.check_all(D.product_fn, sizes=(1200,))
print('ASAN RUN OK')
"""


@pytest.mark.parametrize("flags", [{"DADA2B_BIMFWD": "0"}, {"DADA2B_BIMFWD": "1"}, {}], ids=["traceback", "bimfwd", "default_bimfwd16"])
def test_bimera_and_merge_kernels_are_memory_clean_under_asan(flags):
    """dd_bimera.cu / dd_bimfwd.cu / dd_merge.cu / dd_derep.cu (SURVEY.md 8(f3), (f4), (f1)) under the same memcheck stand-in."""
    asan = _preload()
    if asan is None:
        pytest.skip("libasan not found")
    import build_emu
    lib = build_emu.build(asan=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", **flags)
    out = subprocess.run([sys.executable, "-c", SCRIPT_F % (ROOT, lib)], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert "AddressSanitizer" not in out.stderr, out.stderr[-4000:]
    assert out.returncode == 0 and "ASAN RUN OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
