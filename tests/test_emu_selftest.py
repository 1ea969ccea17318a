"""Self-test of the host SIMT emulator (tests/emu): the collectives behave like the hardware's, and the scheduling knob
(CUEMU_SCHED) exposes a missing __syncwarp() -- the property that makes schedule-invariance of the real kernels a
meaningful check."""
import os
import platform
import re
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
sys.path.insert(0, EMU)

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture(scope="module")
def selftest_bin():
    import build_emu
    os.makedirs(build_emu.OUT, exist_ok=True)
    cpp = os.path.join(build_emu.OUT, "selftest.emu.cpp")
    with open(os.path.join(EMU, "selftest.cu")) as f:
        body = build_emu.transform(f.read())
    with open(cpp, "w") as f:
        f.write(body)
    exe = os.path.join(build_emu.OUT, "selftest")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O1", "-g1", "-std=c++17", "-I", os.path.join(EMU, "stub"), "-include",
                           os.path.join(EMU, "cuda_emu.h"), cpp, os.path.join(EMU, "cuda_emu.cpp"), "-o", exe, "-ldl", "-pthread"])
    return exe


def _run(exe, sched):
    env = dict(os.environ)
    env.pop("CUEMU_SCHED", None)
    if sched:
        env["CUEMU_SCHED"] = str(sched)
    out = subprocess.run([exe], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "collectives bad=0" in out.stdout
    return int(re.search(r"missing_syncwarp stale=(\d+)", out.stdout).group(1))


def test_collectives_under_every_schedule_and_missing_syncwarp_is_exposed(selftest_bin):
    stale = {s: _run(selftest_bin, s) for s in (0, 1, 5, 11)}
    assert stale[0] == 31         # thread order: every lane but the last reads a slot its neighbour has not written yet
    assert stale[1] == 1          # reverse order: only the lane that runs first reads a stale slot
    assert len(set(stale.values())) > 2      # random orders land in between: the bug shows as schedule dependence


@pytest.mark.parametrize("sched", [7])
def test_real_kernels_are_schedule_invariant(sched):
    """One e2e golden with every experimental path on, under a random thread schedule (CUEMU_SCHED=1 reverses it) (own process: the
    emulator reads CUEMU_SCHED once)."""
    import build_emu
    lib = build_emu.build()
    script = (
        "import sys; sys.path.insert(0, %r)\n"
        "import dada2_b200.api as api\n"
        "api._LIBPATH = %r; api._LIB = None\n"
        "import tests.test_gpu_parity as T\n"
        "T.test_e2e_matches_reference_golden('syn800_default', None)\n"
        "T.test_pair_corpus_kernels_match_reference()\n"
        "print('SCHED OK')\n") % (os.path.dirname(HERE), lib)
    env = dict(os.environ, CUEMU_SCHED=str(sched))
    out = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600, cwd=os.path.dirname(HERE))
    assert out.returncode == 0 and "SCHED OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]


@pytest.mark.parametrize("sched,bimfwd", [(1, "0"), (7, "1"), (5, "2")])
def test_new_kernels_are_schedule_invariant(sched, bimfwd):
    """dd_bimera.cu / dd_bimfwd.cu / dd_merge.cu / dd_derep.cu under a reversed (1) and a pseudo-random (7) thread schedule: a
    missing __syncwarp() / __syncthreads() between a shared-memory (or scratch) write and its reader would show here."""
    import build_emu
    lib = build_emu.build()
    script = (
        "import sys; sys.path.insert(0, %r)\n"
        "import dada2_b200.api as api\n"
        "api._LIBPATH = %r; api._LIB = None\n"
        "from tests import bimera_cases as B, merge_cases as M, derep_cases as D\n"
        "B.check_pairs(B.product_pair_fn, shifts=[16], limit=40)\n"
        "B.check_pairs_vs_oracle(B.product_pair_fn, shifts=(16, 50), npairs=10)\n"
        "B.check_table('t40_one_sample', B.product_table_fn, [1])\n"
        "B.check_table('t150_short', B.product_table_fn, [0])\n"
        "M.check(M.product_fn, opt_ids=[0, 4], limit=20, maxlen=160)\n"
        "D.check_all(D.product_fn, sizes=(1200,))\n"
        "print('SCHED OK')\n") % (os.path.dirname(HERE), lib)
    env = dict(os.environ, CUEMU_SCHED=str(sched))
    env["DADA2B_BIMFWD"] = bimfwd
    out = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600, cwd=os.path.dirname(HERE))
    assert out.returncode == 0 and "SCHED OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
