"""dada()'s aligners pair by pair at the length-driven switches of the core, on the host SIMT emulator (CPU suite): every pair set
of tests/longpair_cases.py at emulator size through dada2b_test_pairs and dada2b_test_loop_nw against the reference's alignments and
lambda, and small long-read samples through dada_uniques against the oracle at the default SM count and at DADA2B_SMS=1.  Scores
(mismatch -40) and a 900-column err bring the switches to a few hundred nt; tests/test_gpu_zz_longpairs.py runs them at the lengths
of the default scores on the GPU."""
import ctypes
import os
import platform
import sys

import pytest

from oracle import port

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

pytestmark = [pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only"),
              pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle_port.so is not built")]


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    h = ctypes.CDLL(lib)
    h.cuemu_launches.restype = ctypes.c_long
    h.cuemu_launches.argtypes = [ctypes.c_char_p]
    h.cuemu_reset_launches()
    yield h


def _sms():
    return int(os.environ.get("CUEMU_SMS", "2"))


def test_emu_longpair_stage(emu):
    import dada2_b200.api as api
    from tests import longpair_cases as P
    recs = P.run_cases(api.Resident, P.make_cases("emu", num_sms=_sms()), _sms())
    P.check_coverage(recs, one_sided=("smem G=16 ND=8", "smem G=32 ND=8"))
    for k in (b"k_nwfwd<", b"k_nwrow<", b"k_nwlane<", b"k_align"):
        assert emu.cuemu_launches(k) > 0, k


@pytest.mark.parametrize("sms", [None, "1"])
def test_emu_longpair_e2e(emu, monkeypatch, sms):
    import dada2_b200.api as api
    from tests import longpair_cases as P
    if sms:
        monkeypatch.setenv("DADA2B_SMS", sms)
    infos = [P.check_e2e(api.dada_uniques, s) for s in P.e2e_samples("emu")]
    assert infos[1]["p0_births"] > 0, infos[1]
    assert [i["fast_ok"] for i in infos[2:]] == [True, False]
