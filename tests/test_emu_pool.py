"""The sample-pooling kernels (dd_pool.cu) on the host SIMT emulator against the host combineDereps2, on every case of
tests/pool_cases.py, plus the resident pooled context and one AddressSanitizer run -- CPU suite."""
import os
import platform
import subprocess
import sys

import numpy as np
import pytest

from tests import pool_cases as P

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.derep as dr
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(dr, "_BOUND", False)
    yield lib


def test_emu_pool_matches_combineDereps2(emu):
    P.check_all()


def test_emu_pool_refusals(emu):
    P.check_refusals()


def test_emu_pool_resident_runs_dada_on_the_pooled_derep(emu):
    import dada2_b200
    from dada2_b200.derep import combineDereps2, pool_dereps
    from tests import cases
    ds = P.sam_dereps()
    want = combineDereps2(ds)
    got, rs = pool_dereps(ds, want_quals=False, resident=True)
    assert got["quals"] is None and got["uniques"] == want["uniques"]
    cases.assert_same(rs.run(cases.tperr1()), dada2_b200.dada_uniques(want["uniques"], want["abundances"], None, cases.tperr1(), want["quals"]),
                      rtol=0, label="pool_resident sam1F+sam2F")
    rs.close()
    name, ds, pr = P.cases()[1]                                 # ragged lengths, with prior flags carried into the context
    want = P.expected(ds, pr)
    got, rs = pool_dereps(ds, priors=pr, resident=True)
    err = np.full((16, 45), 0.01); err[[0, 5, 10, 15]] = 0.97
    cases.assert_same(rs.run(err), dada2_b200.dada_uniques(want["uniques"], want["abundances"], want["prior"], err, want["quals"]),
                      rtol=0, label="pool_resident priors")
    rs.close()


SCRIPT = """
import sys
sys.path.insert(0, %r)
import dada2_b200.api as api
api._LIBPATH = %r; api._LIB = None
from tests import pool_cases as P
P.check_all()
print('ASAN RUN OK')
"""


def test_emu_pool_memory_clean_under_asan():
    from tests.test_emu_asan import _preload
    asan = _preload()
    if asan is None:
        pytest.skip("libasan not found")
    import build_emu
    lib = build_emu.build(asan=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1")
    out = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, lib)], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert "AddressSanitizer" not in out.stderr, out.stderr[-4000:]
    assert out.returncode == 0 and "ASAN RUN OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
