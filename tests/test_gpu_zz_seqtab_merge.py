"""mergeSequenceTables' kernels (dd_seqtab.cu) on hardware: every hand case, seeded merges against the restatement --
one of 12 runs x 96 samples with some 10^5 distinct columns (the column sort wraps many radix tiles, runs in reverse
orientation collapse, and repeated sample names make tables meet in the accumulator), tryRC on and off -- and a merge
whose result has more than 2^16 columns."""
import time

import numpy as np
import pytest

from tests import seqtab_merge_cases as G

pytestmark = pytest.mark.gpu


def test_gpu_seqtab_merge_hand_cases():
    G.check_hand()


@pytest.mark.parametrize("tryRC", [False, True])
def test_gpu_seqtab_merge_seeded_small(tryRC):
    runs = G.make_runs(11, nruns=4, nsamp=12, pool=400, per_run=150)
    G.check_seeded(runs, tryRC=tryRC)
    G.check_seeded(runs, tryRC=tryRC, orderBy="nsamples")


@pytest.mark.parametrize("tryRC", [False, True])
def test_gpu_seqtab_merge_twelve_runs(tryRC):
    runs = G.make_runs(7, nruns=12, nsamp=96, pool=200000, per_run=20000, shared_frac=0.25)
    t0 = time.perf_counter()
    mat, cols, rows = G.check_seeded(runs, tryRC=tryRC, repeats="sum")
    print("12 runs, tryRC=%s: %d x %d, %.1f s with the restatement" % (tryRC, mat.shape[0], mat.shape[1], time.perf_counter() - t0))
    assert mat.shape[1] > 100000 and len(rows) < 12 * 96


def test_gpu_seqtab_merge_wide():
    """ncol_out above 2^16."""
    runs = G.make_runs(9, nruns=2, nsamp=3, pool=300000, per_run=40000, rc_every=0, dup_frac=0.0, merged_frac=0.0)
    mat, cols, rows = G.check_seeded(runs, orderBy=None)
    assert mat.shape[1] > 1 << 16
