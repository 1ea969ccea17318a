"""The quality profile's kernels (dd_qprofile.cu) and plotQualityProfile / plotComplexity on hardware: every case of
tests/qprofile_cases.py, then in-memory tallies at run scale compared exactly with np.bincount: 4e6 x 250-nt reads with
full-range and with NovaSeq-binned scores, and 1e5 PacBio-like reads of 1000-2500 nt with scores up to 93."""
import time

import numpy as np
import pytest

from tests import qprofile_cases as G
from tests import qprofile_ref as R

pytestmark = pytest.mark.gpu


def test_gpu_qprofile_cases(tmp_path):
    G.check_profiles(str(tmp_path))
    G.check_complexity(str(tmp_path))
    G.check_edges_and_refusals(str(tmp_path))


def test_gpu_qprofile_aggregate_vignette():
    import dada2_b200
    fl = [G.gold("sam1F"), G.gold("sam2F")]
    G.check_frames("vignette", dada2_b200.plotQualityProfile(fl, aggregate=True), R.plot_quality_profile(fl, aggregate=True))


def _tally(off, qual, label):
    from dada2_b200 import qc
    t0 = time.perf_counter()
    got, st = qc.quality_tally(off, qual)
    wall = time.perf_counter() - t0
    want = R.tally_packed(off, qual)
    assert np.array_equal(got, want), label
    print("%s: %d bases, call %.1f ms, h2d %.2f ms, kernels %.3f ms" % (label, st["nbases"], wall * 1e3, st["ms_h2d"], st["ms_kernels"]))


@pytest.mark.parametrize("kind", ["full", "binned"])
def test_gpu_qprofile_illumina_scale(kind):
    n, L = 4000000, 250
    rng = np.random.default_rng(21 if kind == "full" else 22)
    if kind == "full":
        qual = rng.integers(0, 94, n * L, dtype=np.uint8)
    else:
        qual = np.array([2] * 2 + [12] * 5 + [23] * 13 + [37] * 80, np.uint8)[rng.integers(0, 100, n * L, dtype=np.uint8)]
    _tally(np.arange(n + 1, dtype=np.int64) * L, qual, "%d x %d %s" % (n, L, kind))


def test_gpu_qprofile_pacbio_scale():
    rng = np.random.default_rng(23)
    lens = rng.integers(1000, 2501, 100000)
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    qual = rng.integers(0, 94, int(off[-1]), dtype=np.uint8)
    _tally(off, qual, "1e5 PacBio-like")
