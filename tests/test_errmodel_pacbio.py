"""PacBioErrfun (R/errorModels.R:183-196): the three branches on the number of quality columns, and the selfConsist loop
with it as errorEstimationFunction at ncol = 94 -- CPU suite."""
import numpy as np
import pytest

from dada2_b200 import errmodel


def _trans(Q, seed=1):
    rng = np.random.default_rng(seed)
    t = np.zeros((16, Q))
    q = np.arange(Q)
    for i in range(4):
        for j in range(4):
            t[4 * i + j] = rng.poisson(2000 + 50 * q) if i == j else rng.poisson(40 * np.exp(-q / 25.0) + 1)
    return t


def test_q94_is_loess_on_0_92_plus_the_observed_rate_at_93():
    t = _trans(94)
    err = errmodel.PacBioErrfun(t)
    assert err.shape == (16, 94)
    assert np.array_equal(err[:, :93], errmodel.loessErrfun(t[:, :93]))          # bit for bit
    tot93 = np.array([t[4 * (r // 4):4 * (r // 4) + 4, 93].sum() for r in range(16)])
    assert np.array_equal(err[:, 93], (t[:, 93] + 1) / (tot93 + 4))
    assert np.allclose(err[:, 93].reshape(4, 4).sum(axis=1), (tot93[::4] + 4) / (tot93[::4] + 4))


def test_more_than_94_columns_is_refused():
    with pytest.raises(ValueError, match="Max qual score of 93 not the last column as expected."):
        errmodel.PacBioErrfun(_trans(95))


def test_fewer_than_94_columns_falls_back_to_loess(capsys):
    t = _trans(41)
    err = errmodel.PacBioErrfun(t)
    assert "The max qual score of 93 was not detected. Using standard error fitting." in capsys.readouterr().out
    assert np.array_equal(err, errmodel.loessErrfun(t))


def test_learn_errors_with_pacbio_errfun_terminates_at_ncol_94():
    seen = []

    def runner(err, max_clust):                          # a stand-in for one resident dada_uniques() pass
        seen.append(np.asarray(err).shape)
        return {"subqual": _trans(94, seed=7)}
    out = errmodel.learnErrors(runner, ncol=94, errorEstimationFunction=errmodel.PacBioErrfun)
    assert out["err_out"].shape == (16, 94) and out["passes"] <= 11
    assert all(s == (16, 94) for s in seen)
    assert np.array_equal(out["err_out"], errmodel.PacBioErrfun(_trans(94, seed=7)))
