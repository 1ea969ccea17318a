"""dada() over samples (dada2_b200/denoise.py) with every dada_uniques pass run by the reference's own C++
(oracle.ref.dada_uniques) instead of the GPU: options, validation messages, the err extension, initializeErr, the
selfConsist loop, the pseudo-pooling pass and the expansion of a pooled result -- CPU suite."""
import os

import numpy as np
import pytest

from tests import cases

HERE = os.path.dirname(os.path.abspath(__file__))
NA = np.iinfo(np.int32).min


@pytest.fixture()
def ref_runner(monkeypatch):
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref was not built")
    import dada2_b200.denoise as dn
    calls = []

    def run(seqs, ab, priors, err, quals, **kw):
        calls.append({"err": np.array(err), "max_clust": kw["max_clust"], "priors": list(priors) if priors is not None else None})
        return ref.dada_uniques(seqs, ab, priors, err, quals, **kw)
    monkeypatch.setattr(dn.api, "dada_uniques", run)
    yield calls


def sam1():
    from oracle import derep as O
    from tests import derep_cases as D
    return O.derep_reads(*D.sam1F_reads())


def test_err_extension_and_initializeErr(ref_runner):
    from dada2_b200.denoise import dada, extend_err, initial_err
    e = cases.tperr1()
    x = extend_err(e[:, :30], 38)
    assert x.shape == (16, 39) and np.array_equal(x[:, :30], e[:, :30]) and (x[:, 30:] == e[:, 29:30]).all()
    assert extend_err(e, 20) is not None and extend_err(e, 20).shape == e.shape
    assert initial_err(38).shape == (16, 41) and initial_err(60).shape == (16, 61) and (initial_err(60) == 1).all()
    d = sam1()
    dada(d, err=e[:, :30], MAX_CONSIST=1)
    qmax = int(np.ceil(np.nanmax(d["quals"])))
    assert ref_runner[0]["err"].shape == (16, max(30, qmax + 1)) and ref_runner[0]["max_clust"] == 0
    ref_runner.clear()
    r = dada(d, err=None, selfConsist=True, MAX_CONSIST=2, MAX_CLUST=7)
    assert (ref_runner[0]["err"] == 1).all() and ref_runner[0]["err"].shape == (16, max(41, qmax + 1))
    assert ref_runner[0]["max_clust"] == 1 and ref_runner[1]["max_clust"] == 7
    assert (r["err_in"][0][[0, 5, 10, 15]] == 1).all()          # self-transitions of the initial estimate forced to 1


def test_selfconsist_convergence_and_MAX_CONSIST(ref_runner):
    from dada2_b200.denoise import dada
    from dada2_b200.errmodel import accumulateTrans, loessErrfun
    d = sam1()
    r = dada(d, err=cases.tperr1(), selfConsist=True, MAX_CONSIST=2)
    assert r["passes"] == 2 and len(r["err_in"]) == 2 and len(ref_runner) == 2
    assert np.array_equal(r["err_in"][1], loessErrfun(accumulateTrans([dada_pass(d, r["err_in"][0])])))
    ref_runner.clear()
    full = dada(d, err=cases.tperr1(), selfConsist=True)
    errs = full["err_in"]
    assert full["passes"] == len(errs) <= 10
    assert len(errs) == 10 or any(np.array_equal(e, full["err_out"]) for e in errs)   # stopped on a repeat, or at MAX_CONSIST


def dada_pass(d, err):
    from oracle import ref
    from dada2_b200.denoise import extend_err
    return ref.dada_uniques(d["uniques"], d["abundances"], None, extend_err(err, int(np.ceil(np.nanmax(d["quals"])))), d["quals"])["subqual"]


def test_pseudo_two_pass_loop(ref_runner):
    from dada2_b200.denoise import dada
    from tests.test_gpu_zz_denoise import _noqual, _pseudo_samples
    ds, V = _pseudo_samples()
    err = np.full((16, 41), 1e-3); err[[0, 5, 10, 15]] = 1 - 3e-3
    seen = []

    def errfun(trans):
        seen.append(np.array(trans))
        return _noqual(trans)
    r = dada(ds, err=err, pool="pseudo", errorEstimationFunction=errfun)
    assert len(ref_runner) == 6 and r[0]["passes"] == 2
    assert all(np.array_equal(c["err"], err) for c in ref_runner[:3])
    assert all(np.array_equal(c["err"], _noqual(seen[0])) for c in ref_runner[3:])   # pass 2: the refit of pass 1's trans
    assert np.array_equal(r[0]["err_in"], err) and np.array_equal(r[0]["err_out"], _noqual(seen[1]))
    assert V in r[0]["pseudo_priors"]
    assert [c["priors"] for c in ref_runner[3:]] == [[s in r[0]["pseudo_priors"] for s in d["uniques"]] for d in ds]
    assert V in r[2]["denoised"]


def test_validation_messages():
    import warnings
    from dada2_b200.denoise import dada
    d = {"uniques": ["ACGTACGTAC", "ACGTACGTAA"], "abundances": np.array([5, 2], np.int32), "quals": np.full((2, 10), 30.0),
         "map": np.array([1, 1, 2], np.int32)}
    e = cases.tperr1()
    with pytest.raises(ValueError, match="must be derep-class object"):
        dada(42, err=e)
    with pytest.raises(ValueError, match="filenames provided do not exist"):
        dada(["/nonexistent/x.fastq.gz"], err=e)
    with pytest.raises(ValueError, match="Invalid pool argument"):
        dada([d, d], err=e, pool="yes")
    with pytest.raises(ValueError, match="OMEGA_A must be between zero and one"):
        dada(d, err=e, OMEGA_A=1)
    with pytest.raises(ValueError, match="OMEGA_P must be between zero and one"):
        dada(d, err=e, OMEGA_P=-1)
    with pytest.raises(ValueError, match="Some error correction required"):
        dada(d, err=e, selfConsist=True, OMEGA_C=1)
    with pytest.raises(ValueError, match="Must provide a function"):
        dada(d, err=e, errorEstimationFunction=None)
    with pytest.raises(ValueError, match="Error matrix"):
        dada(d, err=None)
    with pytest.raises(ValueError, match="Sequences must be made up only of A/C/G/T"):
        dada(dict(d, uniques=["ACGTNCGTAC", "ACGTACGTAA"]), err=e)
    with pytest.raises(ValueError, match="must include quals"):
        dada(dict(d, quals=None), err=e)
    with pytest.raises(ValueError, match="one row for each"):
        dada(dict(d, quals=np.full((1, 10), 30.0)), err=e)
    with pytest.raises(ValueError, match="as many columns"):
        dada(dict(d, quals=np.full((2, 9), 30.0)), err=e)
    q = np.full((2, 10), 30.0); q[1, 4] = np.nan
    with pytest.raises(ValueError, match="NAs in derep"):
        dada(dict(d, quals=q), err=e)
    with pytest.raises(ValueError, match="Quality values must be positive"):
        dada(dict(d, quals=np.full((2, 10), -1.0)), err=e)
    with pytest.raises(ValueError, match="Sample 2 has an invalid maximum Phred Quality Scores of 251"):
        dada([d, dict(d, quals=np.full((2, 10), 250.5))], err=e)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        with pytest.raises(ValueError, match="OMEGA_A"):
            dada(d, err=e, NOT_AN_OPTION=1, OMEGA_A=2)
        assert any("NOT_AN_OPTION is not a valid DADA option." in str(x.message) for x in w)
        with pytest.raises(ValueError, match="OMEGA_A"):
            dada(d, err=e, priors=["ACGT"], OMEGA_P=1e-50, OMEGA_A=2)


def test_gap_options(ref_runner):
    from dada2_b200.denoise import dada
    d = sam1()
    r = dada(d, err=cases.tperr1(), GAP_PENALTY=8, HOMOPOLYMER_GAP_PENALTY=3)
    assert r["opts"]["GAP_PENALTY"] == -8 and r["opts"]["HOMOPOLYMER_GAP_PENALTY"] == -3 and not r["opts"]["VECTORIZED_ALIGNMENT"]
    r = dada(d, err=cases.tperr1(), BAND_SIZE=0)
    assert r["opts"]["HOMOPOLYMER_GAP_PENALTY"] == -8 and not r["opts"]["VECTORIZED_ALIGNMENT"]
    r = dada(d, err=cases.tperr1())
    assert r["opts"]["VECTORIZED_ALIGNMENT"]
    cases.assert_same(r, dada_ref(d), rtol=0, label="one sample")


def dada_ref(d):
    from oracle import ref
    return ref.dada_uniques(d["uniques"], d["abundances"], None, cases.tperr1(), d["quals"])


def test_pool_expansion_hand_worked():
    """Three samples over five pooled uniques P1..P5 denoised into three clusters (P1, P2 -> 1, P3 -> 2, P4 -> 3, P5
    unassigned), birth_subs in clusters 2 and 3."""
    from dada2_b200.denoise import _expand_pooled
    pres = {"map": np.array([1, 1, 2, 3, NA], np.int32), "pval": np.arange(5.0), "trans": np.ones((16, 3)),
            "clustering": {"sequence": ["S1", "S3", "S4"], "abundance": np.array([16, 10, 7], np.int32),
                           "pval": np.array([0.0, 1e-9, 1e-12])},
            "birth_subs": {"pos": np.array([5, 7, 9], np.int32), "clust": np.array([2, 3, 3], np.int32), "ref": ["A", "C", "G"],
                           "sub": ["T", "T", "A"], "qual": np.array([30.0, 31.0, 32.0])},
            "quality": np.arange(12.0).reshape(3, 4)}
    a = _expand_pooled(pres, np.array([1, 2, 5]), np.array([10, 4, 1]), 3)
    assert a["denoised"] == {"S1": 14} and a["map"].tolist() == [1, 1, NA] and a["birth_subs"]["clust"].tolist() == []
    assert a["quality"].tolist() == [[0.0, 1.0, 2.0, 3.0]]
    b = _expand_pooled(pres, np.array([4, 3, 1]), np.array([6, 3, 2]), 3)
    assert b["denoised"] == {"S1": 2, "S3": 3, "S4": 6} and b["map"].tolist() == [3, 2, 1]
    assert b["birth_subs"]["clust"].tolist() == [2, 3, 3] and b["birth_subs"]["pos"].tolist() == [5, 7, 9]
    c = _expand_pooled(pres, np.array([3, 4]), np.array([7, 1]), 3)
    assert c["denoised"] == {"S3": 7, "S4": 1} and c["map"].tolist() == [1, 2] and c["sequence"] == ["S3", "S4"]
    assert c["birth_subs"]["clust"].tolist() == [1, 2, 2] and c["birth_subs"]["ref"] == ["A", "C", "G"]
    assert c["clustering"]["abundance"].tolist() == [7, 1] and c["clustering"]["pval"].tolist() == [1e-9, 1e-12]
    assert c["quality"].tolist() == [[4.0, 5.0, 6.0, 7.0], [8.0, 9.0, 10.0, 11.0]]
    assert c["pval"] is pres["pval"] and c["trans"] is pres["trans"]            # pooled pval and trans kept, as in R


def test_makeSequenceTable_accepts_dada_results(ref_runner):
    from dada2_b200.denoise import dada
    from dada2_b200.seqtab import makeSequenceTable
    from tests.test_gpu_zz_denoise import _pseudo_samples
    ds, V = _pseudo_samples()
    err = np.full((16, 41), 1e-3); err[[0, 5, 10, 15]] = 1 - 3e-3
    r = dada({"a": ds[0], "b": ds[1]}, err=err)
    mat, cols, rows = makeSequenceTable(r)
    assert rows == ["a", "b"] and mat.sum() == sum(sum(x["denoised"].values()) for x in r.values())
