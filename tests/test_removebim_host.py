"""removeBimeraDenovo's host logic (dada2_b200/bimera.py) with the device flag functions replaced by the test reference
(tests/removebim_ref.py): every input form and method, containers, duplicated sequences, keyword arguments, R's
messages and errors, output shapes.  CPU only."""
import numpy as np
import pytest

from dada2_b200 import bimera, Dada2bError, removeBimeraDenovo
from tests import removebim_cases as RC
from tests import removebim_ref as R


@pytest.fixture(autouse=True)
def host_flags(monkeypatch):
    calls = []

    def denovo(mat, seqs, zero_queries, device=0, **rule):
        assert len(set(seqs)) == len(seqs)                     # duplicates are collapsed before the flag function
        calls.append(("denovo", np.asarray(mat).shape, bool(zero_queries), rule))
        return R.denovo_flags(mat, seqs, zero_queries, **rule)

    def table(mat, seqs, min_fold=1.5, min_abund=2, allow_one_off=False, min_one_off_par_dist=4, max_shift=16, device=0, **_):
        calls.append(("table", np.asarray(mat).shape))
        nflag, nsam = R.backend().table_bimera(mat, seqs, min_fold=min_fold, min_abund=min_abund, allow_one_off=allow_one_off,
                                               min_one_off_par_dist=min_one_off_par_dist, max_shift=max_shift)
        return {"nflag": nflag, "nsam": nsam}
    monkeypatch.setattr(bimera, "denovo_flags", denovo)
    monkeypatch.setattr(bimera, "C_table_bimera2", table)
    return calls


def _vec(name="s_edge", row=None):
    seqs, mat = RC.table(name)
    ab = mat.sum(axis=0) if row is None else mat[row]
    return seqs, ab


def test_uniques_dict_dada_and_derep(host_flags):
    seqs, ab = _vec()
    bim = R.is_bimera_denovo(seqs, ab)
    assert bim.any() and not bim.all()
    want = {s: int(a) for s, a, b in zip(seqs, ab, bim) if not b}
    u = {s: int(a) for s, a in zip(seqs, ab)}
    assert removeBimeraDenovo(u) == want
    assert host_flags[-1][2] is True                           # vectors: every entry is a query, zero abundances too
    assert removeBimeraDenovo({"denoised": u, "clustering": {}, "sequence": seqs}) == want
    assert removeBimeraDenovo({"uniques": seqs, "abundances": np.asarray(ab, np.int32), "quals": None}) == want
    # isBimeraDenovo's arguments reach the rule; multithread is accepted and ignored
    bim1 = R.is_bimera_denovo(seqs, ab, allowOneOff=True, minParentAbundance=2.5)
    got = removeBimeraDenovo(u, allowOneOff=True, minParentAbundance=2.5, multithread=True)
    assert got == {s: int(a) for s, a, b in zip(seqs, ab, bim1) if not b}
    assert host_flags[-1][3] == dict(allowOneOff=True, minParentAbundance=2.5)


def test_merger_rows_and_duplicates(host_flags, capsys):
    seqs, ab = _vec()
    seqs = seqs + [seqs[3]]                                    # a duplicated merged sequence: summed, verdict to both copies
    ab = np.concatenate([ab, [7]]).astype(np.int32)
    n = len(seqs)
    m = {"sequence": list(seqs), "abundance": ab, "forward": np.arange(1, n + 1, dtype=np.int32), "nmatch": list(range(n)),
         "accept": np.ones(n, bool)}
    bim = R.is_bimera_denovo(seqs, ab)
    assert bim[3] == bim[-1]
    got = removeBimeraDenovo(m, verbose=True)
    keep = ~bim
    assert got["sequence"] == [s for s, k in zip(seqs, keep) if k] and got["nmatch"] == [x for x, k in zip(range(n), keep) if k]
    assert np.array_equal(got["abundance"], ab[keep]) and np.array_equal(got["forward"], m["forward"][keep])
    err = capsys.readouterr().err
    assert "Duplicate sequences detected." in err
    assert "Identified %d bimeras out of %d input sequences." % (bim.sum(), n) in err


@pytest.mark.parametrize("name", ["s_edge", "s_dup"])
def test_tables_per_sample_and_pooled(host_flags, name, capsys):
    seqs, mat = RC.table(name)
    rows = ["r%d" % i for i in range(mat.shape[0])]
    # per-sample: the golden flag matrix (every cell evaluated, as R does) gives the same table
    out, cols, rn = removeBimeraDenovo((mat, seqs, rows), method="per-sample", verbose=True)
    flags = RC.golden()[name + "_o0_persample"].astype(bool)
    wmat, wcols = R.remove_table(mat, seqs, "per-sample", flags=flags)
    assert rn is rows and cols == wcols and np.array_equal(out, wmat)
    assert host_flags[-1][1] == (mat.shape[0], len(set(seqs))) and host_flags[-1][2] is False
    err = capsys.readouterr().err
    assert err.count("Identified ") == mat.shape[0]            # one isBimeraDenovo call per row, as in R
    # pooled: column sums, zero sums are queries
    out, cols = removeBimeraDenovo((mat, seqs), method="pooled", minFoldParentOverAbundance=1.0, minParentAbundance=1)
    pf = RC.golden()[name + "_o3_pooled"].astype(bool)
    assert cols == [s for s, b in zip(seqs, pf) if not b] and np.array_equal(out, mat[:, ~pf])
    assert host_flags[-1][1] == (1, len(set(seqs))) and host_flags[-1][2] is True


def test_table_consensus(host_flags, capsys):
    seqs, mat = RC.table("t40_one_sample")
    out, cols = removeBimeraDenovo((mat, seqs), verbose=True, minSampleFraction=0.5, allowOneOff=True)
    wmat, wcols = R.remove_table(mat, seqs, "consensus", minSampleFraction=0.5, allowOneOff=True)
    assert cols == wcols and np.array_equal(out, wmat) and len(cols) < len(seqs)
    assert host_flags[-1][0] == "table"
    assert "Identified %d bimeras out of %d input sequences." % (len(seqs) - len(cols), len(seqs)) in capsys.readouterr().err
    with pytest.raises(Dada2bError, match="Duplicate sequences detected in input."):
        removeBimeraDenovo((mat, seqs[:-1] + seqs[:1]))


def test_containers(host_flags):
    seqs, ab = _vec()
    u = {s: int(a) for s, a in zip(seqs, ab)}
    seqs2, mat2 = RC.table("s_dup")
    one = removeBimeraDenovo(u)
    tab = removeBimeraDenovo((mat2, seqs2), method="per-sample")
    got = removeBimeraDenovo([u, (mat2, seqs2)], method="per-sample")
    assert isinstance(got, list) and got[0] == one and np.array_equal(got[1][0], tab[0]) and got[1][1] == tab[1]
    got = removeBimeraDenovo({"a": u, "b": dict(u)})
    assert list(got) == ["a", "b"] and got["a"] == one and got["b"] == one
    assert removeBimeraDenovo({"only": u}) == one and removeBimeraDenovo([u]) == one        # one element comes back unwrapped
    assert removeBimeraDenovo([]) == []


def test_arguments_and_errors(host_flags):
    seqs, mat = RC.table("s_edge")
    u = {s: int(a) for s, a in zip(seqs, mat.sum(axis=0))}
    with pytest.raises(ValueError, match="DEFUNCT: The tableMethod argument has been replaced by the method argument"):
        removeBimeraDenovo(u, tableMethod="pooled")
    with pytest.raises(ValueError, match="Valid values for method: 'pooled', 'consensus', or 'per-sample'"):
        removeBimeraDenovo((mat, seqs), method="sample")
    assert removeBimeraDenovo(u, method="sample") == removeBimeraDenovo(u)      # method only matters for tables, as in R
    with pytest.raises(TypeError, match="unused argument"):
        removeBimeraDenovo(u, minSampleFraction=0.5)                            # an isBimeraDenovoTable argument
    with pytest.raises(TypeError, match="unused argument"):
        removeBimeraDenovo((mat, seqs), method="pooled", ignoreNNegatives=0)
    with pytest.raises(TypeError, match="unused argument"):
        removeBimeraDenovo((mat, seqs), minFold=2)
    with pytest.raises(ValueError, match="Unrecognized format"):
        removeBimeraDenovo("ACGT")
    with pytest.raises(ValueError, match="Unrecognized format"):
        removeBimeraDenovo([{"x": 1.5}])
    big = np.full((2, len(seqs)), 2 ** 30 + 1, np.int32)
    with pytest.raises(Dada2bError, match="int32"):
        removeBimeraDenovo((big, seqs), method="pooled")
