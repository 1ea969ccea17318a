"""The de novo bimera kernels (dd_bimera.cu: k_bim_need's de novo rule, k_bim_denovo_flag) on the host SIMT emulator
against the removeBimeraDenovo goldens -- CPU suite.  Same assertions as tests/test_gpu_zz_removebim.py, at sizes the
emulator finishes in seconds: per-sample flags with and without zero-count queries, pooled flags, batches of three
queries (DADA2B_BIM_JB=3), every alignment kernel (DADA2B_BIMFWD=0/1/2), and removeBimeraDenovo end to end."""
import os
import platform
import sys

import numpy as np
import pytest

from tests import bimera_cases as B
from tests import removebim_cases as RC

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    monkeypatch.setenv("DADA2B_BIMFWD", "0")        # the traceback kernel; the variant test below overrides
    import build_emu
    import dada2_b200.api as api
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    import dada2_b200.bimera as bm
    monkeypatch.setattr(bm, "_BOUND", False)
    yield lib


def test_emu_denovo_per_sample_and_pooled(emu):
    RC.check_per_sample("s_edge", RC.product_flag_fn)
    RC.check_per_sample("s_edge", RC.product_flag_fn, opt_ids=[0, 4], zero_queries=True)
    RC.check_pooled("s_edge", RC.product_flag_fn)
    RC.check_per_sample("s_dup", RC.product_flag_fn, opt_ids=[0, 3])
    RC.check_pooled("s_dup", RC.product_flag_fn, opt_ids=[0, 3])
    RC.check_pooled("t40_one_sample", RC.product_flag_fn, opt_ids=[0, 1])


def test_emu_denovo_batches_and_pair_count(emu, monkeypatch):
    """Batches of three queries: the slot-to-query mapping of k_bim_need, the record matrix and k_bim_denovo_flag across
    eight batches; every needed (query, parent) pair is aligned exactly once over all rows."""
    from dada2_b200 import bimera
    monkeypatch.setenv("DADA2B_BIM_JB", "3")
    RC.check_per_sample("s_edge", RC.product_flag_fn, opt_ids=[1])
    RC.check_pooled("s_edge", RC.product_flag_fn, opt_ids=[4])
    seqs, mat = RC.table("s_edge")
    for zq in (False, True):
        flags, st = bimera.denovo_bimera(mat, seqs, zero_queries=zq, return_stats=True)
        assert st["n_pairs"] == RC.need_pairs(mat, zq), (zq, st["n_pairs"])
    monkeypatch.delenv("DADA2B_BIM_JB")
    _, st1 = bimera.denovo_bimera(mat, seqs, zero_queries=False, return_stats=True)
    assert st1["n_pairs"] == st["n_pairs"] - (RC.need_pairs(mat, True) - RC.need_pairs(mat, False))
    assert st1["gpu_launches"] < st["gpu_launches"]


@pytest.mark.parametrize("variant,name,oi", [("1", "s_edge", 2), ("2", "s_edge", 6), ("2", "s_dup", 1)])
def test_emu_denovo_alignment_kernels(emu, monkeypatch, variant, name, oi):
    monkeypatch.setenv("DADA2B_BIMFWD", variant)
    RC.check_per_sample(name, RC.product_flag_fn, opt_ids=[oi])


def test_emu_is_bimera_denovo_unchanged(emu):
    B.check_is_bimera("t40_one_sample", B.product_denovo_fn)


def test_emu_remove_bimera_denovo_forms(emu, capsys):
    from dada2_b200 import Dada2bError, bimera, removeBimeraDenovo
    seqs, mat = RC.table("s_edge")
    flags = RC.golden()["s_edge_o0_persample"].astype(bool)
    out, cols = removeBimeraDenovo((mat, seqs), method="per-sample")
    keep = np.where(flags, 0, mat).sum(axis=0) > 0
    assert cols == [s for s, k in zip(seqs, keep) if k] and np.array_equal(out, np.where(flags, 0, mat)[:, keep])
    pooled = RC.golden()["s_edge_o0_pooled"].astype(bool)
    u = {s: int(a) for s, a in zip(seqs, mat.sum(axis=0))}
    assert removeBimeraDenovo(u, verbose=True) == {s: a for (s, a), b in zip(u.items(), pooled) if not b}
    assert "Identified %d bimeras out of %d input sequences." % (pooled.sum(), len(seqs)) in capsys.readouterr().err
    # errors of the device call: an empty sequence (returnRejects' "" rows), negative counts, other letters
    with pytest.raises(Dada2bError, match="Empty sequences"):
        removeBimeraDenovo({"sequence": seqs[:3] + [""], "abundance": np.array([50, 40, 3, 1], np.int32)})
    with pytest.raises(Dada2bError, match="negative"):
        bimera.denovo_bimera(np.array([[3, -1]], np.int32), seqs[:2])
    with pytest.raises(Dada2bError, match="A/C/G/T"):
        bimera.denovo_bimera(np.array([[3, 1]], np.int32), [seqs[0], "ACGTN" + seqs[1]])
    assert bimera.isBimeraDenovo([], []).shape == (0,)
