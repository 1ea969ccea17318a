"""Taxonomic classification (dd_taxonomy.cu) on the H100: every check of the emulator file, the ten_16s training set,
a 2 000-genus synthetic database with 2*10^4 250-nt and 2 000 full-length queries (500 restated exactly), and the man
page's example against the reference's golden output."""
import os
import random

import numpy as np
import pytest

from tests import taxonomy_cases as G
from tests import taxonomy_ref as T
from tests import taxonomy_synth as S

pytestmark = pytest.mark.gpu


def test_gpu_taxonomy_example_exact():
    db, lgk, nbad = G.run_all(gpu=True)
    print("example: 1-ulp table entries %d of %d" % (nbad, lgk.size))


def test_gpu_taxonomy_chunking(monkeypatch):
    G.check_chunking(monkeypatch, seqs_n=6)


def test_gpu_taxonomy_refusals():
    G.check_refusals()


def test_gpu_taxonomy_ten16s():
    from dada2_b200 import taxonomy as tx
    ids, refs = T.ten16s()
    refs2, gu, r2g, gm, td = tx.parse_training(ids, refs)
    db = tx.TaxDB((ids, refs))
    lgk, nbad = G.check_table(db, refs2, r2g, "ten_16s")
    print("ten_16s: 1-ulp table entries %d of %d" % (nbad, lgk.size))
    rng = random.Random(5)
    q = rng.sample(refs, 150)
    win = [s[500:750] if k % 2 == 0 else T.revcomp(s[500:750]) for k, s in enumerate(q)]
    G.check_exact(db, q, False, 7, lgk=lgk, label="ten_16s full")
    G.check_exact(db, win, True, 8, lgk=lgk, label="ten_16s windows")
    G.check_logp_hook(db, win[:5], lgk)


def test_gpu_taxonomy_synthetic_scale():
    from dada2_b200 import taxonomy as tx
    refs, r2g, gm, gseq = S.database(20000, 2000, seed=11)
    db = tx.TaxDB.from_arrays(refs, r2g, gm)
    print("build:", {k: db.info[k] for k in ("table_bytes", "ms_device", "ms_total")})
    lgk = G.product_table(db)
    short = S.queries(gseq, 20000, seed=12)
    full = S.queries(gseq, 2000, seed=13, full=True, rc_half=False)
    rng = np.random.default_rng(3)
    for qs, rc, lab, ns in ((short, True, "250 nt, tryRC", 400), (full, False, "full length", 100)):
        got = db.raw(qs, rc, None, 99)
        st = got["stats"]
        print("%s: %d queries, %.1f ms device (%.1f kernels), %d launches" % (lab, len(qs), st["ms_device"], st["ms_kernels"], st["gpu_launches"]))
        only = np.sort(rng.choice(len(qs), ns, replace=False))
        want = T.classify(lgk, gm, qs, rc, 99, None, only=only)
        for k in ("tax", "boot", "boot_tax", "used_rc"):
            np.testing.assert_array_equal(got[k][only], want[k][only], err_msg=lab + " " + k)
        np.testing.assert_array_equal(got["logp"][only].view(np.int32), want["logp"][only].view(np.int32))
        ties = int((~want["boot_strict"][only]).sum())
        print("%s: %d of %d sampled bootstraps were exact ties" % (lab, ties, only.size * T.NBOOT))
        if rc:
            assert got["used_rc"].sum() > 0.4 * len(qs)


def test_gpu_taxonomy_man_page_example_golden():
    from dada2_b200 import taxonomy as tx
    g = np.load(os.path.join(T.GOLDEN, "taxonomy.npz"))
    seqs = G.example_seqs()
    for name, qs, rc in (("fwd", seqs, False), ("rc", [T.revcomp(s) for s in seqs], True)):
        d = tx.assignTaxonomy(qs, G.TRAIN, tryRC=rc, outputBootstraps=True, seed=int(g["seed"]))
        db = G.example_db()
        got = db.raw(qs, rc, None, int(g["seed"]))
        strict = g[name + "/strict"]
        np.testing.assert_array_equal(got["tax"][strict], g[name + "/tax"][strict])
        bs = g[name + "/boot_strict"] & strict[:, None]
        np.testing.assert_array_equal(got["boot_tax"][bs], g[name + "/boot_tax"][bs])
        free = strict & g[name + "/boot_strict"].all(axis=1)
        np.testing.assert_array_equal(got["boot"][free], g[name + "/boot"][free])
        np.testing.assert_array_equal(d["boot"], got["boot"])
        assert d["tax"].shape == (len(qs), db.td) and d["levels"] == ["Kingdom", "Phylum", "Class", "Order", "Family", "Genus"][:db.td]
        print("man page %s: %d/%d strict, %d tie-free" % (name, strict.sum(), len(qs), free.sum()))
