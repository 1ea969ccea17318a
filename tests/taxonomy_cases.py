"""Taxonomy cases shared by the emulator and the H100 files: the product (dd_taxonomy.cu) against the numpy restatement,
bit for bit, with the restatement's sums fed the product's own table (fetched through the table hook); the table itself
against the restatement's under the 1-ulp rule; chunking, a resident TaxDB, explicit uniforms and every refusal."""
import os
import random

import numpy as np
import pytest

from tests import taxonomy_ref as T

TRAIN = os.path.join(T.GOLDEN, "example_train_set.fa.gz")
EXAMPLE = os.path.join(T.GOLDEN, "example_seqs.fa")


def product_table(db):
    return db.table(np.arange(T.NK), np.arange(db.ngenus)).T.copy()          # [G, 65536]


def check_table(db, refs, ref_to_genus, label=""):
    """Table hook against the restatement: bit-exact but for 1-ulp entries (fp64 log, rounded once); returns that count."""
    got = product_table(db)
    want = T.table(refs, ref_to_genus, db.ngenus)
    bad = got.view(np.int32) != want.view(np.int32)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1, (label, int(ulps.max()))
    nbad = int(bad.sum())
    assert nbad <= 3 + got.size * 1e-7, (label, nbad)
    for g, k in zip(*np.nonzero(bad)):
        print("%s: 1-ulp table entry genus %d k-mer %d: %r vs %r" % (label, g, k, got[g, k], want[g, k]))
    return got, nbad


def check_exact(db, seqs, try_rc, seed, unifs=None, lgk=None, label=""):
    """Product classification == restatement on the product's table (tax, boot, boot_tax, logp bits, used_rc)."""
    lgk = product_table(db) if lgk is None else lgk
    got = db.raw(seqs, try_rc, unifs, seed)
    want = T.classify(lgk, db.genusmat, seqs, try_rc, seed, unifs)
    for k in ("tax", "boot", "boot_tax", "used_rc"):
        np.testing.assert_array_equal(got[k], want[k], err_msg="%s %s" % (label, k))
    np.testing.assert_array_equal(got["logp"].view(np.int32), want["logp"].view(np.int32), err_msg=label + " logp")
    assert got["stats"]["gpu_launches"] > 0
    return got, want


def check_logp_hook(db, seqs, lgk):
    lp = db.logp(seqs)
    for j, s in enumerate(seqs):
        ka = T.karray(s)
        want_f = T.seq_sums(lgk, ka[None, :])[0]
        want_r = T.seq_sums(lgk, np.sort(T.rc_kmers(ka))[None, :])[0]
        np.testing.assert_array_equal(lp[j, 0].view(np.int32), want_f.view(np.int32))
        np.testing.assert_array_equal(lp[j, 1].view(np.int32), want_r.view(np.int32))


def example_db(**kw):
    from dada2_b200.taxonomy import TaxDB
    return TaxDB(TRAIN, **kw)


def example_seqs():
    return T.read_fasta(EXAMPLE)[1]


def length_queries(db_refs, rng):
    """Both sides of every length-driven layout: under 7, 7, under 50, exactly 50, a 250-nt window, N-rich, all-N, a
    full-length reference (distinct k-mers beyond the staged rows), and the 9 999-k-mer maximum."""
    long_ref = max(db_refs, key=len)
    qs = ["ACGTAC", "ACGTACG", "ACGTACGTACGTAGCTAGCTAGCATCGATCG", db_refs[0][:49], db_refs[0][:50], db_refs[1][100:350],
          db_refs[2][:120] + "N" + db_refs[2][121:260], "N" * 80, long_ref, db_refs[3][:200].lower() + db_refs[3][200:300]]
    big = "".join(rng.choice("ACGT") for _ in range(10006))
    qs.append(big)                                                            # 9 999 k-mers
    return qs


def run_all(gpu=False):
    """Every check on the example training set (and the length cases); the GPU adds more queries."""
    from dada2_b200 import taxonomy as tx
    db = example_db()
    ids, refs = tx.read_fasta(TRAIN)
    refs2, gu, r2g, gm, td = tx.parse_training(ids, refs)
    lgk, nbad = check_table(db, refs2, r2g, "example")
    seqs = example_seqs()
    rng = random.Random(7)
    qs = seqs + length_queries(refs2, rng) + [T.revcomp(s) for s in seqs[:3]]
    check_logp_hook(db, qs[:6] + qs[-4:], lgk)
    for try_rc in (False, True):
        check_exact(db, qs, try_rc, seed=11 + try_rc, lgk=lgk, label="example rc=%d" % try_rc)
    # explicit uniforms equal to the seeded draws give the seeded result; other uniforms give the restatement's
    u = T.unifs_buffer(qs, 5)
    a = db.raw(qs, True, u, 5)
    b = db.raw(qs, True, None, 5)
    for k in ("tax", "boot", "boot_tax"):
        np.testing.assert_array_equal(a[k], b[k])
    u2 = np.random.default_rng(3).random(u.size)
    check_exact(db, qs, True, 9, unifs=u2, lgk=lgk, label="explicit unifs")
    # resident reuse == one-shot, and the one-shot mirror
    r1 = db.raw(seqs, False, None, 21)
    r2 = db.raw(seqs, False, None, 21)
    one = tx.C_assign_taxonomy2(seqs, None, refs2, r2g, gm, False, seed=21)
    for k in ("tax", "boot", "boot_tax", "logp"):
        np.testing.assert_array_equal(r1[k], r2[k])
        np.testing.assert_array_equal(r1[k], one[k])
    return db, lgk, nbad


def check_chunking(monkeypatch, seqs_n=6):
    """DADA2B_TAX_CHUNK_GENERA=7 (chunks rebuilt per call) equals one resident table; so does max_table_bytes."""
    from dada2_b200 import taxonomy as tx
    seqs = example_seqs()[:seqs_n]
    base = example_db().raw(seqs, True, None, 3)
    monkeypatch.setenv("DADA2B_TAX_CHUNK_GENERA", "7")
    db = example_db()
    assert db.info["nchunk"] == -(-db.ngenus // 7)
    got = db.raw(seqs, True, None, 3)
    for k in ("tax", "boot", "boot_tax", "logp", "used_rc"):
        np.testing.assert_array_equal(got[k], base[k])
    ks = np.array([0, 1, 12345, 65535])
    monkeypatch.delenv("DADA2B_TAX_CHUNK_GENERA")
    np.testing.assert_array_equal(db.table(ks, np.arange(db.ngenus)), example_db().table(ks, np.arange(db.ngenus)))
    assert tx.TaxOpts  # the option form is covered by the ABI test


def check_refusals():
    from dada2_b200 import Dada2bError, taxonomy as tx
    db = example_db()
    with pytest.raises(Dada2bError, match="No seqs provided"):
        db.raw([], False)
    with pytest.raises(Dada2bError, match="at most 9999"):
        db.raw(["ACGT" * 2502], False)                                        # 10 001 k-mers
    with pytest.raises(Dada2bError, match="unifs must hold"):
        db.raw(["ACGT" * 20], False, unifs=np.zeros(3))
    with pytest.raises(Dada2bError, match="Invalid map"):
        tx.TaxDB.from_arrays(["ACGT" * 10], [2], np.ones((1, 2), np.int32))
    with pytest.raises(Dada2bError, match="Invalid map"):
        tx.TaxDB.from_arrays(["ACGT" * 10], [0], np.ones((1, 2), np.int32))
    with pytest.raises(Dada2bError, match="Length mismatch"):
        tx.TaxDB.from_arrays(["ACGT" * 10], [1, 1], np.ones((1, 2), np.int32))
    with pytest.raises(Dada2bError, match="No seqs provided"):
        tx.C_assign_taxonomy2([], [], ["ACGT" * 10], [1], np.ones((1, 2), np.int32), False)
    check_nref_limit()


def check_nref_limit():
    """nref >= 2^24 is refused before any reference is read (the pointers below cover a single one)."""
    import ctypes as C
    from dada2_b200 import taxonomy as tx
    L = tx._lib()
    off = np.zeros(2, np.int64)
    refs = tx.TaxSeqs(1 << 24, 0, b"\0", off.ctypes.data_as(C.POINTER(C.c_int64)))
    rg = np.ones(1, np.int32)
    gm = np.ones((1, 1), np.int32)
    db = C.c_void_p()
    eb = C.create_string_buffer(tx.ERRLEN)
    assert L.dada2b_tax_db_build(C.byref(refs), rg.ctypes.data, gm.ctypes.data, 1, 1, None, 0, C.byref(db), eb) != 0
    assert b"2^24" in eb.value and not db
