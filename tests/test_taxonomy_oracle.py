"""The restatement (tests/taxonomy_ref.py) against the reference's C_assign_taxonomy2 compiled unmodified
(oracle/_ref/libdada2ref_taxonomy.so), with the same injected uniforms; and the R wrapper rules on crafted fastas.

The reference's table uses glibc's logf and its ties are drawn with std::random_device, so a (query, replicate) is
compared only where the restatement's arg-max leads the runner-up by more than the sums could move under 1-ulp table
differences; boot counts are compared on queries where the main assignment and all 100 bootstraps are such."""
import gzip
import os
import random
import warnings

import numpy as np
import pytest

from tests import taxonomy_ref as T

needs_ref = pytest.mark.skipif(T.ref_lib() is None, reason="oracle/_ref/libdada2ref_taxonomy.so is not built")


def _tol(lp, n):
    return n * (2.0 * np.spacing(np.float32(abs(lp))) + 4e-6)


def compare(seqs, refs, r2g, gm, try_rc, seed, label, min_free=0.8):
    lgk = T.table(refs, r2g, gm.shape[0])
    u = T.unifs_buffer(seqs, seed)
    want = T.classify(lgk, gm, seqs, try_rc, seed, u)
    keep = [j for j, s in enumerate(seqs) if len(s) >= 7]                # shorter queries make the reference's call fail
    got = T.ref_assign([seqs[j] for j in keep], refs, r2g, gm, try_rc, _ref_unifs(seqs, keep, u), nthreads=4)
    nmain = nboot = free = 0
    for i, j in enumerate(keep):
        if want["tax"][j] == T.NA:
            assert got["tax"][i] == T.NA and not got["boot"][i].any()
            continue
        n = len(T.karray(seqs[j]))
        main_ok = want["strict"][j] and want["gap"][j] > _tol(want["logp"][j], n)
        if main_ok:
            nmain += 1
            assert got["tax"][i] == want["tax"][j], (label, j)
        boots_ok = want["boot_strict"][j] & (want["boot_gap"][j] > _tol(want["logp"][j], max(n // 8, 1)))
        for b in np.flatnonzero(boots_ok if main_ok else np.zeros(T.NBOOT, bool)):
            nboot += 1
            assert got["boot_tax"][i, b] == want["boot_tax"][j, b], (label, j, b)
        if main_ok and boots_ok.all():
            free += 1
            np.testing.assert_array_equal(got["boot"][i], want["boot"][j], err_msg="%s %d" % (label, j))
    nq = sum(1 for j in keep if want["tax"][j] != T.NA)
    print("%s: %d/%d queries tie-free (%.1f%%), %d strict main assignments, %d strict bootstraps" %
          (label, free, nq, 100.0 * free / max(nq, 1), nmain, nboot))
    assert free >= min_free * nq, (label, free, nq)


def _ref_unifs(seqs, keep, u):
    """The reference sees only the queries of at least 7 nt (shorter ones fail its call).  Neighbouring queries read
    overlapping stretches of the buffer, so the short queries go last: the kept ones keep their indices, and the
    reference's (shorter) buffer is a prefix of the full one."""
    assert keep == list(range(len(keep)))
    return u[: len(keep) * T.NBOOT * (T.max_arraylen(seqs) // 8)]


@needs_ref
def test_oracle_example_set():
    from dada2_b200 import taxonomy as tx
    ids, refs = tx.read_fasta(os.path.join(T.GOLDEN, "example_train_set.fa.gz"))
    refs, gu, r2g, gm, td = tx.parse_training(ids, refs)
    seqs = T.read_fasta(os.path.join(T.GOLDEN, "example_seqs.fa"))[1]
    short = [seqs[0][:40], seqs[1][:50], seqs[2][:60] + "NNN" + seqs[2][63:200], "N" * 70, "ACGTA"]
    compare(seqs + short, refs, r2g, gm, False, 1, "example", min_free=0.5)
    compare(seqs + [T.revcomp(s) for s in seqs], refs, r2g, gm, True, 2, "example tryRC", min_free=0.5)


@needs_ref
def test_oracle_ten16s_held_out():
    from dada2_b200 import taxonomy as tx
    ids, refs = T.ten16s()
    rng = random.Random(16)
    idx = list(range(len(refs)))
    rng.shuffle(idx)
    held = set(idx[: len(idx) // 10])
    train = [i for i in range(len(refs)) if i not in held]
    refs2, gu, r2g, gm, td = tx.parse_training([ids[i] for i in train], [refs[i] for i in train])
    assert sum(1 for r in refs if set(r) - set("ACGT")) > 0                     # N-containing references are in the set
    q = [refs[i] for i in sorted(held)][:60]
    win = []
    for k, s in enumerate(q):
        a = 500 + (k * 13) % 40 if len(s) > 800 else 0
        w = s[a:a + 250]
        win.append(T.revcomp(w) if k % 2 else w)
    compare(q, refs2, r2g, gm, False, 3, "ten_16s full length", min_free=0.5)
    compare(win, refs2, r2g, gm, True, 4, "ten_16s V4-like windows, tryRC", min_free=0.5)


# ---- wrapper rules (R/taxonomy.R:76-122, 136-159) on crafted fastas ----
def _fasta(path, recs):
    with (gzip.open(path, "wt") if path.endswith(".gz") else open(path, "w")) as f:
        for h, s in recs:
            f.write(">%s\n%s\n" % (h, s))


def _seq(rng, n=60):
    return "".join(rng.choice("ACGT") for _ in range(n))


def test_wrapper_rules(tmp_path):
    from dada2_b200 import Dada2bError, taxonomy as tx
    rng = random.Random(1)
    # short references are dropped with R's warning; headers are stripped; ragged depths padded; a missing trailing ';'
    # glues the pad onto the last level
    recs = [("  K1;P1;G1; ", _seq(rng)), ("K1;P1;", _seq(rng)), ("K1;P2;G2;S2;", _seq(rng)), ("K1;P3", _seq(rng)), ("K2;P9;G9;", "ACGT" * 4)]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        refs, gu, r2g, gm, td = tx.parse_training([h for h, _ in recs], [s for _, s in recs])
    assert any("too short" in str(x.message) for x in w)
    assert len(refs) == 4 and td == 4
    assert gu == ["K1;P1;G1;_DADA2_UNSPECIFIED;", "K1;P1;_DADA2_UNSPECIFIED;_DADA2_UNSPECIFIED;", "K1;P2;G2;S2;",
                  "K1;P3_DADA2_UNSPECIFIED;_DADA2_UNSPECIFIED;"]
    assert list(r2g) == [1, 2, 3, 4]
    assert gm.shape == (4, 4) and gm[0, 0] == gm[1, 0] == gm[2, 0] and gm[0, 1] == gm[1, 1] != gm[2, 1]
    # UNITE: sniffed on the first ten headers only, and not below ten references
    unite = ["SH%d|AB%d|SH%d.08FU|refs|k__Fungi;p__Asco;c__unidentified;o__O%d;f__F;g__G%d;s__G%d_sp" % (i, i, i, i, i, i) for i in range(10)]
    unite[1] = unite[1].replace("s__G1_sp", "s__G1_alba_x")
    seqs = [_seq(rng) for _ in range(10)]
    refs, gu, r2g, gm, td = tx.parse_training(unite, seqs)
    assert gu[0] == "k__Fungi;p__Asco;_DADA2_UNSPECIFIED;o__O0;f__F;g__G0;_DADA2_UNSPECIFIED"
    assert gu[1] == "k__Fungi;p__Asco;_DADA2_UNSPECIFIED;o__O1;f__F;g__G1;s__x"          # greedy \w+ up to the last '_'
    assert td == 7
    refs, gu, r2g, gm, td = tx.parse_training(unite[:9], seqs[:9])                   # nine: not UNITE
    assert gu[0] == unite[0]
    # both format errors
    with pytest.raises(Dada2bError, match="looks like a file formatted for assignSpecies"):
        tx.parse_training(["AB1 Genus species"], [_seq(rng)])
    with pytest.raises(Dada2bError, match=r"format for assignTaxonomy\.$"):
        tx.parse_training(["Bacteria"], [_seq(rng)])
    # the output matrix: minBoot prefix, unspecified -> NA, level names, outputBootstraps
    res = {"tax": np.array([1, 3, T.NA], np.int32), "boot": np.array([[100, 90, 40, 0], [100, 100, 100, 60], [0, 0, 0, 0]], np.int32)}
    gu = ["K1;P1;G1;_DADA2_UNSPECIFIED;", "x", "K1;P2;G2;S2;"]
    out, names = tx._assemble(res, ["a", "b", "c"], gu, 4, 50, list(tx.TAX_LEVELS), False)
    assert names == ["Kingdom", "Phylum", "Class", "Order"]
    assert out.tolist() == [["K1", "P1", None, None], ["K1", "P2", "G2", "S2"], [None] * 4]
    out, names = tx._assemble(res, ["a", "b", "c"], gu, 4, 0, ["L1", "L2"], False)
    assert names == ["L1", "L2", None, None] and out[0].tolist() == ["K1", "P1", "G1", None]
    d = tx._assemble(res, ["a", "b", "c"], gu, 4, 50, list(tx.TAX_LEVELS), True)
    assert (d["boot"] == res["boot"]).all() and d["tax"][1].tolist() == ["K1", "P2", "G2", "S2"]
    # inputs: strings, a makeSequenceTable result, a dada result
    assert tx.get_sequences("ACGT") == ["ACGT"]
    assert tx.get_sequences((np.zeros((1, 2)), ["A", "C"], None)) == ["A", "C"]
    assert tx.get_sequences({"clustering": {"sequence": ["G"]}}) == ["G"]
    # the fasta reader: gzip by magic bytes, multi-line records, upper case
    p = str(tmp_path / "r.fa.gz")
    _fasta(p, [("K;P;", "acgt\nACGT"), ("K;Q;", "GG GG")])
    assert tx.read_fasta(p) == (["K;P;", "K;Q;"], ["ACGTACGT", "GGGG"])
