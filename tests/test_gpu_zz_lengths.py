"""derep, filter, merge, bimera and collapse at real amplicon lengths on hardware, and on both sides of every
length-driven layout switch of their kernels (tests/length_cases.py computes each threshold from the host code's own
formula).  Regimes: MiSeq 2 x 300 pairs and 400-480 nt amplicons, V3-V4 tables of 400-460 nt ASVs, PacBio full-length
16S at 1400-1600 nt with qualities up to 93.  Every output is compared exactly with the CPU oracle, which is pinned on
the reference's goldens, and, where oracle/_ref was built, with the compiled reference on a subset.  One subprocess with
a timeout per step; each prints the regimes it ran and its wall time."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HEAD = textwrap.dedent('''
    import os, sys, time
    sys.path.insert(0, %r)
    import numpy as np
    from tests import length_cases as LC
    from oracle import port, ref
    REF = ref.available()
    T0 = time.time()
    def done(name, regimes):
        print("%%s: %%s; %%.1f s wall" %% (name, ", ".join(regimes), time.time() - T0), flush=True)
''') % ROOT

MERGE = textwrap.dedent('''
    from dada2_b200 import merge, Dada2bError
    from tests import merge_cases as M
    OPTS = M.golden()["meta"]["opts"]
    def check(pool, s1, s2, pref, o, sample=1, with_ref=0):
        got = merge.merge_align(pool, s1, s2, pref, **o)
        for x in range(0, len(s1), sample):
            w = port.merge_pair(pool[s1[x]], pool[s2[x]], prefer=int(pref[x]), **o)
            g = (int(got["nmatch"][x]), int(got["nmismatch"][x]), int(got["nindel"][x]), got["sequence"][x])
            assert g == (w["nmatch"], w["nmismatch"], w["nindel"], w["sequence"]), (o, x, g, w)
            if REF and x < with_ref:
                r = ref.merge_pair(pool[s1[x]], pool[s2[x]], prefer=int(pref[x]), **o)
                assert g == (r["nmatch"], r["nmismatch"], r["nindel"], r["sequence"]), (o, x, g, r)
        return got
    def refused(pool, s1, s2, pref, o):
        try:
            merge.merge_align(pool, s1, s2, pref, **o)
        except Dada2bError as e:
            assert "N-W Align out of range" in str(e), e
            return True
        return False
    regimes = []
    # MiSeq 2 x 300 over 400-480 nt amplicons: every option set; banded sets leave the band here, as in the reference
    pool, s1, s2, pref = LC.miseq_pairs(1500, seed=5)
    for o in OPTS:
        if o.get("band", -1) >= 0:
            assert refused(pool, s1, s2, pref, o), o
            with_err = 0
            for x in range(20):
                try:
                    port.merge_pair(pool[s1[x]], pool[s2[x]], **o)
                except RuntimeError:
                    with_err += 1
            assert with_err > 0
        else:
            got = check(pool, s1, s2, pref, o, with_ref=200)
    acc = sum(1 for x in range(len(s1)) if got["nmatch"][x] >= 12 and got["nmismatch"][x] + got["nindel"][x] == 0)
    regimes.append("miseq 2x300 1500 pairs x %d option sets (%d merge exactly)" % (len(OPTS), acc))
    # the scratch switch, unbanded: a batch entirely below, one entirely above, and one mixing both
    sw = LC.scratch_switch(-1)
    lo, hi = LC.merge_batch_at(sw - 1, 400, seed=1), LC.merge_batch_at(sw, 400, seed=2)
    n0 = len(lo[0])
    mixed = (lo[0] + hi[0], np.concatenate([lo[1], hi[1] + n0]), np.concatenate([lo[2], hi[2] + n0]), np.concatenate([lo[3], hi[3]]))
    for name, b in (("below", lo), ("above", hi), ("mixed", mixed)):
        lens = [len(s) for s in b[0]]
        cls = LC.nw_layout(max(lens), min(lens), -1)
        assert cls == ("smem" if name == "below" else "global"), (name, cls)
        for o in OPTS:
            if o.get("band", -1) < 0:
                check(*b, o, with_ref=50)
        regimes.append("unbanded maxlen %d (%s, %s)" % (max(lens), name, cls))
    # band 16 over equally long reads, at the switch and one below, overlaps within the band
    sw = LC.scratch_switch(16)
    for L in (sw - 1, sw):
        b = LC.merge_batch_at(L, 200, seed=L, overlap=(L - 10, L), equal=True)
        lens = [len(s) for s in b[0]]
        cls = LC.nw_layout(max(lens), min(lens), 16)
        assert cls == ("smem" if L < sw else "global"), (L, cls)
        for o in OPTS:
            check(*b, dict(o, band=16), sample=3, with_ref=10)
        regimes.append("band 16 maxlen %d (%s)" % (L, cls))
    done("merge", regimes)
    print("MERGE OK")
''')

BIMERA = textwrap.dedent('''
    from dada2_b200 import bimera
    VARIANTS = ("0", "1", "2")
    def pairs(seqs, q, p, label, with_ref=0, **sc):
        want = [port.bimera_pair(seqs[a], seqs[b], allow_one_off=True, **sc) for a, b in zip(q, p)]
        want = np.array([[w["left"], w["right"], w["left_oo"], w["right_oo"], w["ham"]] for w in want], np.int32)
        if REF:
            for n in range(min(with_ref, len(q))):
                r = ref.bimera_pair(seqs[q[n]], seqs[p[n]], allow_one_off=True, **sc)
                assert list(want[n]) == [r["left"], r["right"], r["left_oo"], r["right_oo"], r["ham"]], (label, n)
        for v in VARIANTS:
            os.environ["DADA2B_BIMFWD"] = v
            got = bimera.test_bimera_pairs(seqs, q, p, allow_one_off=True, **sc)
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert len(bad) == 0, (label, "DADA2B_BIMFWD=" + v, bad[:5], got[bad[:3]], want[bad[:3]])
    regimes = []
    # the 16-bit kernel's int16 headroom, at the default scores and two others
    for sc, spread in ((dict(), 5), (dict(match=2, mismatch=-7, gap_p=-10), 5), (dict(match=5, mismatch=-40, gap_p=-8), 0)):
        s = dict(match=5, mismatch=-4, gap_p=-8); s.update(sc)
        top = LC.bim16_maxlen(s["match"], s["mismatch"], s["gap_p"])
        routes = [LC.bim_route(L, L - spread, 16, s["match"], s["mismatch"], s["gap_p"]) for L in (top, top + 1)]
        assert routes == ["k_bimfwd16", "k_bimfwd"], (s, top, routes)
        for L in (top, top + 1):
            seqs, q, p = LC.bimera_pairs_at(L, spread, 40, seed=L)
            pairs(seqs, q, p, "int16 %s L=%d" % (s, L), with_ref=20, **s)
        regimes.append("int16 headroom %d/%d at %d/%d/%d" % (top, top + 1, s["match"], s["mismatch"], s["gap_p"]))
    # slot classes: V3-V4 lengths with spreads on each side of every class bound
    for bound, below, above in LC.slot_spreads(16):
        cls = [LC.bim_class(LC.bim_slots(440, 440 - d, 16)) for d in (below, above)]
        assert cls[0][0] == bound and (cls[1] is None or cls[1][0] > bound), (bound, cls)
        for d in (below, above):
            seqs, q, p = LC.bimera_pairs_at(440, d, 60, seed=bound * 1000 + d)
            pairs(seqs, q, p, "slots bound %d spread %d" % (bound, d), with_ref=10)
        regimes.append("slots %d: spread %d/%d" % (bound, below, above))
    # PacBio pairs with a real length spread, wider bands
    seqs, q, p = LC.bimera_pairs_at(1560, 40, 30, seed=77)
    for ms in (16, 32):
        pairs(seqs, q, p, "pacbio max_shift %d" % ms, with_ref=10, max_shift=ms)
    regimes.append("pacbio pairs 1520-1560 nt")
    # whole tables and isBimeraDenovo
    for name, (seqs, mat) in (("v3-v4", LC.v34_table(400, 8, seed=4)), ("pacbio", LC.pacbio_table(120, 4, seed=5))):
        ab = mat.sum(axis=0)
        for o in (dict(), dict(allow_one_off=True)):
            want = port.table_bimera(mat, seqs, **o)
            if REF and name == "pacbio":
                r = ref.table_bimera(mat, seqs, **o)
                assert np.array_equal(r[0], want[0]) and np.array_equal(r[1], want[1]), (name, o)
            oo = o.get("allow_one_off", False)
            want_dn = np.zeros(len(seqs), bool)
            for i in range(len(seqs)):
                pars = np.nonzero((ab > 2 * ab[i]) & (ab > 8))[0]
                if len(pars) >= 2:
                    want_dn[i] = port.is_bimera(seqs[i], [seqs[k] for k in pars], allow_one_off=oo)
            for v in VARIANTS:
                os.environ["DADA2B_BIMFWD"] = v
                got = bimera.C_table_bimera2(mat, seqs, **o)
                assert np.array_equal(got["nflag"], want[0]) and np.array_equal(got["nsam"], want[1]), (name, o, v)
                dn = bimera.isBimeraDenovo(seqs, ab, allowOneOff=oo)
                assert np.array_equal(dn, want_dn), (name, o, v, np.nonzero(dn != want_dn)[0][:5])
        lens = [len(s) for s in seqs]
        regimes.append("%s table %d seqs %d-%d nt (%d flagged, %d denovo)" % (name, len(seqs), min(lens), max(lens), int((want[0] > 0).sum()), int(want_dn.sum())))
    done("bimera x DADA2B_BIMFWD=0/1/2", regimes)
    print("BIMERA OK")
''')

COLLAPSE = textwrap.dedent('''
    from dada2_b200 import seqtab, Dada2bError
    from tests import collapse_ref as R
    def pairs(seqs, q, r, label, sample=1, with_ref=0, **o):
        out = seqtab.test_collapse_pairs(seqs, q, r, **o)
        sc = {k: o[k] for k in ("match", "mismatch", "gap") if k in o}
        for x in range(0, len(q), sample):
            a, b = seqs[q[x]], seqs[r[x]]
            w = R.port_nwhamming(a, b, vec=o["vec"], band=o["band"], **sc)
            assert out[x, 2] == w, (label, o, x, out[x], w)
            assert out[x, 0] == R.screen(a, b, o["minOverlap"]), (label, o, x)
            assert out[x, 1] == R.overlap_filter(a, b, o.get("match", 5), o.get("mismatch", -4), o["band"]), (label, o, x)
            if REF and x < with_ref * sample:
                assert w == R.ref_nwhamming(a, b, vec=o["vec"], band=o["band"], **sc), (label, o, x)
        return out
    regimes = []
    for name, L, n in (("v3-v4", 460, 300), ("pacbio", 1600, 60)):
        seqs, q, r = LC.collapse_pairs_at(L, n, seed=L, spread=60)
        for vec in (True, False):
            for band in (-1, 16):
                out = pairs(seqs, q, r, name, with_ref=10, minOverlap=20, vec=vec, band=band)
        regimes.append("%s pairs %d-%d nt (%d of %d with nwhamming 0)" % (name, L - 60, L, int((out[:, 2] == 0).sum()), n))
    # the alignment kernel's scratch switch (same plan as mergePairs), unbanded
    sw = LC.scratch_switch(-1)
    for L in (sw - 1, sw):
        seqs, q, r = LC.collapse_pairs_at(L, 200, seed=L, spread=20)
        lens = [len(s) for s in seqs]
        assert LC.nw_layout(max(lens), min(lens), -1) == ("smem" if L < sw else "global")
        for vec in (True, False):
            pairs(seqs, q, r, "switch", minOverlap=20, vec=vec, band=-1)
    regimes.append("scratch switch %d/%d" % (sw - 1, sw))
    # the vectorized aligner's int16 limit: default scores with band 16 (unbanded, shared memory runs out first) and
    # a score set that brings it to PacBio lengths
    for sc, band in ((dict(match=5, mismatch=-4, gap=-8), 16), (dict(match=5, mismatch=-20, gap=-30), -1)):
        top = LC.vec_maxlen(**sc)
        assert LC.vec_fits(top, **sc) and not LC.vec_fits(top + 1, **sc)
        for L in (top, top + 1):
            seqs, q, r = LC.collapse_pairs_at(L, 10, seed=L, spread=8)
            if L > top:
                for f in (lambda: seqtab.test_collapse_pairs(seqs, q, r, vec=True, band=band, **sc),
                          lambda: seqtab.collapse_reps(seqs, vec=True, band=band, **sc)):
                    try:
                        f(); raise AssertionError("accepted maxlen %d" % L)
                    except Dada2bError as e:
                        assert LC.VEC_REFUSAL in str(e), e
                pairs(seqs, q, r, "vec=FALSE past the limit", minOverlap=20, vec=False, band=band, **sc)
            else:
                pairs(seqs, q, r, "vec limit", with_ref=2, minOverlap=20, vec=True, band=band, **sc)
        regimes.append("vec limit %d/%d at %s band %d" % (top, top + 1, sc, band))
    # collapseNoMismatch on whole tables against the R loop restated over the CPU port's nwhamming
    for name, (mat, cols) in (("v3-v4", LC.collapse_table(60, seed=6)), ("pacbio", LC.collapse_table(12, seed=7, L=(1400, 1601)))):
        for vec in (True, False):
            for band in (-1, 16):
                m, c = seqtab.collapseNoMismatch(mat, cols, vec=vec, band=band)
                wm, wc = R.collapse(mat, cols, vec=vec, band=band, nwhamming=R.port_nwhamming)
                assert c == wc and np.array_equal(m, wm), (name, vec, band)
        regimes.append("%s table %d columns -> %d" % (name, len(cols), len(c)))
    done("collapse", regimes)
    print("COLLAPSE OK")
''')

DEREP = textwrap.dedent('''
    import dada2_b200
    from dada2_b200 import derep, Dada2bError
    from oracle import derep as O
    from tests import derep_cases as D
    from tests import cases
    regimes = []
    for L in LC.DEREP_LENGTHS:
        nreads = 20000 if L <= 300 else (4000 if L <= 1500 else 150)
        s, q = LC.derep_reads(L, 200 if L <= 300 else 40, nreads, seed=L, qmax=93)
        for n in (1000000, 997):
            D.assert_same(derep.derep_reads(s, q, n=n), O.derep_reads(s, q, n=n), "L=%d n=%d" % (L, n))
        regimes.append("%d x %d nt" % (nreads, L))
    s, q = LC.derep_reads(LC.SEQLEN, 2, 4, seed=1)
    try:
        derep.derep_reads(s, q); raise AssertionError("accepted %d nt" % LC.SEQLEN)
    except Dada2bError as e:
        assert str(e) == LC.DEREP_REFUSAL, e
    regimes.append("%d nt refused" % LC.SEQLEN)
    # the resident hand-off into dada() at 1.5 kb against the two-call form
    s, q = LC.derep_reads(1500, 30, 3000, seed=15, qmax=40)
    d, res = derep.derep_reads(s, q, resident=True)
    a = res.run(cases.tperr1())
    res.close()
    b = dada2_b200.dada_uniques(d["uniques"], d["abundances"], None, cases.tperr1(), d["quals"])
    cases.assert_same(a, b, rtol=0, label="derep_resident 1.5 kb")
    regimes.append("resident hand-off 1500 nt, %d uniques -> %d ASVs" % (len(d["uniques"]), len(a["clustering"]["sequence"])))
    done("derep", regimes)
    print("DEREP OK")
''')

FILTER = textwrap.dedent('''
    from dada2_b200 import filter as fl
    from tests import filter_cases as G
    from tests import filter_ref as R
    ph = G.phix()
    regimes = []
    rd = LC.pacbio_reads(3000, seed=8, phix=ph)
    for phx in (True, False):
        o = R.Opts(minLen=1000, maxLen=1600, maxEE=2, rm_phix=phx)
        case = {"name": "pacbio phix=%s" % phx, "opts": [o], "reads": rd, "orient": LC.PACBIO_PRIMER, "n": 100000}
        want = G.want_from_restatement(case)
        G.check_case(case, G.run_product(case, fl.filter_reads), want)
        regimes.append("pacbio 3000 reads 950-1700 nt phix=%s (reasons %s)" % (phx, np.bincount(want[0], minlength=13).tolist()))
    sub = {"name": "pacbio stages", "opts": [R.Opts(minLen=1000, maxLen=1600, maxEE=2, rm_phix=True)], "reads": rd[:600],
           "orient": LC.PACBIO_PRIMER, "n": 100000}
    G.check_stages(sub, fl.test_filter_stages)
    if R.ref_lib() is not None:
        st = fl.test_filter_stages([r[0] for r in rd], [np.array(r[1], np.uint8) for r in rd], orient_fwd=LC.PACBIO_PRIMER, phix=G.PHIX_FA,
                                   **{k: v for k, v in sub["opts"][0].kw().items() if k != "rm_phix"})
        idx = [i for i in range(len(rd)) if st[i]["trim_fail"] == 0 and not st[i]["flipped"]][:1500]
        qs = [rd[i][1][st[i]["start"]:st[i]["end"]] for i in idx]
        assert [x.hex() for x in R.ref_matrix_ee(qs)] == [float(st[i]["ee"]).hex() for i in idx]
        regimes.append("EE of %d trimmed reads = compiled C_matrixEE" % len(idx))
    pr = LC.miseq_read_pairs(6000, seed=9)
    for tl in ((280, 220), (300, 300)):
        ops = [R.Opts(truncLen=tl[0], maxEE=2, maxN=0), R.Opts(truncLen=tl[1], maxEE=2, maxN=0, trimLeft=10)]
        case = {"name": "miseq truncLen=%s" % (tl,), "opts": ops, "reads": pr, "orient": None, "n": 2500}
        want = G.want_from_restatement(case)
        G.check_case(case, G.run_product(case, fl.filter_reads), want)
        regimes.append("miseq 6000 pairs 2x300 truncLen=%s (reasons %s)" % (tl, np.bincount(want[0], minlength=13).tolist()))
    done("filter", regimes)
    print("FILTER OK")
''')


STEPS = {"merge": (MERGE, 600), "bimera": (BIMERA, 900), "collapse": (COLLAPSE, 900), "derep": (DEREP, 600), "filter": (FILTER, 600)}


@pytest.mark.parametrize("step", list(STEPS))
def test_lengths(step):
    body, timeout = STEPS[step]
    out = subprocess.run([sys.executable, "-c", HEAD + body], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    print(out.stdout)
    assert out.returncode == 0 and step.upper() + " OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
