"""Primer removal (dd_primer.cu) on hardware, through the C-ABI of include/dada2b_primer.h: every golden case and the hit
hook on them, files and refusals; then 2 x 10^5 seeded CCS-like reads whose hits (5 000 sampled reads) must equal the
restatement's and whose reasons and flips must equal rules 4-7 applied, vectorised, to the hook's hits; then the man
page's removePrimers call on samPBprimers, whose output must equal the restatement's record for record and which is
denoised end to end (filterAndTrim -> derepFastq -> dada with BAND_SIZE 32 and the homopolymer gap penalty, the error
matrix learnt with PacBioErrfun on samPB, resident).  Runs in a subprocess with a timeout."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import gzip, os, sys, tempfile, time
    sys.path.insert(0, %r)
    import numpy as np
    from tests import primer_cases as G
    from tests import primer_ref as R
    import dada2_b200
    from dada2_b200 import primer as pm, filter as fl, derep, errmodel
    g = G.load_golden()
    for case in G.cases():
        G.check_case(case, G.run_product(case, pm.remove_primers_reads), G.want_from_golden(g, case))
        G.check_hits(case, pm.test_primer_hits, g[case["name"] + "/hits"])
    with tempfile.TemporaryDirectory() as d:
        G.check_files(d)
    G.check_errors()
    print("goldens ok", flush=True)

    # ---- 2 x 10^5 CCS-like reads ----
    N = 200000
    t0 = time.time()
    rd, is_rc = G.synthetic_ccs(N, seed=3)
    print("generated %%.1f s" %% (time.time() - t0), flush=True)
    pf, pr = G.F27, R.rc(G.R1492)
    got = pm.remove_primers_reads(rd, None, pf, pr)
    print("removePrimers %%d reads" %% N, got["stats"], flush=True)
    hits = pm.test_primer_hits(rd, None, pf, pr)
    lens = np.diff(rd.off)
    assert not got["skipped"]
    reason, flags = R.vector_decide(hits, lens, True)
    assert np.array_equal(got["reason"], reason), np.nonzero(got["reason"] != reason)[0][:10]
    assert np.array_equal(got["flags"], flags)
    assert np.array_equal(got["src"], np.nonzero(reason == 0)[0])
    print("reasons", np.bincount(got["reason"], minlength=5).tolist(), "flipped", int((flags & 1).sum()), "multi",
          int(((flags & 6) != 0).sum()), "out of limits",
          int(((hits["count"] > 0) & ((hits["first_start"] <= 0) | (hits["last_end"] > lens[:, None]))).any(axis=1).sum()),
          flush=True)
    assert int((flags & 1).sum()) > N // 3 and ((flags & 6) != 0).any()
    sample = np.sort(np.random.default_rng(5).choice(N, 5000, replace=False))
    s = rd.strings()
    sub = [(s[i], list(rd.qual[rd.off[i]:rd.off[i + 1]])) for i in sample]
    for j, i in enumerate(sample):
        want = np.array(R.scans(sub[j][0], pf, pr, 2), np.int32)
        have = np.stack([hits[f][i] for f in ("count", "first_start", "first_end", "last_start", "last_end")], axis=-1)
        assert np.array_equal(have, want), (i, have.tolist(), want.tolist())
    w = R.remove_primers(sub, pf, pr, 2)
    assert np.array_equal(w["reason"], got["reason"][sample]) and np.array_equal(w["flags"], got["flags"][sample])
    pos = {int(x): k for k, x in enumerate(got["src"])}
    r = got["reads"]
    for src, seq, q in w["out"]:
        k = pos[int(sample[src])]
        a, b = r.off[k], r.off[k + 1]
        assert r.seq[a:b].decode() == seq and r.qual[a:b].tolist() == q
    print("large set ok", flush=True)

    # ---- the man page's example, then denoised ----
    with tempfile.TemporaryDirectory() as d:
        nop = os.path.join(d, "noprime.fastq.gz")
        io = dada2_b200.removePrimers(G.SAM_PB_PRIMERS, nop, primer_fwd=pf, primer_rev=pr, orient=True, verbose=True)
        ids, a = fl.read_fastq_records(G.SAM_PB_PRIMERS)
        st = a.strings()
        w = R.remove_primers([(st[i], list(a.qual[a.off[i]:a.off[i + 1]])) for i in range(len(a))], pf, pr, 2)
        assert io.tolist() == [[len(a), len(w["out"])]]
        assert gzip.open(nop).read() == R.fastq_bytes([ids[o[0]] for o in w["out"]], [o[1] for o in w["out"]], [o[2] for o in w["out"]])
        print("samPBprimers", io.tolist(), "flipped", int((w["flags"] & 1).sum()), flush=True)
        filt = [os.path.join(d, "filt_nop.fastq.gz"), os.path.join(d, "filt_pb.fastq.gz")]
        kw = dict(minQ=3, minLen=1000, maxLen=1600, maxN=0, rm_phix=False, maxEE=2)
        io2 = dada2_b200.filterAndTrim([nop, G.SAM_PB], filt, **kw)
        print("filterAndTrim", io2.tolist(), flush=True)
        opts = dict(band_size=32, vectorized_alignment=False, homo_gap=-1)
        sq, qq = derep.read_fastq(filt[1])
        dr, res_pb = derep.derep_reads(sq, qq, resident=True)
        learnt = errmodel.learnErrors(lambda e, mc: res_pb.run(e, max_clust=mc, **opts), ncol=94,
                                      errorEstimationFunction=errmodel.PacBioErrfun)
        err = learnt["err_out"]
        assert err.shape == (16, 94) and np.all(np.isfinite(err))
        print("learnErrors", learnt["passes"], "passes on", len(dr["uniques"]), "uniques", flush=True)
        sq, qq = derep.read_fastq(filt[0])
        dr, res = derep.derep_reads(sq, qq, resident=True)
        out = res.run(err, **opts)
        print("samPBprimers:", len(sq), "reads", len(dr["uniques"]), "uniques ->", len(out["clustering"]["sequence"]), "ASVs", flush=True)
        assert 1 <= len(out["clustering"]["sequence"]) <= len(dr["uniques"])
    print("PRIMER OK")
''') % ROOT


def test_primers_match_goldens_rules_and_man_page_example():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=1500)
    print(out.stdout[-4000:])
    assert out.returncode == 0 and "PRIMER OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
