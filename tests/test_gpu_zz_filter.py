"""The read filter's kernels (dd_filter.cu) on hardware, through the C-ABI of include/dada2b_filter.h: every golden case
and the stage hook on them; then a seeded set of 2 x 10^6 paired 250-nt reads whose reason codes must equal the
restated predicates applied, vectorised, to the hook's per-stage values (20 000 sampled pairs also end to end against
tests/filter_ref.py, EE against the compiled reference where it is present); then the vignette's filterAndTrim call on
sam1F / sam1R, whose output files must equal the restatement's byte for byte and feed derepFastq -> dada_uniques.
Runs in a subprocess with a timeout."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import gzip, math, os, sys, tempfile, time
    sys.path.insert(0, %r)
    import numpy as np
    from tests import filter_cases as G
    from tests import filter_ref as R
    from tests import cases
    import dada2_b200
    from dada2_b200 import filter as fl, derep
    g = G.load_golden()
    for case in G.all_cases():
        G.check_case(case, G.run_product(case, fl.filter_reads), G.want_from_golden(g, case))
    for case in G.single_cases():
        G.check_stages(case, fl.test_filter_stages)
    G.check_errors_and_helpers()
    print("goldens ok", flush=True)

    # ---- 2 x 10^6 pairs ----
    N, L = 2000000, 250
    t0 = time.time()
    rd = [G.synthetic_reads(N, L, seed=s) for s in (1, 2)]
    print("generated %%.1f s" %% (time.time() - t0), flush=True)
    ph = G.phix()
    optsF = R.Opts(trimLeft=10, truncLen=240, maxN=0, maxEE=2, rm_lowcomplex=6)
    optsR = R.Opts(trimLeft=5, truncLen=200, truncQ=3, maxN=1, minQ=4, maxEE=3, rm_phix=True)
    kw = {k: (optsF.kw()[k], optsR.kw()[k]) for k in optsF.kw()}
    t0 = time.time()
    got = fl.filter_reads(rd[0], None, (rd[1], None), phix=G.PHIX_FA, **kw)
    print("filter %%d pairs: %%.1f s wall" %% (N, time.time() - t0), got["stats"], flush=True)
    st = [fl.test_filter_stages(rd[m], None, phix=G.PHIX_FA, **{k: v for k, v in o.kw().items() if k != "rm_phix"})
          for m, o in enumerate((optsF, optsR))]
    want_reason, want_flags = G.vector_reasons(st, (optsF, optsR))
    assert np.array_equal(got["reason"], want_reason), np.nonzero(got["reason"] != want_reason)[0][:10]
    assert np.array_equal(got["flags"], want_flags)
    assert np.array_equal(got["src"], np.nonzero(want_reason == 0)[0])
    print("reasons", np.bincount(got["reason"], minlength=13).tolist(), flush=True)
    rng = np.random.default_rng(7)
    sample = np.sort(rng.choice(N, 20000, replace=False))
    sub = [(G.read_at(rd[0], i), G.read_at(rd[1], i)) for i in sample]
    r_reason, r_flags, r_out = R.filter_chunks(sub, [optsF, optsR], None, ph, 10 ** 9)
    assert np.array_equal(got["reason"][sample], r_reason) and np.array_equal(got["flags"][sample], r_flags)
    pos = {int(s): k for k, s in enumerate(got["src"])}
    for src, mates in r_out:
        k = pos[int(sample[src])]
        for m in range(2):
            r = got["reads"][m]
            a, b = r.off[k], r.off[k + 1]
            assert r.seq[a:b].decode() == mates[m][0] and list(r.qual[a:b]) == mates[m][1]
    for m, o in enumerate((optsF, optsR)):
        ok = st[m]["trim_fail"][sample] == 0
        for i in sample[ok][:2000]:
            s, q = G.read_at(rd[m], i)
            sv = st[m][i]
            w = q[sv["start"]:sv["end"]]
            assert float(sv["ee"]).hex() == R.matrix_ee(w).hex()
        if R.ref_lib() is not None:
            idx = sample[ok][:5000]
            qs = [G.read_at(rd[m], i)[1][st[m][i]["start"]:st[m][i]["end"]] for i in idx]
            assert [x.hex() for x in R.ref_matrix_ee(qs)] == [float(st[m][i]["ee"]).hex() for i in idx]
            ws = [G.read_at(rd[m], i)[0][st[m][i]["start"]:st[m][i]["end"]] for i in idx]
            assert np.array_equal(R.ref_match_ref(ws, ph, 16, True), st[m]["hits_fwd"][idx])
            assert np.array_equal(R.ref_match_ref(ws, R.rc(ph), 16, True), st[m]["hits_rc"][idx])
    print("large set ok", flush=True)

    # ---- the vignette's call ----
    gd = os.path.join(%r, "tests", "golden")
    with tempfile.TemporaryDirectory() as d:
        fF, fR = os.path.join(d, "F.fastq.gz"), os.path.join(d, "R.fastq.gz")
        io = dada2_b200.filterAndTrim(os.path.join(gd, "sam1F.fastq.gz"), fF, os.path.join(gd, "sam1R.fastq.gz"), fR, trimLeft=10,
                                      truncLen=(240, 200), maxN=0, maxEE=2, phix=G.PHIX_FA)
        print("filterAndTrim", io.tolist(), flush=True)
        idsF, a = fl.read_fastq_records(os.path.join(gd, "sam1F.fastq.gz"))
        idsR, b = fl.read_fastq_records(os.path.join(gd, "sam1R.fastq.gz"))
        pairs = [(G.read_at(a, i), G.read_at(b, i)) for i in range(len(a))]
        o1, o2 = R.Opts(trimLeft=10, truncLen=240, maxN=0, maxEE=2), R.Opts(trimLeft=10, truncLen=200, maxN=0, maxEE=2)
        _, _, out = R.filter_chunks(pairs, [o1, o2], None, ph, 100000)
        assert io.tolist() == [[len(a), len(out)]]
        for m, (path, ids) in enumerate(((fF, idsF), (fR, idsR))):
            want = R.fastq_bytes([ids[s] for s, _ in out], [x[1][m][0] for x in out], [x[1][m][1] for x in out])
            assert gzip.open(path).read() == want, m
        for path in (fF, fR):
            dr = derep.derepFastq(path)
            res = dada2_b200.dada_uniques(dr["uniques"], dr["abundances"], None, cases.tperr1(), dr["quals"])
            print(path[-10:], len(dr["uniques"]), "uniques ->", len(res["clustering"]["sequence"]), "ASVs", flush=True)
    print("FILTER OK")
''') % (ROOT, ROOT)


def test_filter_matches_goldens_predicates_and_vignette():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0 and "FILTER OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
