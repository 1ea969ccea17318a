"""De novo bimera detection (dada2b_denovo_bimera in dd_bimera.cu) and removeBimeraDenovo on hardware: every golden of
tests/golden/removebim.npz (per-sample flags with and without zero-count queries, pooled flags) under each alignment
kernel and across batch boundaries, a 1500-sequence x 12-sample table against the CPU restatement, and
removeBimeraDenovo end to end on every input form, with dada() results and mergePairs mergers of the sam1 / sam2
fixtures.  In a subprocess with a timeout, like the other GPU tests."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import os, sys, tempfile, time
    from concurrent.futures import ProcessPoolExecutor
    sys.path.insert(0, %r)
    import numpy as np
    import dada2_b200
    from dada2_b200 import bimera, derep, removeBimeraDenovo
    from tests import bimera_cases as B, removebim_cases as RC, removebim_ref as R

    # ---- a larger table against the CPU restatement (rows / query chunks spread over the host cores) ----
    def port_rows(args):
        row, seqs, zq, queries = args
        return R.is_bimera_denovo(seqs, row, queries if queries is not None else (None if zq else row > 0), "port")
    from tools import synth
    seqs, mat = synth.bimera_table(1500, 12, seed=9, lenvar=6)
    cs = mat.sum(axis=0, dtype=np.int64)
    with ProcessPoolExecutor(max_workers=max(1, min(32, os.cpu_count() or 1))) as ex:
        t0 = time.time()
        want_ps = np.array(list(ex.map(port_rows, [(r, seqs, False, None) for r in mat])))
        chunks = [np.arange(len(seqs)) %% 24 == c for c in range(24)]
        want_po = np.logical_or.reduce(list(ex.map(port_rows, [(cs, seqs, True, q) for q in chunks])))
        t1 = time.time()
    for name in RC.table_names():
        RC.check_per_sample(name, RC.product_flag_fn)
        RC.check_per_sample(name, RC.product_flag_fn, zero_queries=True)
        RC.check_pooled(name, RC.product_flag_fn)
        B.check_is_bimera(name, B.product_denovo_fn) if name in B.table_names() else None
    os.environ["DADA2B_BIM_JB"] = "7"
    for name in ("t160_ragged", "s_dup"):
        RC.check_per_sample(name, RC.product_flag_fn)
        RC.check_pooled(name, RC.product_flag_fn, opt_ids=[0, 4])
    del os.environ["DADA2B_BIM_JB"]
    print("goldens ok", flush=True)

    got_ps, st_ps = bimera.denovo_bimera(mat, seqs, zero_queries=False, return_stats=True)
    got_po, st_po = bimera.denovo_bimera(cs[None, :], seqs, zero_queries=True, return_stats=True)
    assert np.array_equal(got_ps, want_ps), int((got_ps != want_ps).sum())
    assert np.array_equal(got_po[0], want_po), int((got_po[0] != want_po).sum())
    assert st_ps["n_pairs"] == RC.need_pairs(mat, False) and st_po["n_pairs"] == RC.need_pairs(cs[None, :], True)
    print("1500x12 per-sample: %%d flagged, %%d pairs, %%.1f ms; pooled: %%d flagged, %%d pairs, %%.1f ms; port %%.1f s" %% (
        got_ps.sum(), st_ps["n_pairs"], st_ps["ms_total"], got_po.sum(), st_po["n_pairs"], st_po["ms_total"], t1 - t0), flush=True)

    # ---- removeBimeraDenovo on every input form, from the sam1 / sam2 fixtures ----
    from tests import cases, filter_cases as G
    gd = os.path.join(%r, "tests", "golden")
    with tempfile.TemporaryDirectory() as d:
        drF, drR = [], []
        for sam in ("sam1", "sam2"):
            fF, fR = os.path.join(d, sam + "F.fastq.gz"), os.path.join(d, sam + "R.fastq.gz")
            dada2_b200.filterAndTrim(os.path.join(gd, sam + "F.fastq.gz"), fF, os.path.join(gd, sam + "R.fastq.gz"), fR,
                                     truncLen=(240, 160), maxEE=2, phix=G.PHIX_FA)
            drF.append(derep.derepFastq(fF)); drR.append(derep.derepFastq(fR))
    tperr1 = cases.tperr1()
    ddF = dada2_b200.dada(drF, err=tperr1, verbose=False)
    ddR = dada2_b200.dada(drR, err=tperr1, verbose=False)
    mg = dada2_b200.mergePairs(ddF, drF, ddR, drR)

    def keep_of(seqs, ab, **kw):
        return ~R.is_bimera_denovo(list(seqs), list(ab), **kw)
    for kw in (dict(), dict(allowOneOff=True, minFoldParentOverAbundance=1.5)):
        dn = ddF[0]["denoised"]
        k = keep_of(dn.keys(), dn.values(), **kw)
        assert removeBimeraDenovo(ddF[0], **kw) == {s: a for (s, a), x in zip(dn.items(), k) if x}, ("dada", kw)
        k = keep_of(drF[0]["uniques"], drF[0]["abundances"], **kw)
        want = {s: int(a) for s, a, x in zip(drF[0]["uniques"], drF[0]["abundances"], k) if x}
        assert removeBimeraDenovo(drF[0], **kw) == want, ("derep", kw)
        m = mg[0]
        k = keep_of(m["sequence"], m["abundance"], **kw)
        got = removeBimeraDenovo(m, **kw)
        assert got["sequence"] == [s for s, x in zip(m["sequence"], k) if x] and np.array_equal(got["abundance"], m["abundance"][k]), ("merger", kw)
        both = removeBimeraDenovo({"s1": ddF[0], "s2": ddF[1]}, **kw)
        assert list(both) == ["s1", "s2"] and both["s1"] == removeBimeraDenovo(ddF[0], **kw)
    mat, cols, rows = dada2_b200.seqtab.makeSequenceTable(mg)
    for method in ("consensus", "pooled", "per-sample"):
        out, oc, orows = removeBimeraDenovo((mat, cols, rows), method=method)
        wmat, wcols = R.remove_table(mat, cols, method)
        assert oc == wcols and np.array_equal(out, wmat) and orows == rows, method
        print("seqtab %%s %%s -> %%d columns" %% (mat.shape, method, len(oc)), flush=True)
    print("REMOVEBIM OK")
''') % (ROOT, ROOT)


@pytest.mark.parametrize("variant", ["traceback", "register", "simd16"])
def test_removebim_matches_reference_goldens_and_oracle(variant):
    env = dict(os.environ)
    env["DADA2B_BIMFWD"] = {"traceback": "0", "register": "1", "simd16": "2"}[variant]
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "REMOVEBIM OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
