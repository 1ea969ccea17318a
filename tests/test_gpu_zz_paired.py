"""mergePairs over whole samples (dd_pairs.cu + dd_merge.cu, include/dada2b_merge.h) on the H100 against the restatement
(tests/paired_ref.py), field by field: the sam1 / sam2 paired fixtures through filterAndTrim -> derepFastq -> dada() ->
mergePairs -> makeSequenceTable, per-sample and pooled; then ~50 synthetic samples of 2 x 250 nt reads at real amplicon
lengths in one and in several batches.  In a subprocess with a timeout, like the other GPU tests."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import os, sys, tempfile, time
    sys.path.insert(0, %r)
    import numpy as np
    import dada2_b200
    from dada2_b200 import derep
    from tests import cases, filter_cases as G, paired_cases as P, paired_ref as R

    def check(got, sets, label, **kw):
        for i, (g, c) in enumerate(zip(got, sets)):
            R.assert_same(g, R.merge_sample(*c, **kw), "%%s sample %%d" %% (label, i))

    # ---- (a) the paired fixtures, vignette style ----
    gd = os.path.join(%r, "tests", "golden")
    with tempfile.TemporaryDirectory() as d:
        drF, drR = [], []
        for sam in ("sam1", "sam2"):
            fF, fR = os.path.join(d, sam + "F.fastq.gz"), os.path.join(d, sam + "R.fastq.gz")
            io = dada2_b200.filterAndTrim(os.path.join(gd, sam + "F.fastq.gz"), fF, os.path.join(gd, sam + "R.fastq.gz"), fR,
                                          truncLen=(240, 160), maxEE=2, phix=G.PHIX_FA)
            print(sam, "filterAndTrim", io.tolist(), flush=True)
            drF.append(derep.derepFastq(fF)); drR.append(derep.derepFastq(fR))
        tperr1 = cases.tperr1()
        for pool in (False, True):
            ddF = dada2_b200.dada(drF, err=tperr1, pool=pool, verbose=False)
            ddR = dada2_b200.dada(drR, err=tperr1, pool=pool, verbose=False)
            sets = list(zip(ddF, drF, ddR, drR))
            for kw in (dict(), dict(returnRejects=True, propagateCol=("n0", "birth_ham")), dict(maxMismatch=1, trimOverhang=True),
                       dict(justConcatenate=True)):
                got = dada2_b200.mergePairs(ddF, drF, ddR, drR, **kw)
                check(got, sets, "sam pool=%%s %%s" %% (pool, kw), **kw)
            mg = dada2_b200.mergePairs({"sam1": ddF[0], "sam2": ddF[1]}, {"sam1": drF[0], "sam2": drF[1]},
                                       {"sam1": ddR[0], "sam2": ddR[1]}, {"sam1": drR[0], "sam2": drR[1]})
            mat, cols, rows = dada2_b200.seqtab.makeSequenceTable(mg)
            assert rows == ["sam1", "sam2"] and mat.shape[1] == len(set(mg["sam1"]["sequence"]) | set(mg["sam2"]["sequence"]))
            assert mat.sum() == sum(int(m["abundance"].sum()) for m in mg.values())
            print("sam pool=%%s: %%s pairings accepted, seqtab %%s" %% (pool, [len(m["sequence"]) for m in mg.values()], mat.shape), flush=True)
        # fastq paths as derep inputs
        one = dada2_b200.mergePairs(ddF[0], os.path.join(d, "sam1F.fastq.gz"), ddR[0], os.path.join(d, "sam1R.fastq.gz"))
        R.assert_same(one, R.merge_sample(ddF[0], drF[0], ddR[0], drR[0]), "paths")
    print("fixtures ok", flush=True)

    # ---- (b) ~50 synthetic samples x 2e5 reads, 2 x 250 nt over 253..480 nt amplicons ----
    t0 = time.time()
    sets = P.synth_set(48, 200000, seed=3, namp=16)
    print("synthetic set built in %%.1f s" %% (time.time() - t0), flush=True)
    args = [list(x) for x in zip(*sets)]
    allm = None
    for batch in (None, "1000000"):
        if batch is None:
            os.environ.pop("DADA2B_PAIRS_BATCH", None)
        else:
            os.environ["DADA2B_PAIRS_BATCH"] = batch
        for kw in (dict(returnRejects=True), dict(), dict(maxMismatch=1, trimOverhang=True, returnRejects=True, propagateCol=("n0",)),
                   dict(justConcatenate=True)):
            t0 = time.time()
            got, st = dada2_b200.mergePairs(*args, return_stats=True, **kw)
            t1 = time.time()
            check(got, sets, "synthetic batch=%%s %%s" %% (batch, kw), **kw)
            t2 = time.time()
            if kw == dict(returnRejects=True):
                allm = allm or [R.merge_sample(*c, returnRejects=True) for c in sets]
                assert st["n_aligned"] == R.distinct_triples(args[0], args[2], allm)
                assert st["n_pairings"] == sum(len(m["forward"]) for m in allm)
            print("batch=%%s %%s: %%d reads, %%d pairings, %%d aligned, %%d batches; k_tab %%.2f ms, k_merge %%.2f ms, native %%.1f ms, "
                  "mergePairs %%.2f s, restatement %%.2f s" %% (batch, kw, st["n_reads"], st["n_pairings"], st["n_aligned"], st["n_batches"],
                  st["ms_k_tab"], st["ms_k_merge"], st["ms_total"], t1 - t0, t2 - t1), flush=True)
    print("PAIRED OK")
''') % (ROOT, ROOT)


def test_merge_pairs_matches_restatement_on_fixtures_and_synthetic_samples():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=1500)
    print(out.stdout[-6000:])
    assert out.returncode == 0 and "PAIRED OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
