"""nwalign's kernel (dd_align.cu) and isShiftDenovo's pipeline (dd_collapse.cu) on hardware: both golden sets; then, on
the seeded ~19 000 ASV table of tests/collapse_cases.large_table() with column sums as abundances, isShiftDenovo's flags
against the any-reduction of the stage hook's predicate over every screened directed pair, sampled pairs against the CPU
port, and the top sequences by abundance against the restated R loop over the compiled reference aligner when
oracle/_ref is present; and nwalign on ~100 000 mixed-length pairs, sampled in every mode.  Runs in a subprocess with a
timeout."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import sys, time
    sys.path.insert(0, %r)
    import numpy as np
    from tests import collapse_cases as G
    from tests import nwalign_cases as N
    from tests import shift_cases as K
    from tests import shift_ref as S
    from dada2_b200 import align, bimera, isShiftDenovo
    from oracle import port, ref
    N.check(align.nwalign, align.eval_counts)
    K.check_flags(isShiftDenovo)
    K.check_pairs(lambda s, q, p, m: bimera.test_shift_pairs(s, q, p, minOverlap=m))
    print("goldens ok", flush=True)

    mat, seqs = G.large_table()
    ab = mat.sum(axis=0, dtype=np.int64)
    flag, st = bimera.shift_flags(seqs, ab, return_stats=True)
    print("large table", len(seqs), st, flush=True)
    assert st["n_candidates"] == st["n_filtered"] + st["n_aligned"] == st["n_screened"] - st["n_equal"]
    q, r = G.screen_pairs(seqs, 20)
    assert st["n_screened"] == len(q), (st["n_screened"], len(q))
    neq = ab[q] != ab[r]
    assert st["n_equal"] == int(np.count_nonzero(~neq))
    q, r = q[neq], r[neq]
    lo = np.where(ab[q] < ab[r], q, r).astype(np.int32)
    hi = np.where(ab[q] < ab[r], r, q).astype(np.int32)
    t0 = time.time()
    out = bimera.test_shift_pairs(seqs, lo, hi)
    print("pair hook on %%d directed pairs: %%.1f s" %% (len(lo), time.time() - t0), flush=True)
    assert np.all(out[:, 0] == 1)
    L = np.array([len(s) for s in seqs])
    sh = (out[:, 2] < L[lo]) & (out[:, 2] < L[hi]) & (out[:, 2] >= 20) & (out[:, 3] == 0) & (out[:, 4] == 0)
    assert not np.any(sh & (out[:, 1] == 0)), "the filter rejected a shift"
    assert np.count_nonzero(out[:, 1] == 0) == st["n_filtered"]
    want = np.zeros(len(seqs), bool)
    want[lo[sh]] = True
    assert np.array_equal(flag.astype(bool), want), (int(flag.sum()), int(want.sum()))
    assert st["n_flagged"] == int(want.sum())
    print("flags ok: %%d flagged, %%d shift pairs" %% (int(want.sum()), int(sh.sum())), flush=True)
    rng = np.random.default_rng(3)
    for x in np.concatenate([rng.choice(len(lo), 300, replace=False), np.nonzero(sh)[0][:50]]):
        a, b = seqs[lo[x]], seqs[hi[x]]
        pm = port.merge_pair(a, b, match=5, mismatch=-4, gap_p=-8)
        assert tuple(out[x, 2:]) == (pm["nmatch"], pm["nmismatch"], pm["nindel"]), x
        assert bool(out[x, 1]) == S.shift_filter(a, b), x
    if ref.available():
        o = np.argsort(-ab, kind="stable")
        k = 400
        while ab[o[k - 1]] == ab[o[k]]:
            k += 1
        top = {seqs[i]: int(ab[i]) for i in o[:k]}
        t0 = time.time()
        f = S.is_shift_denovo(top, minOverlap=20)
        print("restated R loop on the top %%d: %%.1f s" %% (k, time.time() - t0), flush=True)
        assert [f[seqs[i]] for i in o[:k]] == flag[o[:k]].astype(bool).tolist()
        assert isShiftDenovo(top).tolist() == [f[s] for s in top]

    rng = np.random.default_rng(9)
    def rs(n):
        return "".join("ACGT"[i] for i in rng.integers(0, 4, n))
    A, B = [], []
    for x in range(100000):
        l1 = int(rng.choice([int(rng.integers(1, 120)), int(rng.integers(200, 300)), int(rng.integers(400, 1500))], p=[0.3, 0.6, 0.1]))
        a = rs(l1)
        b = a[int(rng.integers(0, 8)):] + rs(int(rng.integers(0, 8))) if rng.random() < 0.6 else rs(max(1, l1 + int(rng.integers(-20, 20))))
        A.append(a); B.append(b or "A")
    pick = rng.choice(len(A), 150, replace=False)
    for mode, kw in N.MODES.items():
        for band in (-1, 16):
            t0 = time.time()
            got = align.nwalign(A, B, band=band, **kw)
            print("nwalign mode %%d band %%d: %%d pairs in %%.1f s" %% (mode, band, len(A), time.time() - t0), flush=True)
            for x in pick:
                if not ref.available():
                    break
                m = 1 if mode == 0 and min(len(A[x]), len(B[x])) == 1 else mode
                assert got[x] == ref.align(A[x], B[x], band=band, mode=m, homo_gap=N.HOMO_GAP), (mode, band, x)
    print("ALIGN OK")
''') % ROOT


def test_nwalign_and_shift_match_goldens_and_restatements_at_size():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert out.returncode == 0 and "ALIGN OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
