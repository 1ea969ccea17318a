"""collapseNoMismatch's kernels (dd_collapse.cu) on hardware, through the C-ABI of include/dada2b_collapse.h: the golden
tables and every golden pair, then a seeded table of about 20 000 V4-like ASVs x 96 samples whose output must equal the
greedy loop run over the pair hook's nwhamming of every candidate pair, with sampled pairs checked against the CPU port.
Runs in a subprocess with a timeout."""
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
    from tests import collapse_ref as R
    from dada2_b200 import seqtab
    G.check_tables(seqtab.collapseNoMismatch)
    G.check_pairs(lambda s, q, r, m, v, b: seqtab.test_collapse_pairs(s, q, r, minOverlap=m, vec=v, band=b))
    print("goldens ok", flush=True)
    mat, cols = G.large_table()
    seqs = R.query_order(mat, cols)
    rep, st = seqtab.collapse_reps(seqs, return_stats=True)
    print("large table", mat.shape, st, flush=True)
    q, r = G.screen_pairs(seqs, 20)
    assert st["n_candidates"] == len(q), (st["n_candidates"], len(q))
    t0 = time.time()
    out = seqtab.test_collapse_pairs(seqs, q, r)
    print("pair hook on %%d candidates: %%.1f s" %% (len(q), time.time() - t0), flush=True)
    assert np.all(out[:, 0] == 1)
    assert not np.any((out[:, 1] == 0) & (out[:, 2] == 0)), "the filter rejected a pair with nwhamming 0"
    assert np.count_nonzero(out[:, 1] == 0) == st["n_filtered"]
    zero = np.nonzero(out[:, 2] == 0)[0]
    assert len(zero) == st["n_zero"]
    want = R.greedy(len(seqs), [(int(q[x]), int(r[x])) for x in zero])
    assert np.array_equal(rep, want)
    rng = np.random.default_rng(3)
    for x in np.concatenate([rng.choice(len(q), 300, replace=False), zero[:100]]):
        assert out[x, 2] == R.port_nwhamming(seqs[q[x]], seqs[r[x]]), x
        assert out[x, 1] == R.overlap_filter(seqs[q[x]], seqs[r[x]]), x
    m, c = seqtab.collapseNoMismatch(mat, cols)
    assert m.shape[1] == int(np.count_nonzero(rep == np.arange(len(rep)))) and m.sum() == mat.sum()
    print("COLLAPSE OK", m.shape)
''') % ROOT


def test_collapse_matches_goldens_and_greedy_loop_at_size():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "COLLAPSE OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
