"""The bound pass of the two-phase loop NW on the H100: every case of tests/bound_cases.py at full size (a k_nwrow<BOUND> list of
more than 16 384 jobs, a round at 1e5 uniques) through the stage hooks dada2b_test_raw_bounds / dada2b_test_bound against the plain
restatement tests/bound_ref.py, and the replay of every NW comparison of syn2000_default's later rounds with the E_minmax each met.
Prints per-kernel counts of kept, dropped and either jobs and the replay's drop fraction.  In a subprocess with a timeout, like the
other zz files, so that a device fault could not poison the other tests' CUDA context."""
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
    import dada2_b200
    from tests import bound_cases as BC
    t0 = time.time()
    for case in BC.all_cases("gpu"):
        t = time.time()
        BC.run_case(dada2_b200.Resident, case, log=lambda s: print(s, flush=True))
        print("%%s: %%d jobs, %%.1f s" %% (case["label"], len(case["jobs"]), time.time() - t), flush=True)
    tot = BC.replay(dada2_b200.Resident, "syn2000_default", log=lambda s: print(s, flush=True))
    for which, (dropped, n) in tot.items():
        assert n > 1000 and dropped > 0.5 * n, (which, dropped, n)
    print("total %%.1f s" %% (time.time() - t0))
    print("BOUND OK")
''') % ROOT


def test_bound_pass_matches_exact_bound_on_round_sized_job_lists():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    print(out.stdout[-6000:])
    assert out.returncode == 0 and "BOUND OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
