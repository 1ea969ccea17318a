"""The k-mer screen pair by pair on the GPU: every case of tests/screen_cases.py through the stage hook dada2b_test_screen, on both
paths, against the plain restatement tests/screen_ref.py -- plus, at the device's full SM count, more than 4 * 3 * SMs * 128 raws so
that every CTA of k_prescreen reuses every stage of its TMA ring (mbarrier phase parity 1, re-armed stages).  In a subprocess with a
timeout, like the other zz files, so that a device fault could not poison the other tests' CUDA context."""
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
    import torch
    import dada2_b200
    from tests import screen_cases as SC
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for case in SC.small_cases() + [SC.full_grid_case(sms)]:
        t = time.time()
        n = SC.run_case(dada2_b200.Resident, case, sms)
        print("%%s: %%d raws, %%d hook calls, %%.1f s" %% (case["label"], len(case["seqs"]), n, time.time() - t), flush=True)
    print("SCREEN OK")
''') % ROOT


def test_screen_stage_matches_reference_pair_by_pair():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0 and "SCREEN OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
