"""dada()'s aligners pair by pair at long-read lengths on the H100: every pair set of tests/longpair_cases.py at full size (the
scalar and vectorized fast_ok switches near 995 and 3 272 nt, each k_nwfwd instantiation's shared-memory limit near 1 150, 2 370 and
4 740 nt, k_align's move matrix on both sides of its shared-memory switch, bands 8 / 16 / 32 / unbanded at 1 500 nt, lambda from the
normal range down to subnormal and exact 0) through dada2b_test_pairs and dada2b_test_loop_nw against the reference's alignments
and lambda, bit for bit; then long-read samples through dada_uniques against the oracle and the reference at the default SM count
and at DADA2B_SMS=1 (every later round counts as large).  Prints per-kernel counts of pairs compared and handed on, and the lambda
regimes reached.  In a subprocess with a timeout, like the other zz files, so that a device fault could not poison the other
tests' CUDA context."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

STAGE = textwrap.dedent('''
    import sys, time
    sys.path.insert(0, %r)
    import torch
    import dada2_b200
    from tests import longpair_cases as P
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    t0 = time.time()
    recs = P.run_cases(dada2_b200.Resident, P.make_cases("gpu", num_sms=sms), sms, log=lambda s: print(s, flush=True))
    tot, reg = P.check_coverage(recs)
    for k in sorted(tot):
        print("%%-36s %%d pairs" %% (k, tot[k]))
    print("lambda regimes (pairs):", reg)
    print("total %%.1f s" %% (time.time() - t0))
    print("LONGPAIRS OK")
''') % ROOT

E2E = textwrap.dedent('''
    import sys, time
    sys.path.insert(0, %r)
    import dada2_b200
    from tests import longpair_cases as P
    t0 = time.time()
    infos = [P.check_e2e(dada2_b200.dada_uniques, s, log=lambda s: print(s, flush=True)) for s in P.e2e_samples("gpu")]
    assert infos[1]["p0_births"] > 0 and not infos[1]["g4_fits"] and infos[1]["g8_fits"], infos[1]
    assert [i["fast_ok"] for i in infos[2:]] == [True, False], infos
    print("total %%.1f s" %% (time.time() - t0))
    print("LONGPAIRS E2E OK")
''') % ROOT


def _run(script, env, marker, timeout):
    out = subprocess.run([sys.executable, "-c", script], cwd=ROOT, capture_output=True, text=True, timeout=timeout,
                         env=dict(os.environ, **env))
    print(out.stdout[-8000:])
    assert out.returncode == 0 and marker in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def test_long_pairs_match_reference_pair_by_pair():
    _run(STAGE, {}, "LONGPAIRS OK", 1800)


@pytest.mark.parametrize("sms", [None, "1"])
def test_long_read_samples_match_oracle(sms):
    _run(E2E, {"DADA2B_SMS": sms} if sms else {}, "LONGPAIRS E2E OK", 1800)
