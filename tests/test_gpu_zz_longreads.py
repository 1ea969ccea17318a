"""BASELINE config 5 flavour (PacBio-like ~1.5 kb uniques, BAND_SIZE=32, homopolymer gap penalty) at a size the CPU
oracle finishes in seconds.  It runs in a subprocess so that a device fault could not poison the other tests' CUDA context."""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import sys
    sys.path.insert(0, %r)
    import numpy as np
    from tools import synth
    from tests import cases
    from oracle import port
    import dada2_b200
    seqs, ab, q = synth.pacbio(120, L=1500, nvar=6, seed=5)
    err = synth.extend_err(cases.tperr1(), 94)
    for opts in (dict(band_size=32, vectorized_alignment=False, homo_gap=-1),      # nwalign_endsfree_homo path
                 dict(band_size=32)):                                              # vectorized path, ragged lengths
        o = dict(opts); o.setdefault("homo_gap", -8)
        got = dada2_b200.dada_uniques(seqs, ab, None, err, q, **opts)
        want = port.dada_uniques(seqs, ab, None, err, q, **o)
        cases.assert_same(got, want, rtol=1e-10, label=str(opts))
        cases.assert_same_screen_counts(got, want, label=str(opts))
    print("LONGREADS OK")
''') % ROOT


def test_pacbio_like_long_reads_match_oracle():
    out = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "LONGREADS OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
