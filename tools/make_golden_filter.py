"""Writes tests/golden/filter.npz: for every case of tests/filter_cases.py, the restated reason codes, flags, source
indices and output reads of tests/filter_ref.py.  Where the compiled reference is present (oracle/_ref, built by
oracle/filter.mk) the restatement's C_matchRef hits and C_matrixEE are asserted equal to it on every read of the pool,
and the reference's values are stored.  The complexity of every read that reaches the rm.lowcomplex stage is asserted
to lie farther than 1e-12 from its threshold unless it is exactly 1.0.

    python tools/make_golden_filter.py
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import filter_cases as G  # noqa: E402
from tests import filter_ref as R  # noqa: E402


def main():
    out = {}
    reads, _ = G.single_pool()
    seqs = [r[0] for r in reads]
    ph = G.phix()
    if R.ref_lib() is None:
        sys.exit("oracle/_ref/libdada2ref_filter.so is not built (python __graft_entry__.py)")
    for w in (1, 8, 15, 16):
        for nov in (True, False):
            for ref in (ph, R.rc(ph)):
                assert np.array_equal(R.ref_match_ref(seqs, ref, w, nov), R.match_ref(seqs, ref, w, nov)), (w, nov)
    ee = R.ref_matrix_ee([r[1] for r in reads])
    assert [x.hex() for x in ee] == [R.matrix_ee(r[1]).hex() for r in reads]
    out["pool/ref_ee"] = ee
    out["pool/ref_hits16"] = R.ref_match_ref(seqs, ph, 16, True)
    out["pool/ref_hits16_rc"] = R.ref_match_ref(seqs, R.rc(ph), 16, True)
    for case in G.all_cases():
        reason, flags, src, mates = G.want_from_restatement(case)
        k = case["name"]
        out[k + "/reason"], out[k + "/flags"], out[k + "/src"] = reason, flags, src
        for m, (s, q) in enumerate(mates):
            off = np.zeros(len(s) + 1, np.int64)
            np.cumsum([len(x) for x in s], out=off[1:])
            out[k + "/off%d" % m] = off
            out[k + "/seq%d" % m] = np.frombuffer("".join(s).encode(), np.uint8)
            out[k + "/qual%d" % m] = np.array([x for y in q for x in y], np.uint8)
        for m, o in enumerate(case["opts"]):
            if o.rm_lowcomplex:
                for r in case["reads"]:
                    s = r[m][0] if len(case["opts"]) == 2 else r[0]
                    cx = R.complexity(s)
                    assert math.isnan(cx) or cx == 1.0 or abs(cx - o.rm_lowcomplex) > 1e-12, (k, cx)
        print(k, len(reason), "->", len(src), np.bincount(reason, minlength=13).tolist())
    np.savez_compressed(G.GOLDEN, **out)
    print("wrote", G.GOLDEN)


if __name__ == "__main__":
    main()
