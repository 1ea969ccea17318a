"""Writes tests/golden/nwalign.npz: the rows and C_eval_pair counts of the reference's own compiled aligners
(oracle/_ref's ref_align: nwalign_vectorized2 with end gap 0 and with end gap = gap, nwalign_endsfree,
nwalign_endsfree_homo and the global nwalign) on tests/nwalign_cases.inputs(), in bands -1, 0, 8 and 32."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref  # noqa: E402
from tests import collapse_ref as R  # noqa: E402
from tests import nwalign_cases as N  # noqa: E402


def main():
    A, B = N.inputs()
    out = {"s1": np.array(A), "s2": np.array(B)}
    for mode in N.MODES:
        for band in N.BANDS:
            rows = [ref.align(a, b, band=band, mode=mode, homo_gap=N.HOMO_GAP) for a, b in zip(A, B)]
            out[N.key(mode, band, "al1")] = np.array([r[0] for r in rows])
            out[N.key(mode, band, "al2")] = np.array([r[1] for r in rows])
            out[N.key(mode, band, "counts")] = np.array([R.eval_pair(*r) for r in rows], np.int32).reshape(-1, 3)
    np.savez_compressed(N.GOLDEN, **out)
    print(N.GOLDEN, len(A), "pairs", os.path.getsize(N.GOLDEN), "bytes")


if __name__ == "__main__":
    main()
