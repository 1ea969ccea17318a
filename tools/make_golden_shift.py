"""Writes tests/golden/shift.npz: isShiftDenovo's flags from tests/shift_ref.py (R/chimeras.R:380-421 restated line by
line over the reference's compiled nwalign_endsfree and C_eval_pair) on tests/shift_cases.cases() at every minOverlap of
shift_cases.MIN_OVERLAPS, and (match, mismatch, indel) of every directed (query, more abundant parent) pair."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import shift_cases as K  # noqa: E402
from tests import shift_ref as S  # noqa: E402


def main():
    out = {}
    for name, u in K.cases().items():
        seqs, ab = list(u), np.array(list(u.values()), np.int64)
        out[name + "_seqs"] = np.array(seqs)
        out[name + "_abund"] = ab
        q, p = S.directed_pairs(seqs, ab)
        counts = np.array([S.shifted_pair_counts(seqs[i], seqs[j]) for i, j in zip(q, p)], np.int32).reshape(-1, 3)
        out[name + "_pq"], out[name + "_pp"], out[name + "_counts"] = q, p, counts
        for m in K.MIN_OVERLAPS:
            f = S.is_shift_denovo(u, minOverlap=m)
            out[K.flag_key(name, m)] = np.array([f[s] for s in seqs], bool)
            print(name, len(seqs), "seqs", len(q), "pairs, minOverlap", m, ":", int(out[K.flag_key(name, m)].sum()), "flagged")
    np.savez_compressed(K.GOLDEN, **out)
    print(K.GOLDEN, os.path.getsize(K.GOLDEN), "bytes")


if __name__ == "__main__":
    main()
