"""The isShiftDenovo goldens (tests/golden/shift.npz, written by tools/make_golden_shift.py from tests/shift_ref.py's
restated R loop over the reference's compiled aligner) and the checks shared by the emulator and GPU suites."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "shift.npz")
MIN_OVERLAPS = (-1, 0, 1, 20, 50)


def config1_uniques():
    """The denoised clusters of dada(sam1F) (the e2e_config1 golden; R's own example in man/isShiftDenovo.Rd)."""
    g = np.load(os.path.join(HERE, "golden", "e2e_config1.npz"))
    return {str(s): int(a) for s, a in zip(g["clustering__sequence"], g["clustering__abundance"])}


def synthetic(seed=7):
    """Families with true shifts, containments, equal-abundance shifts, periodic sequences with several exact shifts and
    sequences shorter than minOverlap.  -> {sequence: abundance}"""
    rng = np.random.default_rng(seed)

    def rs(n):
        return "".join("ACGT"[i] for i in rng.integers(0, 4, n))

    u = {}

    def put(s, a):
        if s and s not in u:
            u[s] = int(a)

    for f in range(6):
        B = rs(int(rng.integers(80, 160)))
        put(B, 1000 - f)
        put(B[3:] + rs(3), 50 + f)             # true shift (left)
        put(rs(4) + B[:-4], 40 + f)            # true shift (right)
        put(B[5:-5], 30 + f)                   # containment: not a shift
        put(B[:-7], 20 + f)                    # prefix: containment
        put(B[2:] + rs(2), 1000 - f)           # equal abundance to its parent: never compared
        s = list(B[1:] + rs(1)); p = int(rng.integers(20, 60)); s[p] = "ACGT"[("ACGT".index(s[p]) + 1) % 4]
        put("".join(s), 10 + f)                # shift with a substitution: not a shift
        put(B[60:] + rs(60), 5 + f)            # shift with overlap len - 60 (below minOverlap 50 for short B)
    for unit, n in (("ACGT", 30), ("AAC", 40), ("ACGTTGCA", 15)):
        P = unit * n
        put(P, 500)
        put(P[1:] + unit[0], 300)              # periodic: many exact shifts
        put(P[len(unit):], 200)
    for L in (5, 12, 19, 25):
        S = rs(L)
        put(S, 90)
        put(S[2:] + rs(2), 9)                  # short sequences, around minOverlap
    return u


def cases():
    return {"config1": config1_uniques(), "synthetic": synthetic()}


def load():
    return np.load(GOLDEN)


def case(g, name):
    seqs = [str(s) for s in g[name + "_seqs"]]
    return seqs, g[name + "_abund"].astype(np.int64)


def flag_key(name, m):
    return "%s_flags_m%d" % (name, m) if m >= 0 else "%s_flags_mneg%d" % (name, -m)


def check_flags(is_shift_denovo):
    """isShiftDenovo(dict) on every golden case and minOverlap."""
    g = load()
    for name in cases():
        seqs, ab = case(g, name)
        for m in MIN_OVERLAPS:
            got = is_shift_denovo(dict(zip(seqs, (int(a) for a in ab))), minOverlap=m)
            assert np.array_equal(np.asarray(got, bool), g[flag_key(name, m)]), (name, m)


def check_pairs(hook):
    """The stage hook on every directed golden pair: screen, filter and (match, mismatch, indel) of the alignment."""
    from tests import shift_ref as S
    g = load()
    for name in cases():
        seqs, ab = case(g, name)
        q, p = g[name + "_pq"], g[name + "_pp"]
        want = g[name + "_counts"]
        for m in MIN_OVERLAPS:
            out = hook(seqs, q, p, m)
            assert np.array_equal(out[:, 2:], want), (name, m)
            scr = np.array([S.screen(seqs[i], seqs[j], m) for i, j in zip(q, p)], bool)
            assert np.array_equal(out[:, 0].astype(bool), scr), (name, m)
            flt = np.array([S.shift_filter(seqs[i], seqs[j], m) for i, j in zip(q, p)], bool)
            assert np.array_equal(out[:, 1].astype(bool), flt), (name, m)
            sh = (want[:, 0] < np.array([len(seqs[i]) for i in q])) & (want[:, 0] < np.array([len(seqs[j]) for j in p])) & \
                 (want[:, 0] >= m) & (want[:, 1] == 0) & (want[:, 2] == 0)
            assert not np.any(sh & ~out[:, 0].astype(bool)), (name, m, "the screen rejected a shift")
            assert not np.any(sh & ~out[:, 1].astype(bool)), (name, m, "the filter rejected a shift")
