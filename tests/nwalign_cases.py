"""The nwalign goldens (tests/golden/nwalign.npz, written by tools/make_golden_nwalign.py from the reference's compiled
aligners) and the checks shared by the emulator and GPU suites."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "nwalign.npz")

# reference aligner mode (oracle/ref_shim.cpp ref_align) -> nwalign's arguments
MODES = {0: dict(vec=True), 1: dict(), 2: dict(homo_gap=-3), 4: dict(endsfree=False), 5: dict(vec=True, endsfree=False)}
BANDS = (-1, 0, 8, 32)
HOMO_GAP = -3


def inputs(seed=11):
    """Structured and random pairs from 1 to ~1500 nt: shifts, substitutions, indels, homopolymer runs, periodic repeats,
    length differences larger than the band, and one-base sequences.  -> (list s1, list s2)"""
    rng = np.random.default_rng(seed)

    def rs(n):
        return "".join("ACGT"[i] for i in rng.integers(0, 4, n))

    def mut(s, k):
        s = list(s)
        for p in rng.choice(len(s), min(k, len(s)), replace=False):
            s[p] = "ACGT"[("ACGT".index(s[p]) + 1 + int(rng.integers(0, 3))) % 4]
        return "".join(s)

    A, B = [], []
    for L in (1, 2, 3, 5, 9, 17, 33, 60, 120, 250, 251, 400):
        a = rs(L)
        A += [a, a, a, a]
        B += [mut(a, max(1, L // 20)), a[L // 4:] + rs(L // 4), rs(max(1, L + int(rng.integers(-3, 4)))), a[: max(1, L - 40)]]
    for L in (40, 120, 300):                                              # homopolymer runs
        a = "".join(c * int(rng.integers(1, 7)) for c in rs(L // 3))
        b = list(a)
        for _ in range(3):
            p = int(rng.integers(1, len(b)))
            b.insert(p, b[p - 1]) if rng.random() < 0.5 else b.pop(p)
        A.append(a); B.append("".join(b))
    for unit, n1, n2 in (("ACGT", 20, 23), ("AAC", 30, 27), ("ACGTTGCA", 10, 12), ("AT", 50, 47)):   # periodic repeats
        A.append(unit * n1); B.append((unit * n2)[1:])
    a = rs(200)
    A += [a, a[:60], "A" * 40]                                            # length differences beyond the bands
    B += [a[:60], a, "A" * 3]
    for L in (1000, 1500):                                                # long reads
        a = rs(L)
        A += [a, mut(a, 30)]
        B += [a[7:] + rs(5), a[: L - 200]]
    return A, B


def load():
    return np.load(GOLDEN)


def key(mode, band, what):
    return "m%d_b%d_%s" % (mode, band if band >= 0 else 99, what)


def expected(g, mode, band, x):
    """Golden rows of pair x.  The reference's vectorized ends-free aligner mis-aligns a one-base sequence (it returns a
    mismatch column where an end gap scores higher); nwalign here returns nwalign_endsfree's optimal alignment there."""
    a, b = str(g["s1"][x]), str(g["s2"][x])
    if mode == 0 and min(len(a), len(b)) == 1:
        mode = 1
    return str(g[key(mode, band, "al1")][x]), str(g[key(mode, band, "al2")][x])


def check(nwalign, eval_counts, modes=MODES, bands=BANDS):
    """Every golden pair in every mode and band: the rows of nwalign and the counts of eval_counts."""
    g = load()
    A, B = [str(s) for s in g["s1"]], [str(s) for s in g["s2"]]
    for mode in modes:
        for band in bands:
            got = nwalign(A, B, band=band, **MODES[mode])
            for x in range(len(A)):
                assert got[x] == expected(g, mode, band, x), (mode, band, x, len(A[x]), len(B[x]))
            cnt = eval_counts(A, B, band=band, **MODES[mode])
            want = g[key(mode, band, "counts")].copy()
            if mode == 0:
                one = np.array([min(len(a), len(b)) == 1 for a, b in zip(A, B)])
                want[one] = g[key(1, band, "counts")][one]
            assert np.array_equal(cnt, want), (mode, band)
