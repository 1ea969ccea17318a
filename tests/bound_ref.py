"""Plain restatement of the two-phase loop NW's bound (DESIGN.md 9.3) for the stage hooks dada2b_test_raw_bounds / dada2b_test_bound.

A later cluster's loop comparison of (centre, raw) is dropped by the bound pass when
    S_r * rho_r^nsubs * total_reads * (1 + 1e-9) <= E_minmax[r]      (and the product is not below 1e-280),
where S_r is the product of the raw's self-transition factors and rho_r its largest substitution / self ratio (dd_round.cu:k_raw_bounds).
Every alignment with nsubs substitutions has lambda <= S_r * rho_r^nsubs exactly, so such a pair fails the store rule of
cluster.cpp:192 (lambda * total_reads > E_minmax).

raw_factors restates k_raw_bounds' fp64 arithmetic in its own order (the library is built with -fmad=false and IEEE division, so
the device must agree bit for bit).  exact_factors / exact_bound give S*, rho* and B* = S* rho*^ns T as exact rationals over the
err doubles; decision() says which jobs any correct bound pass must keep, which it must drop, and which it may do either with.
"""
import math
from fractions import Fraction

import numpy as np

CODE = {"A": 0, "C": 1, "G": 2, "T": 3}
UNDERFLOW = 1e-280                      # below this the kernels keep the pair: the fp product is no safe bound there
MARGIN = Fraction(1) + Fraction(1, 10 ** 9)
DBL_MIN = 2.2250738585072014e-308
KEEP, DROP, EITHER = 1, 0, 2


def round_quals(quals):
    """(uint8_t) round(q) of containers.cpp:34 as the upload computes it for q >= 0: trunc(q) + (q - trunc(q) >= 0.5), both terms
    exact in fp64 (unlike floor(q + 0.5), which rounds 0.49999999999999994 up).  NaN (beyond a read's end) -> 0."""
    q = np.nan_to_num(np.asarray(quals, dtype=np.float64), nan=0.0)
    t = np.trunc(q)
    return (t + (q - t >= 0.5)).astype(np.int64)


def _codes(seqs, L):
    s = np.zeros((len(seqs), L), np.int64)
    for i, x in enumerate(seqs):
        s[i, :len(x)] = np.frombuffer(x.encode(), np.uint8)
    lut = np.zeros(256, np.int64)
    for c, v in CODE.items():
        lut[ord(c)] = v
    return lut[s]


def raw_factors(seqs, quals, err, use_quals=True):
    """(S, rho) per raw as k_raw_bounds computes them: positions in order, s *= self; rh = fmax(rh, err[4 a0 + b][q] / self) over
    a0 = 0..3, a0 != b (fmax ignores a NaN ratio); the quality rounded as at upload and clamped to ncol - 1; column 0 without quals."""
    err = np.asarray(err, dtype=np.float64)
    ncol = err.shape[1]
    lens = np.array([len(x) for x in seqs])
    L = int(lens.max())
    b = _codes(seqs, L)
    q = np.minimum(round_quals(np.asarray(quals)[:, :L]), ncol - 1) if use_quals else np.zeros((len(seqs), L), np.int64)
    S = np.ones(len(seqs)); rho = np.zeros(len(seqs))
    with np.errstate(divide="ignore", invalid="ignore", under="ignore", over="ignore"):
        for p in range(L):
            on = p < lens
            bp, qp = b[:, p], q[:, p]
            self_ = err[5 * bp, qp]
            S = np.where(on, S * self_, S)
            for a0 in range(4):
                r = err[4 * a0 + bp, qp] / self_
                rho = np.where(on & (a0 != bp), np.fmax(rho, r), rho)
    return S, rho


def raw_factors_loop(seq, qrow, err, use_quals=True):
    """raw_factors for one raw, written as the kernel's loop (the cross-check of the vectorised form)."""
    ncol = err.shape[1]
    s, rh = 1.0, 0.0
    for p, c in enumerate(seq):
        b = CODE[c]
        qq = min(int(qrow[p]), ncol - 1) if use_quals else 0
        self_ = float(err[5 * b, qq])
        s *= self_
        for a0 in range(4):
            if a0 != b:
                num = float(err[4 * a0 + b, qq])
                r = num / self_ if self_ != 0.0 else (math.nan if num == 0.0 else math.inf)
                if not math.isnan(r):
                    rh = max(rh, r)
    return s, rh


def exact_factors(seq, qrow, err, use_quals=True):
    """S* (Fraction) and rho* (Fraction, or math.inf when some used self transition is 0 while a substitution is not) over the err
    doubles, exactly.  Ratios 0 / 0 are ignored, as fmax ignores the NaN."""
    ncol = err.shape[1]
    counts = {}
    for p, c in enumerate(seq):
        k = (CODE[c], min(int(qrow[p]), ncol - 1) if use_quals else 0)
        counts[k] = counts.get(k, 0) + 1
    S = Fraction(1)
    rho = Fraction(0)
    for (b, qq), n in counts.items():
        self_ = Fraction(float(err[5 * b, qq]))
        S *= self_ ** n
        for a0 in range(4):
            if a0 == b:
                continue
            num = Fraction(float(err[4 * a0 + b, qq]))
            if self_ == 0:
                if num != 0:
                    rho = math.inf
            elif rho is not math.inf:
                rho = max(rho, num / self_)
    return S, rho


def exact_bound(S, rho, ns, T):
    """B* = S* rho*^ns T exactly; None where it is undefined (0 * inf)."""
    if rho is math.inf:
        if ns == 0:
            return S * T
        return None if S == 0 else math.inf
    return S * rho ** ns * T


def decision(ns, lam_ref, E, T, B, S_fp=1.0):
    """KEEP: the reference stores the pair (fl(lam_ref T) > E), or B* is below 1e-280 (with a relative margin of 1e-6) or undefined,
    or the raw's fp S_r is 0 (the kernels' bound is then 0 or NaN, which they keep).
    DROP: B* (1 + 1e-9)(1 + 1e-11) <= E and none of the above; for a subnormal S_r, whose sequential product is accurate to about
    1e-7 only, E must clear B* (1 + 1e-9)(1 + 1e-6).  EITHER: everything else."""
    if lam_ref * float(T) > E or B is None or S_fp == 0.0:
        return KEEP
    if B is math.inf:
        return EITHER if E == math.inf else KEEP
    if B < Fraction(UNDERFLOW) * (1 + Fraction(1, 10 ** 6)):
        return KEEP
    if math.isinf(E) and E > 0:
        return DROP
    slack = Fraction(1, 10 ** 6) if S_fp < DBL_MIN else Fraction(1, 10 ** 11)
    if B * MARGIN * (1 + slack) <= Fraction(E):
        return DROP
    return EITHER


def gapless(cseq, rseq, qrow, err, use_quals=True):
    """(nsubs, lambda) of nwalign_gapless (nwalign_endsfree.cpp:539-555) as compute_lambda_ts multiplies it: raw positions in order,
    the raw's base against the centre's (a raw base beyond the centre's end is a self transition)."""
    ncol = err.shape[1]
    lam, ns = 1.0, 0
    for p, c in enumerate(rseq):
        b = CODE[c]
        a = CODE[cseq[p]] if p < len(cseq) else b
        ns += a != b
        lam = lam * float(err[4 * a + b, min(int(qrow[p]), ncol - 1) if use_quals else 0])
    return ns, lam
