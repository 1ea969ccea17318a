"""Pair sets at long-read lengths for dada()'s aligners, on both sides of every length-driven switch of the core, and the check
that runs them through the stage hooks dada2b_test_pairs (k_classify + k_align) and dada2b_test_loop_nw (k_nwrow<EXACT>, k_nwlane,
k_nwfwd, k_nwrow<BOUND>) against the reference's alignments.

The switches, each restated below from the host code that applies it:
  * k_nwfwd's branch-free interior (fast_ok, dd_driver.cu): allowed while maxlen * max(|mismatch|, |match|) + max(|gap|, |homo_gap|)
    + 16 stays below half the sentinel (-9999 scalar, INT16_MIN - min(mismatch, gap, match, 0) vectorized);
  * k_nwfwd's instantiation (launch_nwfwd, dd_nwfwd.cu): slot class of fwd_slots, the G = 4 / ND = 10 kernel for large rounds in
    the narrowest class, and the 160 KB of shared memory each instantiation may use;
  * k_align's move matrix in shared memory or in global scratch (setup_params, dd_driver.cu);
  * the thread-per-pair row kernels' score headroom (nwrow_applicable, dd_nwrow.cu).
Every case sits at first_len(...) - 1 or first_len(...) of one of them; make_cases asserts that the two uploads of a pair of
cases fall on different sides, so a change of a formula in the host code fails here instead of quietly moving the cases.

Lambda is a sequential fp64 product over the raw's positions (compute_lambda_ts, pval.cpp:144-197).  The lambda cases choose
substitution counts, qualities and err so that lambda lands in the normal range, just above and just below DBL_MIN, deep in the
subnormals and at exact 0; every kernel must round the subnormal product as the reference does.  lambda_ts restates the product
from the reference's alignment strings; lambda_exact gives the same product in 256-bit arithmetic.

A case: dict(label, seqs (raw 0 is the centre of every pair), quals, err, opts, hints (njobs_hint values for k_nwfwd), edge
(threshold name, side)).
"""
import math

import numpy as np

from tests import bound_ref as BR
from tests import length_cases as LC

DBL_MIN = BR.DBL_MIN
SMALL_HINT, BIG_HINT = 1, 1 << 40       # njobs_hint: below / above num_sms * 512 on any device
DEFAULTS = dict(match=5, mismatch=-4, gap=-8, homo_gap=None, band_size=16, vectorized_alignment=True, use_quals=True)


def _o(opts):
    o = dict(DEFAULTS)
    o.update(opts)
    if o["homo_gap"] is None:
        o["homo_gap"] = o["gap"]
    return o


# ---------------------------------------------------------------------------------------------------------------------
# The host formulas
# ---------------------------------------------------------------------------------------------------------------------
def sentinel(opts):
    """setup_params: -9999 for the scalar aligner (nwalign_endsfree.cpp), (int16_t)(INT16_MIN - m) for the vectorized one."""
    o = _o(opts)
    if o["vectorized_alignment"]:
        m = min(o["mismatch"], o["gap"], o["match"], 0)
        return ((-32768 - m + 32768) % 65536) - 32768
    return -9999


def homo(opts):
    """setup_params: homopolymer gap costs (scalar aligner only)."""
    o = _o(opts)
    return (not o["vectorized_alignment"]) and o["homo_gap"] != o["gap"] and o["homo_gap"] <= 0


def fast_ok(maxlen, opts):
    """Run::launch_compare / do_test_loop_nw: k_nwfwd's branch-free interior is allowed for this upload."""
    o = _o(opts)
    worst = maxlen * max(abs(o["mismatch"]), abs(o["match"])) + max(abs(o["gap"]), abs(o["homo_gap"])) + 16
    return worst < abs(sentinel(o)) // 2


def fwd_slots(maxlen, minlen, band):
    """setup_params: band slots k_nwfwd must hold for the upload's widest pair."""
    if band < 0:
        return 1 << 20
    lbmax = min(band + (maxlen - minlen), maxlen)
    return min(2 * band + (maxlen - minlen) + 3, ((lbmax + 1) & ~1) + lbmax + 1)


FWD_CLASSES = (40, 48, 64, 128, 256)


def fwd_instantiation(slots, hint, num_sms):
    """launch_nwfwd: (G, ND) of the kernel for `slots`, or None past the last class."""
    big = hint > num_sms * 512
    if slots <= 40:
        g = (4, 10) if big else (8, 6)
    elif slots <= 48:
        g = (8, 6)
    elif slots <= 64:
        g = (8, 8)
    elif slots <= 128:
        g = (16, 8)
    elif slots <= 256:
        g = (32, 8)
    else:
        return None
    return g if g[0] * g[1] >= slots else None


def fwd_smem(G, maxlen, Q):
    ppw = 32 // G
    sb = (maxlen + 15) & ~15
    return (16 * Q + 2) * 8 + sb + 4 * ppw * (4 * sb + 4 * 64)


def fwd_fits_smem(G, ND, maxlen, Q):
    """launch_nwfwd: the instantiation's dynamic shared memory stays within 160 KB (ND does not enter it)."""
    return fwd_smem(G, maxlen, Q) <= 160 * 1024


def fwd_takes(maxlen, minlen, Q, hint, num_sms, opts):
    """k_nwfwd runs for this upload (launch_nwfwd returns true); every pair of a banded upload then fits its band."""
    band = _o(opts)["band_size"]
    if band < 0:
        return False
    gnd = fwd_instantiation(fwd_slots(maxlen, minlen, band), hint, num_sms)
    return gnd is not None and fwd_fits_smem(gnd[0], gnd[1], maxlen, Q)


def fwd_smem_limit(G, Q):
    """The smallest maxlen at which instantiation G no longer fits its shared memory."""
    return LC.first_len(lambda L: not fwd_fits_smem(G, 0, L, Q), lo=16, hi=40000)


def align_layout(maxlen, minlen, band, Q):
    """setup_params: k_align's move matrix in shared memory ("smem") while fixed + 16 (base_words + ptr_words) <= 56 KB, else in
    global scratch ("global"); refused beyond 200 KB."""
    lbmax = maxlen if band < 0 else min(band + (maxlen - minlen), maxlen)
    wmax = 2 * lbmax + 1
    nchunk = (((wmax + 1) >> 1) + 31) >> 5
    seq_bytes = (maxlen + 15) & ~15
    h_words = (wmax + 2 + 3) & ~3
    ops_words = ((2 * maxlen) // 16 + 2 + 3) & ~3
    ptr_words = (2 * maxlen + 2) * 2 * nchunk
    base = 2 * (seq_bytes // 4) + h_words + ops_words
    fixed = 16 * Q * 8 + 16 * Q * 4
    if fixed + 16 * (base + ptr_words) <= 56 * 1024:
        return "smem"
    return "global" if fixed + 16 * base <= 200 * 1024 else "refused"


def align_ptr_in_smem(maxlen, band, minlen=None, Q=41):
    return align_layout(maxlen, maxlen if minlen is None else minlen, band, Q) == "smem"


def nwrow_applicable(len1, opts):
    """nwrow_applicable (dd_nwrow.cu): plain gap costs, band 8 / 16 / 32 narrower than the centre, score headroom."""
    o = _o(opts)
    band = o["band_size"]
    if homo(o) or band not in (8, 16, 32) or not (band + 2 <= len1 < 16000) or o["match"] < 0:
        return False
    amax = max(abs(o["match"]), abs(o["mismatch"]), abs(o["gap"]))
    return (abs(o["match"]) + amax) * len1 + 80 * (amax + abs(o["match"])) < 15000


def handled(which, maxlen, minlen, len1, len2, Q, hint, num_sms, opts):
    """Whether dada2b_test_loop_nw's kernel `which` takes the pair (centre of length len1, raw of length len2) of this upload.
    The row / lane kernels need their scratch (allocated when nwrow_applicable(maxlen)) and take raws as long as the centre."""
    if which == 2:
        return fwd_takes(maxlen, minlen, Q, hint, num_sms, opts)
    return nwrow_applicable(maxlen, opts) and nwrow_applicable(len1, opts) and len1 == len2


# ---------------------------------------------------------------------------------------------------------------------
# Lambda
# ---------------------------------------------------------------------------------------------------------------------
NTI = {"A": 0, "C": 1, "G": 2, "T": 3}


def _factors(al0, al1, q1, err, use_quals):
    """compute_lambda_ts' factor per raw position, in raw order: err[4 nt0 + nt1][q] at a substitution, err[5 nt1][q] elsewhere."""
    out = []
    i1 = 0
    for a, b in zip(al0, al1):
        if b == "-":
            continue
        q = int(q1[i1]) if use_quals else 0
        row = 4 * NTI[a] + NTI[b] if a != "-" else 5 * NTI[b]
        out.append(float(err[row, q]))
        i1 += 1
    return out


def lambda_ts(al0, al1, q1, err, use_quals=True):
    """compute_lambda_ts restated: lambda = 1.0, then lambda = lambda * factor over the raw's positions in order, in fp64."""
    lam = 1.0
    for f in _factors(al0, al1, q1, np.asarray(err, np.float64), use_quals):
        lam = lam * f
    return lam


def lambda_exact(al0, al1, q1, err, use_quals=True):
    """The same product in 256-bit floating point (mpmath): -> (mpf, number of factors)."""
    import mpmath
    f = _factors(al0, al1, q1, np.asarray(err, np.float64), use_quals)
    with mpmath.workprec(256):
        p = mpmath.mpf(1)
        for x in f:
            p *= mpmath.mpf(x)
    return p, len(f)


def check_lambda_restatement(al0, al1, q1, err, lam, use_quals=True):
    """lambda_ts equals the reference's lambda bit for bit.  In the normal range the fp64 product is also within ncols * 2^-53
    relative of the exact one; below DBL_MIN each step rounds to a coarser grid and no such bound holds: there only bit identity
    with the sequential product counts."""
    import mpmath
    mine = lambda_ts(al0, al1, q1, err, use_quals)
    assert _bits(mine) == _bits(lam), (mine, lam)
    if lam >= DBL_MIN:
        exact, n = lambda_exact(al0, al1, q1, err, use_quals)
        with mpmath.workprec(256):
            rel = abs((mpmath.mpf(lam) - exact) / exact)
            assert rel <= n * mpmath.mpf(2) ** -53, (lam, float(exact), n)


def _bits(x):
    return int(np.float64(x).view(np.uint64))


def regime(lam):
    if lam == 0:
        return "zero"
    if lam < 1e-315:
        return "deep_subnormal"
    if lam < DBL_MIN:
        return "below_min" if lam >= DBL_MIN / 2 ** 20 else "subnormal"
    if lam < DBL_MIN * 2 ** 20:
        return "above_min"
    return "normal"


# ---------------------------------------------------------------------------------------------------------------------
# Sequences
# ---------------------------------------------------------------------------------------------------------------------
def _rs(rng, L):
    return LC.rand_seq(rng, L)


def _fit(rng, s, L):
    return s[:L] if len(s) >= L else s + LC.rand_seq(rng, L - len(s))


def _quals(rng, seqs, lo, hi):
    L = max(len(s) for s in seqs)
    q = np.full((len(seqs), L), np.nan)
    for i, s in enumerate(seqs):
        q[i, :len(s)] = rng.integers(lo, hi + 1, len(s)).astype(np.float64)
    return q


def _distinct(seqs):
    seen, out = set(), []
    for s in seqs:
        if s not in seen:
            seen.add(s)
            out.append(s)
    return out


def pair_set(rng, L, n, spread=0, maxsub=30, indels=True):
    """A centre of length L - spread // 2 (L when spread = 0) and n distinct raws: substitution variants, some with a 1-3 nt indel or
    a homopolymer edit, at lengths in [L - spread, L], one of each end length."""
    lc = L - spread // 2
    root = _rs(rng, L + 8)
    c = root[:lc]
    seqs = [c, c[:L - spread] if spread else LC.substitute(rng, c, 1), _fit(rng, root, L)]
    k = 0
    while len(seqs) < n + 1:
        s = LC.substitute(rng, root, int(rng.integers(0, maxsub)))
        if indels and k % 3 == 1:
            s = LC.indel(rng, s, 10, L - 10)
        elif indels and k % 3 == 2:
            s = LC.homopolymer_edit(rng, s)
        ln = lc if (spread == 0 or k % 4 == 0) else int(rng.integers(L - spread, L + 1))
        seqs = _distinct(seqs + [_fit(rng, s, ln)])
        k += 1
    if seqs[1] == c:
        seqs[1] = LC.substitute(rng, c, 2)
    return seqs


def _case(label, seqs, quals, err, opts, hints, edge):
    err = np.asarray(err, np.float64)
    return dict(label=label, seqs=list(seqs), quals=quals, err=err, opts=dict(opts), hints=list(hints), edge=edge)


def lambda_case(rng, L, n, err, q_base, q_low, opts, label):
    """Substitution-only raws of a centre of length L (so that the alignment is the diagonal), with k substitutions and m positions
    at quality q_low, chosen so that the planned lambda = self(q_base)^(L - k - m) self(q_low)^m sub^k walks across the normal
    range, both sides of DBL_MIN, the subnormals and exact 0.  The reference's lambda, not the plan, decides the regime."""
    uq = _o(opts)["use_quals"]
    qb = q_base if uq else 0
    ql = q_low if uq else 0
    s_b = math.log2(err[0, qb])
    s_l = math.log2(err[0, ql])
    sub = math.log2(err[1, qb])
    c = _rs(rng, L)
    seqs, qrows = [c], [np.full(L, float(q_base))]
    targets = ([-100, -600] + [-1022 + d for d in (6, 3, 1, 0.3)] + [-1022 - d for d in (0.3, 1, 3, 6)] +
               [-1040, -1070, -1073, -1074.2, -1075.5, -1080, -1200])
    step = s_b - sub                                   # log2 lambda drops by this much per substitution
    for t in targets:
        found = None
        for k in range(1, L // 2):
            base = (L - k) * s_b + k * sub
            if base < t - step:
                break
            if uq:
                m = int(round((t - base) / (s_l - s_b)))
                if 0 <= m <= L - k and abs(base + m * (s_l - s_b) - t) < 0.5:
                    found = (k, m)
                    break
            elif abs(base - t) <= step / 2:
                found = (k, 0)
                break
        if found is None:
            continue
        k, m = found
        pos = rng.choice(L, k + m, replace=False)
        s = list(c)
        for p in pos[:k]:
            s[p] = "ACGT"[(NTI[s[p]] + 1 + int(rng.integers(0, 3))) % 4]
        q = np.full(L, float(q_base))
        q[pos[k:]] = float(q_low)
        seqs.append("".join(s))
        qrows.append(q)
    keep = {}
    for s, q in zip(seqs, qrows):
        keep.setdefault(s, q)
    seqs = list(keep)
    while len(seqs) < n + 1:
        s = LC.substitute(rng, c, int(rng.integers(1, 40)))
        if s not in keep:
            seqs.append(s)
            keep[s] = np.full(L, float(q_base))
    quals = np.stack([keep[s] for s in seqs])
    return _case(label, seqs, quals, err, opts, (SMALL_HINT, BIG_HINT), ("lambda", None))


def lambda_err(Q, q_base, q_low, self_base, sub_base, self_low):
    """err with every column tperr1-like except two: q_base (self_base, sub_base for every substitution) and q_low (self_low)."""
    from tests import cases
    from tools import synth
    e = synth.extend_err(cases.tperr1(), Q).copy()
    for b in range(4):
        for a in range(4):
            e[4 * a + b, q_base] = self_base if a == b else sub_base
        e[5 * b, q_low] = self_low
    return e


def make_cases(scale="gpu", num_sms=132, scores=None):
    """All pair sets.  scale 'gpu': the lengths of the host formulas at default scores; 'emu': the same switches, with scores and an
    err table that bring them to lengths the host emulator aligns in seconds (EMU_SCORES, EMU_Q), and fewer raws."""
    from tests import cases
    from tools import synth
    emu = scale == "emu"
    n = 6 if emu else 40
    sc = dict(EMU_SCORES if emu else {}) if scores is None else dict(scores)
    err = cases.tperr1()
    Q = EMU_Q if emu else 41
    err_smem = synth.extend_err(err, Q)
    out = []
    rng = np.random.default_rng(2024)

    def q_for(seqs, lo=20, hi=40):
        return _quals(rng, seqs, lo, hi)

    # 1. k_nwfwd's interior fast path, scalar (plain and homopolymer gap costs) and vectorized
    for name, o, band in (("scalar", dict(vectorized_alignment=False), 16), ("scalar+homo", dict(vectorized_alignment=False, homo_gap=-1), 16),
                          ("vectorized", dict(), 32)):
        o = dict(sc, band_size=band, **o)
        sw = LC.first_len(lambda L: not fast_ok(L, o), lo=32, hi=40000)
        assert fast_ok(sw - 1, o) and not fast_ok(sw, o)
        for L in (sw - 1, sw):
            seqs = pair_set(rng, L, n)
            out.append(_case("fast_ok %s, %d nt, band %d" % (name, L, band), seqs, q_for(seqs), err, o, (SMALL_HINT,),
                             ("fast_ok " + name, fast_ok(L, o))))
    # 2. k_nwfwd's shared-memory limit per instantiation, ragged raws whose spread lands in each slot class
    for bound in FWD_CLASSES:
        spread = LC.first_len(lambda d: fwd_slots(5000, 5000 - d, 16) > bound, lo=0, hi=1000) - 1
        assert fwd_slots(5000, 5000 - spread, 16) <= bound < fwd_slots(5000, 4999 - spread, 16)
        for hint in ((SMALL_HINT, BIG_HINT) if bound == 40 else (SMALL_HINT,)):
            G, ND = fwd_instantiation(fwd_slots(5000, 5000 - spread, 16), hint, num_sms)
            lim = fwd_smem_limit(G, Q)
            if lim > (1400 if emu else 6000):                # G = 32: its limit lies past the lengths the int16 aligner covers
                lens = (400,) if emu else (4700,)
            else:
                lens = (lim - 1, lim)
            for L in lens:
                seqs = pair_set(rng, L, n, spread=spread)
                assert max(map(len, seqs)) - min(map(len, seqs)) == spread
                out.append(_case("slot class <= %d (G=%d ND=%d), %d nt, spread %d" % (bound, G, ND, L, spread), seqs, q_for(seqs), err_smem,
                                 dict(sc, band_size=16), (hint,), ("smem G=%d ND=%d" % (G, ND), fwd_fits_smem(G, ND, L, Q))))
    # 3. k_align's move matrix in shared memory / global scratch
    for band in (16, 32):
        sw = LC.first_len(lambda L: not align_ptr_in_smem(L, band, Q=err.shape[1]), lo=band + 4, hi=20000)
        for L in (sw - 1, sw):
            seqs = pair_set(rng, L, n)
            out.append(_case("k_align move matrix, %d nt, band %d" % (L, band), seqs, q_for(seqs), err, dict(sc, band_size=band),
                             (SMALL_HINT, BIG_HINT), ("ptr_in_smem band %d" % band, align_ptr_in_smem(L, band, Q=err.shape[1]))))
    # 4. bands 8 / 16 / 32 and unbanded at PacBio length
    Lb = 300 if emu else 1500
    for band in (8, 16, 32, -1):
        seqs = pair_set(rng, Lb, n, spread=4)
        out.append(_case("band %d, %d nt" % (band, Lb), seqs, q_for(seqs), err, dict(sc, band_size=band), (SMALL_HINT, BIG_HINT),
                         ("band", band)))
    # 5. lambda: normal, both sides of DBL_MIN, subnormal, 0; quality 93 as the last column of a 94-column err; use_quals = FALSE
    Ll = 200 if emu else 1000
    e94 = lambda_err(94, 93, 11, 1 - 2.0 ** -11 - 1e-9, 1.1e-20 / 3, 0.61)     # few substitutions: the alignments stay gap-free
    out.append(lambda_case(rng, Ll, 2 * n, e94, 93, 11, dict(band_size=16), "lambda regimes, %d nt, Q 93 of 94 columns" % Ll))
    e0 = lambda_err(41, 0, 0, 0.9973, 2.1e-12, 0.9973)
    out.append(lambda_case(rng, 300 if emu else 2500, 2 * n, e0, 0, 0, dict(band_size=16, use_quals=False),
                           "lambda regimes, use_quals = FALSE"))
    return out


EMU_SCORES = dict(match=5, mismatch=-40, gap=-8)     # fast_ok near 124 nt scalar, 408 nt vectorized; row kernels to 252 nt
EMU_Q = 900                                          # a 900-column err fills k_nwfwd's shared memory: its limits fall at 300-700 nt


# ---------------------------------------------------------------------------------------------------------------------
# The check
# ---------------------------------------------------------------------------------------------------------------------
def _ops_to_strings(ops, nops, a, b):
    al0, al1, i, j = [], [], 0, 0
    for c in ops[:nops]:
        if c == 1:
            al0.append(a[i]); al1.append(b[j]); i += 1; j += 1
        elif c == 2:
            al0.append("-"); al1.append(b[j]); j += 1
        elif c == 3:
            al0.append(a[i]); al1.append("-"); i += 1
        else:
            raise AssertionError("bad op %d" % c)
    assert i == len(a) and j == len(b)
    return "".join(al0), "".join(al1)


def expected(case):
    """Per raw: the reference's sub_new + compute_lambda_ts (oracle.ref.pair, the reference's own C++) when it is built, the CPU
    restatement (oracle.port.pair) otherwise; the restated lambda is checked against it on the way."""
    if "_want" in case:
        return case["_want"]
    from oracle import port, ref
    o = _o(case["opts"])
    uq = o["use_quals"]
    qi = BR.round_quals(case["quals"])
    seqs = case["seqs"]
    kw = dict(match=o["match"], mismatch=o["mismatch"], gap=o["gap"], homo_gap=o["homo_gap"], band_size=o["band_size"],
              vectorized_alignment=o["vectorized_alignment"], use_kmers=False)
    want = []
    for r in range(1, len(seqs)):
        q0 = qi[0, :len(seqs[0])].astype(np.uint8)
        q1 = qi[r, :len(seqs[r])].astype(np.uint8)
        if ref.available():
            p = ref.pair(seqs[0], q0 if uq else None, seqs[r], q1 if uq else None, case["err"], **kw)
        else:
            p = port.pair(seqs[0], q0, seqs[r], q1 if uq else None, case["err"], use_quals=uq, **kw)
        check_lambda_restatement(p["al0"], p["al1"], q1, case["err"], p["lam"], uq)
        want.append(p)
    case["_want"] = want
    return want


def check_case(res, case, num_sms, log=None):
    """test_pairs and every loop kernel over (centre 0, raw r) for every raw; -> counts per kernel and lambda regime."""
    o = _o(case["opts"])
    seqs = case["seqs"]
    n = len(seqs) - 1
    lens = np.array([len(s) for s in seqs])
    maxlen, minlen = int(lens.max()), int(lens.min())
    Q = case["err"].shape[1]
    uq = o["use_quals"]
    want = expected(case)
    centre = np.zeros(n, np.uint32)
    raw = np.arange(1, n + 1, dtype=np.uint32)
    tag = case["label"]
    got = res.test_pairs(centre, raw, case["err"], use_kmers=False, kdist_cutoff=0.42, maxlen=maxlen, **case["opts"])
    counts = {"k_align": 0}
    regimes = {}
    for k in range(n):
        w = want[k]
        r = k + 1
        assert got["kind"][k] == (1 if o["band_size"] == 0 else 2), (tag, r, got["kind"][k])
        al = _ops_to_strings(got["ops"][k], got["nops"][k], seqs[0], seqs[r])
        assert al == (w["al0"], w["al1"]), "%s: raw %d alignment differs" % (tag, r)
        ns = int(got["nsubs"][k])
        assert ns == w["nsubs"], (tag, r, ns, w["nsubs"])
        assert list(got["pos"][k, :ns]) == list(w["pos"]), (tag, r)
        assert bytes((got["nt0"][k, :ns] + 1).astype(np.uint8)) == w["nt0"], (tag, r)
        assert bytes((got["nt1"][k, :ns] + 1).astype(np.uint8)) == w["nt1"], (tag, r)
        if uq:
            assert list(got["q1"][k, :ns]) == list(w["q1"]), (tag, r)
        assert _bits(got["lam"][k]) == _bits(w["lam"]), "%s: raw %d lambda %r, reference %r" % (tag, r, got["lam"][k], w["lam"])
        counts["k_align"] += 1
        g = regime(w["lam"])
        regimes[g] = regimes.get(g, 0) + 1
    names = {0: "k_nwrow<EXACT>", 1: "k_nwlane", 2: "k_nwfwd", 3: "k_nwrow<BOUND>"}
    for which in (0, 1, 2, 3):
        for hint in (case["hints"] if which == 2 else (SMALL_HINT,)):
            r = res.test_loop_nw(which, centre, raw, case["err"], njobs_hint=hint, **case["opts"])
            pred = np.array([handled(which, maxlen, minlen, len(seqs[0]), len(seqs[i]), Q, hint, num_sms, o) for i in raw])
            bad = np.flatnonzero(r["handled"].astype(bool) != pred)
            assert len(bad) == 0, "%s: %s hint %d handles raws %s against the prediction %s" % (tag, names[which], hint, raw[bad[:5]], pred[bad[:5]])
            on = np.flatnonzero(pred)
            for k in on:
                assert r["nsubs"][k] == got["nsubs"][k], (tag, names[which], k + 1, r["nsubs"][k], got["nsubs"][k])
                if which != 3:
                    assert _bits(r["lam"][k]) == _bits(got["lam"][k]), (tag, names[which], k + 1, r["lam"][k], got["lam"][k])
            key = names[which]
            if which == 2:
                gnd = fwd_instantiation(fwd_slots(maxlen, minlen, o["band_size"]), hint, num_sms) if o["band_size"] >= 0 else None
                key = "k_nwfwd<%d,%d,%s>" % (gnd + ("homo" if homo(o) else "exact",)) if gnd else "k_nwfwd<none>"
                if gnd and len(on):
                    key += " fast" if fast_ok(maxlen, o) else " checked"
            counts[key] = counts.get(key, 0) + len(on)
            counts[key + " handed on"] = counts.get(key + " handed on", 0) + n - len(on)
    rec = dict(label=tag, edge=case["edge"], maxlen=maxlen, fast_ok=fast_ok(maxlen, o), layout=align_layout(maxlen, minlen, o["band_size"], Q),
               counts=counts, regimes=regimes)
    if log:
        log("%s | maxlen %d, fast_ok %s, k_align %s | %s | lambda %s" % (tag, maxlen, rec["fast_ok"], rec["layout"],
            ", ".join("%s %d" % kv for kv in counts.items()), regimes))
    return rec


def run_cases(make_resident, cases, num_sms, log=None):
    recs = []
    for case in cases:
        res = make_resident(case["seqs"], np.ones(len(case["seqs"]), np.int32), None, case["quals"])
        try:
            recs.append(check_case(res, case, num_sms, log))
        finally:
            res.close()
    return recs


def check_coverage(recs, one_sided=("smem G=32 ND=8",)):
    """Both sides of every threshold were reached (apart from the limits in `one_sided`, which lie past the lengths the cases
    reach), every k_nwfwd instantiation compared pairs, and lambda reached every regime."""
    sides = {}
    for r in recs:
        name, side = r["edge"]
        if name not in ("band", "lambda"):
            sides.setdefault(name, set()).add(side)
    for name, s in sides.items():
        assert s == ({True} if name in one_sided else {True, False}), (name, s)
    tot, reg = {}, {}
    for r in recs:
        for k, v in r["counts"].items():
            tot[k] = tot.get(k, 0) + v
        for k, v in r["regimes"].items():
            reg[k] = reg.get(k, 0) + v
    for G, ND in ((4, 10), (8, 6), (8, 8), (16, 8), (32, 8)):
        assert any(k.startswith("k_nwfwd<%d,%d,exact>" % (G, ND)) and not k.endswith("handed on") and v > 0 for k, v in tot.items()), (G, ND, tot)
    assert tot.get("k_nwfwd<8,6,homo> fast", 0) > 0 and tot.get("k_nwfwd<8,6,homo> checked", 0) > 0, tot
    for k in ("k_nwrow<EXACT>", "k_nwlane", "k_nwrow<BOUND>"):
        assert tot.get(k, 0) > 0, (k, tot)
    for g in ("normal", "above_min", "below_min", "deep_subnormal", "zero"):
        assert reg.get(g, 0) > 0, (g, reg)
    return tot, reg


# ---------------------------------------------------------------------------------------------------------------------
# End to end
# ---------------------------------------------------------------------------------------------------------------------
def longread_sample(seed, n, L, spread, nvar=5, Q=94, maxsub=30):
    """n distinct uniques at lengths in [L - spread, L] (one exactly L): reads of nvar substitution variants of one root (Zipf
    abundances) with 0-2 errors each, homopolymer indels and substitutions, cut or padded back into the length window.  CCS-like
    qualities: mostly Q - 1, some 20 .. Q - 2.  -> (seqs, abundances, quals)"""
    rng = np.random.default_rng(seed)
    root = LC.rand_seq(rng, L + 8)
    variants = [root] + [LC.substitute(rng, root, int(rng.integers(2, maxsub))) for _ in range(nvar - 1)]
    w = 1.0 / np.arange(1, nvar + 1)
    w /= w.sum()
    table = {}
    top = _fit(rng, root, L)
    table[top] = 1
    while len(table) < n:
        v = variants[int(rng.choice(nvar, p=w))]
        for _ in range(int(rng.integers(0, 3))):
            v = LC.homopolymer_edit(rng, v) if rng.random() < 0.6 else LC.substitute(rng, v, 1)
        ln = L - spread // 2 if spread == 0 or rng.random() < 0.7 else int(rng.integers(L - spread, L + 1))
        s = _fit(rng, v, ln)
        table[s] = table.get(s, 0) + 1
    seqs = sorted(table, key=lambda s: (-table[s], s))
    ab = np.array([table[s] for s in seqs], np.int32)
    q = np.full((len(seqs), L), np.nan)
    for i, s in enumerate(seqs):
        row = np.where(rng.random(len(s)) < 0.85, Q - 1, rng.integers(20, Q - 1, len(s)))
        q[i, :len(s)] = row.astype(np.float64)
    return seqs, ab, q


def e2e_samples(scale="gpu"):
    """Small long-read samples for dada_uniques: -> [(label, seqs, abundances, quals, err, opts, edges)]
      * PacBio-length uniques near the vectorized aligner's fast_ok switch, in k_nwfwd's widest slot class;
      * uniques whose comparisons underflow lambda to exact 0 (a 94-column err whose substitutions at quality 93 are 1e-60): p = 0
        births.  The upload sits past the G = 4 / ND = 10 kernel's shared-memory limit and inside G = 8's, so a round that counts as
        large (DADA2B_SMS=1) runs its bound pass and exact pass without k_nwfwd and hands the whole NW list to k_align;
      * the scalar aligner with homopolymer gap costs, one upload on each side of its fast_ok switch."""
    from tests import cases
    from tools import synth
    emu = scale == "emu"
    out = []
    sc = dict(EMU_SCORES) if emu else {}
    Qe = EMU_Q if emu else 94
    # 1.
    o = dict(sc, band_size=16)
    sw = LC.first_len(lambda L: not fast_ok(L, o), lo=32, hi=40000)
    L = sw if not emu else sw - 1
    spread = 100 if not emu else 60
    seqs, ab, q = longread_sample(11, 24 if emu else 80, L, spread)
    out.append(("long uniques %d-%d nt" % (L - spread, L), seqs, ab, q, synth.extend_err(cases.tperr1(), 94), o,
                dict(fast_ok=fast_ok(L, o), slots=fwd_slots(L, L - spread, 16))))
    # 2.
    err = synth.extend_err(cases.tperr1(), Qe).copy()
    for a in range(4):
        for b in range(4):
            if a != b:
                err[4 * a + b, 93] = 1e-60
    g4, g8 = fwd_smem_limit(4, Qe), fwd_smem_limit(8, Qe)
    L = g4 + 40
    assert L < g8
    seqs, ab, q = longread_sample(12, 20 if emu else 60, L, 4, maxsub=12)
    out.append(("lambda underflow, %d nt, past the G=4 shared-memory limit" % L, seqs, ab, q, err, dict(sc, band_size=16),
                dict(g4_fits=fwd_fits_smem(4, 10, L, Qe), g8_fits=fwd_fits_smem(8, 6, L, Qe))))
    # 3.
    o = dict(sc, band_size=16, vectorized_alignment=False, homo_gap=-1)
    sw = LC.first_len(lambda L: not fast_ok(L, o), lo=32, hi=40000)
    for L in (sw - 1, sw):
        seqs, ab, q = longread_sample(13, 20 if emu else 50, L, 4)
        out.append(("scalar + homopolymer gaps, %d nt" % L, seqs, ab, q, synth.extend_err(cases.tperr1(), 94), o,
                    dict(fast_ok=fast_ok(L, o))))
    return out


def check_e2e(dada_uniques, sample, log=None):
    """dada_uniques against the CPU oracle (every output, screen counts) and, when built, the reference's own dada_uniques."""
    from oracle import port, ref
    from tests import cases
    label, seqs, ab, q, err, opts, edges = sample
    o = _o(opts)
    got = dada_uniques(seqs, ab, None, err, q, **opts)
    want = port.dada_uniques(seqs, ab, None, err, q, **o)
    cases.assert_same(got, want, rtol=1e-10, label=label)
    cases.assert_same_screen_counts(got, want, label=label)
    if ref.available():
        cases.assert_same(got, ref.dada_uniques(seqs, ab, None, err, q, **o), rtol=1e-10, label=label + " (reference)")
    bp = np.asarray(got["clustering"]["birth_pval"])
    info = dict(label=label, nclust=len(bp), p0_births=int((bp[1:] == 0).sum()), **edges)
    if log:
        log("e2e %s" % info)
    return info
