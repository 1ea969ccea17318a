"""Seeded job lists on both sides of every threshold of the two-phase bound, and the check that runs them through the stage hooks
dada2b_test_raw_bounds / dada2b_test_bound (include/dada2b_test.h) against the plain restatement tests/bound_ref.py.

A case is one uploaded set of raws, an err matrix, options, a centre, the job list (every other raw) and the kernel launches to make:
    dict(label, seqs, reads, quals, err, opts, centre, jobs, kernels=[(which, njobs_hint)], promises)
E_minmax per job is chosen from the job's reference (nsubs, lambda) and its exact bound B* (prepare()):
    -999, nextafter(fl(lam T), -inf), fl(lam T), B* (1 + 1e-9)(1 - 1e-11), B* (1 + 1e-9)(1 + 1e-11) rounded up, +inf
and neighbouring jobs alternate between the "keep" and the "drop" side, so that every warp's ballot is mixed.  `promises` names what
the case must reach (tests/test_bound_ref.py counts it): keep / drop / either jobs, underflow, nan (undefined bound), ns0, mixed warps,
over16k (a list longer than k_nwlane takes).
"""
import math
import os
import subprocess
import sys
import tempfile
import textwrap
from fractions import Fraction

import numpy as np

from tests import bound_ref as BR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LANE_MAX = 16384                        # dd_driver.cu: job lists of at most this many pairs go to k_nwlane
BIG_HINT = 1 << 40                      # njobs_hint that selects k_nwfwd's "big" (G = 4, ND = 10) instantiation; 0 selects the small one


def _rs(rng, L):
    return "".join("ACGT"[i] for i in rng.integers(0, 4, L))


def _mut(rng, s, k):
    s = list(s)
    for p in rng.choice(len(s), min(k, len(s)), replace=False):
        s[p] = "ACGT"[("ACGT".index(s[p]) + 1 + int(rng.integers(0, 3))) % 4]
    return "".join(s)


def _indel(rng, s, n=1):
    i = int(rng.integers(5, len(s) - 5))
    if rng.random() < 0.5:
        return s[:i] + s[i + n:] + _rs(rng, n)
    return s[:i] + _rs(rng, n) + s[i:-n]


def _qmat(seqs, rng, lo=20, hi=38, fixed=None):
    L = max(len(s) for s in seqs)
    q = np.full((len(seqs), L), np.nan)
    for i, s in enumerate(seqs):
        q[i, :len(s)] = fixed if fixed is not None else rng.integers(lo, hi + 1, len(s)).astype(np.float64)
    return q


def _case(label, seqs, quals, err, opts, kernels, promises, rng, reads=None):
    reads = np.asarray(reads if reads is not None else rng.integers(1, 40, len(seqs)), dtype=np.int32)
    reads[0] = max(int(reads.max()), 1)
    return dict(label=label, seqs=list(seqs), reads=reads, quals=quals, err=np.asarray(err, np.float64), opts=dict(opts), centre=0,
                jobs=np.arange(1, len(seqs), dtype=np.uint32), kernels=list(kernels), promises=set(promises))


def illumina_cases(scale):
    """250-nt Illumina-like uniques (tools/synth.illumina), equal lengths, tperr1, bands 8 / 16 / 32; identical raws (ns = 0) and
    unrelated ones (rho^ns underflows).  scale 'gpu': band 16 with more than 16 384 jobs (a round at 1e5 uniques) for k_nwrow<BOUND>."""
    from tests import cases
    from tools import synth
    out = []
    for band in (8, 16, 32):
        n = 20200 if (scale == "gpu" and band == 16) else (900 if scale == "gpu" else 150)
        seqs, ab, q, _ = synth.illumina(n, L=250, nvar=60, max_subs=40, indel_frac=0.0, seed=40 + band)
        rng = np.random.default_rng(band)
        extra = [seqs[0]] * 3 + [_rs(rng, 250) for _ in range(6)]
        qx = rng.integers(20, 39, (len(extra), 250)).astype(np.float64)
        qx[3:] = 40.0                           # the table's last column: rho ~ 1e-4, so rho^ns underflows for the unrelated raws
        q = np.vstack([q, qx])
        seqs = list(seqs) + extra
        kernels = [(0, 0), (1, 0), (2, 0), (2, BIG_HINT), (3, 0)]
        promises = {"keep", "drop", "either", "mixed", "ns0", "underflow"}
        if len(seqs) - 1 > LANE_MAX:
            promises.add("over16k")
        c = _case("illumina 250 nt band %d, %d jobs" % (band, len(seqs) - 1), seqs, q, cases.tperr1(), dict(band_size=band), kernels,
                  promises, rng, reads=np.concatenate([ab, np.ones(len(extra), np.int32)]))
        if len(seqs) - 1 > LANE_MAX:
            c["lane_jobs"] = LANE_MAX          # k_nwlane gets the first 16 384 jobs: the longest list it takes
        out.append(c)
    return out


# k_nwfwd's slot classes: fwd_slots = 2 band + (maxlen - minlen) + 3 at band 16 -> <= 40, <= 48, <= 64, <= 128, <= 256
SPREADS = {40: 4, 48: 10, 64: 26, 128: 90, 256: 200}


def ragged_cases(scale):
    """Raws of a 120-nt centre with substitutions and indels, cut / extended to lengths that spread by just enough to land the upload in
    each of k_nwfwd's slot classes; the <= 40 class with both instantiations, and through k_nwrow<BOUND> / k_nwlane, which hand the
    raws not as long as the centre back; the <= 48 class through k_gapless_loop (raws longer than the centre: their tail is self
    transitions)."""
    from tests import cases
    out = []
    n = 260 if scale == "gpu" else 70
    for cls, spread in SPREADS.items():
        rng = np.random.default_rng(1000 + cls)
        c = _rs(rng, 120 + spread)
        lo = 120 - spread // 2
        seqs = [c[:120]]
        for k in range(n):
            s = _mut(rng, c, int(rng.integers(0, 30)))
            if k % 3 == 1:
                s = _indel(rng, s, int(rng.integers(1, 4)))
            L = 120 if k % 4 == 0 else int(rng.integers(lo, lo + spread + 1))
            seqs.append(s[:L] if L <= len(s) else s + _rs(rng, L - len(s)))
        seqs[1] = c[:lo]; seqs[2] = c[:lo + spread] if lo + spread <= len(c) else c + _rs(rng, lo + spread - len(c))
        seqs[3] = c[:120]
        kernels = [(2, 0)]
        if cls == 40:
            kernels += [(2, BIG_HINT), (0, 0), (1, 0)]
        if cls == 48:
            kernels.append((3, 0))
        out.append(_case("ragged lengths, k_nwfwd slot class <= %d" % cls, seqs, _qmat(seqs, rng), cases.tperr1(), dict(band_size=16),
                         kernels, {"keep", "drop", "mixed", "ns0", "back"} if cls == 40 else {"keep", "drop", "mixed", "ns0"}, rng))
    return out


def pacbio_case(scale):
    """1500-nt PacBio-like uniques (tools/synth.pacbio), 94 quality columns (quality 93 is the table's last column), band 32."""
    from tests import cases
    from tools import synth
    n = 120 if scale == "gpu" else 16
    seqs, ab, q = synth.pacbio(n, L=1500, nvar=4, seed=9)
    err = synth.extend_err(cases.tperr1(), 94)
    rng = np.random.default_rng(94)
    return _case("pacbio 1500 nt, 94 columns, band 32", seqs, q, err, dict(band_size=32), [(2, 0), (3, 0)],
                 {"keep", "drop", "mixed", "ns0"}, rng, reads=ab)


def _mutants(rng, L, n, maxsub=40):
    c = _rs(rng, L)
    seqs = [c] + [c] * 2 + [_mut(rng, c, int(k)) for k in rng.integers(1, maxsub, n)] + [_rs(rng, L) for _ in range(4)]
    return seqs


def err_cases(scale):
    """err edges on 150-nt mutants of one centre: all ones (S = rho = 1), a zero self transition at a (base, quality) some raws use
    (S = 0, rho = inf; a 0 / 0 ratio beside it), self transitions low enough that S_r is subnormal or flushed to 0 while rho^ns
    brings the bound back above 1e-280, and use_quals = False (column 0 only)."""
    from tests import cases
    n = 400 if scale == "gpu" else 120
    out = []
    t = cases.tperr1()
    rng = np.random.default_rng(7)
    seqs = _mutants(rng, 150, n)
    out.append(_case("err all ones", seqs, _qmat(seqs, rng), np.ones_like(t), dict(band_size=16), [(0, 0), (1, 0), (2, 0), (3, 0)],
                     {"keep", "drop", "mixed", "ns0"}, rng))
    rng = np.random.default_rng(8)
    seqs = _mutants(rng, 150, n)
    q = _qmat(seqs, rng, fixed=30.0)
    for i in range(1, len(seqs), 3):
        q[i, int(rng.integers(0, 150))] = 17.0
    z = t.copy()
    z[5 * 0, 17] = 0.0                           # A -> A at quality 17: S = 0 for every raw with an A there
    z[4 * 1 + 0, 17] = 0.0                       # C -> A at quality 17: the ratio 0 / 0, which fmax ignores
    out.append(_case("zero self transition", seqs, q, z, dict(band_size=16), [(0, 0), (1, 0), (2, 0), (3, 0)],
                     {"keep", "drop", "mixed", "nan"}, rng))
    rng = np.random.default_rng(9)
    seqs = _mutants(rng, 150, n)
    q = _qmat(seqs, rng, lo=28, hi=32)
    lo = t.copy()
    for qq in range(lo.shape[1]):
        for b in range(4):
            lo[5 * b, qq] = 0.0079 + 0.0002 * (qq % 5) + 0.0001 * b
            for a in range(4):
                if a != b:
                    lo[4 * a + b, qq] = 0.3 - 0.01 * a
    out.append(_case("subnormal S_r", seqs, q, lo, dict(band_size=16), [(0, 0), (1, 0), (2, 0), (3, 0)],
                     {"keep", "drop", "mixed", "subnormal", "underflow"}, rng))
    rng = np.random.default_rng(10)
    seqs = _mutants(rng, 150, n)
    out.append(_case("use_quals = FALSE", seqs, _qmat(seqs, rng), t, dict(band_size=16, use_quals=False), [(0, 0), (1, 0), (2, 0), (3, 0)],
                     {"keep", "drop", "either", "mixed", "ns0"}, rng))
    return out


def all_cases(scale="emu"):
    return illumina_cases(scale) + ragged_cases(scale) + [pacbio_case(scale)] + err_cases(scale)


# ------------------------------------------------------------------------------------------------------------------------------
def _qrows(case):
    return BR.round_quals(case["quals"])


def reference(case, mode):
    """Per job: nsubs, lambda and (for 'nw') the alignment strings of the oracle (oracle.port.pair, pinned to the reference on the
    pair corpus), or of nwalign_gapless for 'gl' (k_gapless_loop's jobs)."""
    from oracle import port
    seqs, err, o = case["seqs"], case["err"], case["opts"]
    uq = o.get("use_quals", True)
    qi = _qrows(case)
    c = case["centre"]
    ns = np.zeros(len(case["jobs"]), np.int64); lam = np.zeros(len(case["jobs"])); gapfree = np.zeros(len(case["jobs"]), bool)
    popts = dict(band_size=o.get("band_size", 16))
    for k, r in enumerate(case["jobs"]):
        r = int(r)
        if mode == "gl":
            ns[k], lam[k] = BR.gapless(seqs[c], seqs[r], qi[r], err, uq)
            gapfree[k] = True
            continue
        p = port.pair(seqs[c], qi[c, :len(seqs[c])].astype(np.uint8), seqs[r], qi[r, :len(seqs[r])].astype(np.uint8) if uq else None, err,
                      use_kmers=False, **popts)
        ns[k], lam[k] = p["nsubs"], p["lam"]
        gapfree[k] = "-" not in p["al0"] and "-" not in p["al1"]
    return ns, lam, gapfree


def prepare(case, mode):
    """-> dict(ns, lam, gapfree, E (per job), E_all (per raw), dec (KEEP / DROP / EITHER per job), B (exact bounds), S_fp) for the
    kernels of `mode` ('nw' or 'gl')."""
    key = "_prep_" + mode
    if key in case:
        return case[key]
    seqs, err, o = case["seqs"], case["err"], case["opts"]
    uq = o.get("use_quals", True)
    qi = _qrows(case)
    T = int(np.sum(case["reads"], dtype=np.int64))
    ns, lam, gapfree = reference(case, mode)
    S_fp, _ = BR.raw_factors(seqs, case["quals"], err, uq)
    E = np.zeros(len(case["jobs"])); dec = np.zeros(len(case["jobs"]), np.int64); Bs = []
    fac = {}
    for k, r in enumerate(case["jobs"]):
        r = int(r)
        if r not in fac:
            fac[r] = BR.exact_factors(seqs[r], qi[r], err, uq)
        B = BR.exact_bound(fac[r][0], fac[r][1], int(ns[k]), T)
        Bs.append(B)
        lt = lam[k] * float(T)
        if k % 2 == 0:                                   # the "keep" side: the reference stores the pair
            e = -999.0 if k % 4 == 0 else float(np.nextafter(lt, -math.inf))
        else:                                            # the "drop" side: at or beyond the bound's threshold
            e = math.inf
            if isinstance(B, Fraction) and k % 4 == 1:
                x = B * BR.MARGIN * (1 + Fraction(1, 10 ** 11))
                e = float(x) if x < Fraction(1.7e308) else math.inf
                if e != math.inf and Fraction(e) < x:
                    e = float(np.nextafter(e, math.inf))
        if k % 16 == 7:                                  # "either": exactly fl(lam T), not stored, the bound keeps it
            e = lt
        elif k % 16 == 15 and isinstance(B, Fraction):   # "either": just inside the bound's margin
            x = B * BR.MARGIN * (1 - Fraction(1, 10 ** 11))
            e = float(x) if x < Fraction(1.7e308) else math.inf
        E[k] = e
        dec[k] = BR.decision(int(ns[k]), float(lam[k]), e, T, B, float(S_fp[r]))
    E_all = np.full(len(seqs), -999.0)
    E_all[case["jobs"]] = E
    case[key] = dict(ns=ns, lam=lam, gapfree=gapfree, E=E, E_all=E_all, dec=dec, B=Bs, S_fp=S_fp, T=T)
    return case[key]


def edge_counts(case, mode):
    """What the case reaches: counts of keep / drop / either jobs, underflow and undefined bounds, ns = 0, subnormal S_r, mixed warps
    (32 consecutive jobs with both a keep and a drop), and whether the job list is longer than k_nwlane takes."""
    p = prepare(case, mode)
    dec = p["dec"]
    under = sum(1 for B in p["B"] if isinstance(B, Fraction) and B < Fraction(BR.UNDERFLOW))
    nan = sum(1 for B in p["B"] if B is None)
    S = p["S_fp"][case["jobs"]]
    sub = int(np.sum((S > 0) & (S < BR.DBL_MIN)))
    w = [(dec[i:i + 32] == BR.KEEP).any() and (dec[i:i + 32] == BR.DROP).any() for i in range(0, len(dec), 32)]
    lens = np.array([len(case["seqs"][int(r)]) for r in case["jobs"]])
    return dict(keep=int((dec == BR.KEEP).sum()), drop=int((dec == BR.DROP).sum()), either=int((dec == BR.EITHER).sum()),
                underflow=under, nan=nan, ns0=int((p["ns"] == 0).sum()), subnormal=sub, mixed=int(sum(w)),
                over16k=int(len(dec) > LANE_MAX), back=int((lens != len(case["seqs"][case["centre"]])).sum()))


def check_raw_bounds(res, case):
    """k_raw_bounds' S and rho equal raw_factors bit for bit, for every rank of worlds 1, 2 and 3."""
    uq = case["opts"].get("use_quals", True)
    S, rho = BR.raw_factors(case["seqs"], case["quals"], case["err"], uq)
    for rank, world in ((0, 1), (1, 2), (2, 3)):
        gs, gr = res.test_raw_bounds(case["err"], use_quals=uq, rank=rank, world=world)
        mine = np.arange(len(S)) % world == rank
        assert np.isnan(gs[~mine]).all() and np.isnan(gr[~mine]).all(), case["label"]
        for want, got, name in ((S, gs, "S"), (rho, gr, "rho")):
            bad = np.flatnonzero(mine & ~((want == got) | (np.isnan(want) & np.isnan(got))))
            assert len(bad) == 0, "%s: %s differs at raws %s: got %r want %r" % (case["label"], name, bad[:5], got[bad[:5]].tolist(), want[bad[:5]].tolist())


def check_kernel(res, case, which, hint):
    """One launch of kernel `which` over the case's jobs against the reference; -> per-decision outcome counts."""
    mode = "gl" if which == 3 else "nw"
    p = prepare(case, mode)
    jobs = case["jobs"]
    sel = slice(0, case.get("lane_jobs", len(jobs)) if which == 1 else len(jobs))
    jobs = jobs[sel]
    E_all = np.full(len(case["seqs"]), -999.0)
    E_all[jobs] = p["E"][sel]
    got = res.test_bound(which, case["centre"], 1, jobs, E_all, case["err"], njobs_hint=hint, **case["opts"])
    tag = "%s: which %d hint %d" % (case["label"], which, hint)
    out, nsg, lamg = got["outcome"], got["nsubs"], got["lam"]
    ns, lam, dec, gapfree, E = p["ns"][sel], p["lam"][sel], p["dec"][sel], p["gapfree"][sel], p["E"][sel]
    T = p["T"]
    lc = len(case["seqs"][case["centre"]])
    lens = np.array([len(case["seqs"][int(r)]) for r in jobs])
    back = out == 3
    want_back = (lens != lc) if which in (0, 1) else np.zeros(len(jobs), bool)
    bad = np.flatnonzero(back != want_back)
    assert len(bad) == 0, "%s: handed back differs at jobs %s" % (tag, bad[:10])
    on = ~back
    bad = np.flatnonzero(on & (nsg != ns))
    assert len(bad) == 0, "%s: nsubs differs at jobs %s: got %s want %s" % (tag, bad[:10], nsg[bad[:10]], ns[bad[:10]])
    kept = on & (out != 0)
    bad = np.flatnonzero(on & (dec == BR.KEEP) & ~kept)
    assert len(bad) == 0, "%s: must-keep jobs dropped: %s (ns %s, E %s, lam %s)" % (tag, bad[:10], ns[bad[:10]], E[bad[:10]].tolist(),
                                                                                  lam[bad[:10]].tolist())
    bad = np.flatnonzero(on & (dec == BR.DROP) & kept)
    assert len(bad) == 0, "%s: must-drop jobs survived: %s (ns %s, E %s)" % (tag, bad[:10], ns[bad[:10]], E[bad[:10]].tolist())
    if which == 0:
        assert set(np.unique(out[kept]).tolist()) <= {1, 2}, tag
        bad = np.flatnonzero((out == 2) & ~gapfree)
        assert len(bad) == 0, "%s: gapless-listed jobs whose oracle alignment has gaps: %s" % (tag, bad[:10])
    elif which == 2:
        assert set(np.unique(out[kept]).tolist()) <= {1}, tag
    else:
        assert set(np.unique(out[kept]).tolist()) <= {4, 5}, tag
        stored = out == 4
        want_stored = on & (lam * float(T) > E)
        bad = np.flatnonzero(stored != want_stored)
        assert len(bad) == 0, "%s: stored differs from the store rule at jobs %s" % (tag, bad[:10])
        bad = np.flatnonzero(stored & (lamg != lam))
        assert len(bad) == 0, "%s: stored lambda differs at jobs %s: got %r want %r" % (tag, bad[:10], lamg[bad[:10]].tolist(), lam[bad[:10]].tolist())
        assert np.isnan(lamg[~stored]).all(), tag
        cr = float(case["reads"][case["centre"]])
        want_e = E_all.copy()
        upd = jobs[stored]
        ec = lam[stored] * cr
        want_e[upd] = np.where(ec > E[stored], ec, E[stored])
        bad = np.flatnonzero(got["e_after"] != want_e)
        assert len(bad) == 0, "%s: E_minmax after the launch differs at raws %s" % (tag, bad[:10])
    if which != 1 and which != 3:
        assert np.array_equal(got["e_after"], E_all), tag
    c = got["counters"]
    assert c["back"] == int(back.sum()) and c["surv"] == int((out == 1).sum()) and c["gapless"] == int((out == 2).sum()), (tag, c)
    assert c["stored"] == int((out == 4).sum()), (tag, c)
    return dict(keep=int((on & (dec == BR.KEEP)).sum()), drop=int((on & (dec == BR.DROP)).sum()), either=int((on & (dec == BR.EITHER)).sum()),
                kept=int(kept.sum()), dropped=int((on & ~kept).sum()), back=int(back.sum()))


def run_case(make_resident, case, log=None):
    """Every kernel launch of `case` and the raw factors; -> {(which, hint): counts}."""
    res = make_resident(case["seqs"], case["reads"], None, case["quals"])
    out = {}
    try:
        check_raw_bounds(res, case)
        for which, hint in case["kernels"]:
            out[(which, hint)] = c = check_kernel(res, case, which, hint)
            if log:
                log("%s | kernel %d hint %s: %s" % (case["label"], which, "big" if hint else "small", c))
    finally:
        res.close()
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# one record per NW comparison of b_compare (oracle/port.cpp, PORT_TRACE): round, raw, nsubs, stored, lambda, E_minmax before the
# comparison, total reads
TRACE_DTYPE = np.dtype([("i", "u4"), ("index", "u4"), ("nsubs", "u4"), ("stored", "u4"), ("lam", "f8"), ("emm", "f8"), ("breads", "f8")])


def trace(name):
    """The CPU oracle's NW comparisons of e2e case `name` (tests/cases.py), with E_minmax as each one met it, and the centre of every
    cluster (round i compares the centre of cluster i).  The centres are the raws whose sequences the oracle's clustering lists, in
    cluster order (final_consensus is off in the e2e cases, so a cluster's sequence is its centre's).  -> (records, centres)"""
    script = textwrap.dedent('''
        import sys
        import numpy as np
        sys.path.insert(0, %r)
        from oracle import port
        from tests import cases
        seqs, ab, pri, err, q, opts = cases.build_case(%r)
        assert not opts.get("final_consensus")
        out = port.dada_uniques(seqs, ab, pri, err, q, **opts)
        idx = {s: i for i, s in enumerate(seqs)}
        np.save(sys.argv[1], np.array([idx[s] for s in out["clustering"]["sequence"]], np.int64))
    ''') % (ROOT, name)
    with tempfile.TemporaryDirectory() as d:
        path, cpath = os.path.join(d, "trace.bin"), os.path.join(d, "centres.npy")
        subprocess.check_call([sys.executable, "-c", script, cpath], env=dict(os.environ, PORT_TRACE=path), cwd=ROOT)
        rec = np.fromfile(path, dtype=TRACE_DTYPE)
        centres = np.load(cpath)
    assert len(rec) and rec["i"].max() < len(centres), name
    return rec, centres


def replay(make_resident, name, log=None):
    """Every NW comparison the CPU oracle makes in rounds i > 0 of e2e case `name`, one round at a time (its centre, its raws and their
    E_minmax at that moment), through k_nwrow<BOUND> (raws as long as the centre), k_nwlane (rounds it takes) and k_nwfwd's bound
    pass.  No comparison the oracle stores is dropped, nsubs is the oracle's, and the dropped set is bound_ref's must-drop set apart
    from the "either" jobs.  -> {which: (dropped, replayed)}."""
    from tests import cases
    seqs, ab, pri, err, q, opts = cases.build_case(name)
    rec, centres = trace(name)
    assert rec["index"].max() < len(seqs) and (rec["breads"] == float(np.sum(ab, dtype=np.int64))).all(), name
    rec = rec[rec["i"] > 0]
    uq = opts.get("use_quals", True)
    qi = BR.round_quals(q)
    S_fp, _ = BR.raw_factors(seqs, q, err, uq)
    fac = {}
    res = make_resident(seqs, ab, pri, q)
    tot = {0: [0, 0], 1: [0, 0], 2: [0, 0]}
    try:
        for i in np.unique(rec["i"]):
            rr = rec[rec["i"] == i]
            c = int(centres[i])
            jobs = rr["index"].astype(np.uint32)
            E_all = np.full(len(seqs), -999.0)
            E_all[jobs] = rr["emm"]
            T = int(rr["breads"][0])
            dec = np.zeros(len(rr), np.int64)
            for k, r in enumerate(jobs):
                r = int(r)
                if r not in fac:
                    fac[r] = BR.exact_factors(seqs[r], qi[r], err, uq)
                B = BR.exact_bound(fac[r][0], fac[r][1], int(rr["nsubs"][k]), T)
                dec[k] = BR.decision(int(rr["nsubs"][k]), float(rr["lam"][k]), float(rr["emm"][k]), T, B, float(S_fp[r]))
            assert not ((dec == BR.DROP) & (rr["stored"] == 1)).any()
            for which in (0, 1, 2):
                if which == 1 and len(jobs) > LANE_MAX:
                    continue
                got = res.test_bound(which, c, int(i), jobs, E_all, err, **opts)
                out = got["outcome"]
                on = out != 3
                tag = "%s round %d kernel %d" % (name, i, which)
                assert (on | (which == 0)).all(), tag
                assert np.array_equal(got["nsubs"][on], rr["nsubs"][on].astype(np.int32)), tag
                dropped = on & (out == 0)
                assert not (dropped & (rr["stored"] == 1)).any(), tag + ": a stored comparison was dropped"
                assert not (dropped & (dec == BR.KEEP)).any(), tag + ": a must-keep comparison was dropped"
                assert not (on & ~dropped & (dec == BR.DROP)).any(), tag + ": a must-drop comparison survived"
                if which == 1:
                    st = out == 4
                    assert np.array_equal(st, on & (rr["lam"] * float(T) > rr["emm"])), tag
                    assert np.array_equal(got["lam"][st], rr["lam"][st]), tag
                tot[which][0] += int(dropped.sum()); tot[which][1] += int(on.sum())
    finally:
        res.close()
    if log:
        for w, (d, n) in tot.items():
            log("replay %s kernel %d: %d of %d comparisons dropped (%.3f)" % (name, w, d, n, d / max(n, 1)))
    return tot
