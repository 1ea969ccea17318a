"""Seeded inputs at the edges of the k-mer screen, and the check that runs them through the stage hook dada2b_test_screen
(include/dada2b_test.h) against the plain restatement tests/screen_ref.py.

Every case is generated here at test time.  A case is one uploaded set of raws and a list of screen calls on it:
    dict(label, seqs, reads, calls=[dict(centre, kdist_cutoff, greedy, lock, centre_reads, opts)], worlds, max_sms, path)
Each call runs on both paths (0: the product's selection, k_prescreen -> k_kord -> k_classify for overflowed lists; 1: k_classify
alone), for every rank of every world listed, at every SM cap listed; every result must equal the reference exactly:
kind per raw, the min-sum k_prescreen handed on for each candidate, and the round counters.
"""
import numpy as np

from tests import screen_ref

PS_TILE = 128                  # dd_prescreen.cu: raws per TMA tile
PS_STAGES = 4                  # stages of the ring
PS_CTAS_PER_SM = 3             # launch_prescreen: grid = min(ntiles, 3 * SMs)


def _rs(rng, L):
    return "".join("ACGT"[i] for i in rng.integers(0, 4, L))


def _mut(rng, s, k):
    s = list(s)
    for p in rng.choice(len(s), min(k, len(s)), replace=False):
        s[p] = "ACGT"[("ACGT".index(s[p]) + 1 + int(rng.integers(0, 3))) % 4]
    return "".join(s)


def _indel(rng, s):
    i = int(rng.integers(1, len(s) - 1))
    return s[:i] + s[i + 1:] + "ACGT"[int(rng.integers(0, 4))] if rng.random() < 0.5 else s[:i] + "ACGT"[int(rng.integers(0, 4))] + s[i:-1]


def _calls(centres, cutoffs, greedy=(True,), lock=None, opts=({},), reads=None, centre_reads=None):
    out = []
    for c in centres:
        for kd in cutoffs:
            for g in greedy:
                for o in opts:
                    out.append(dict(centre=c, kdist_cutoff=float(kd), greedy=g, lock=lock, centre_reads=centre_reads, opts=dict(o)))
    return out


def boundary_case():
    """Mutants of one 100-nt centre (0 .. 30 substitutions, some indels): cutoffs exactly at kdist(ms) for min-sums that occur (equal
    is not shrouded: the test is >), their neighbouring doubles, 0.42, 0, values just below 1 and 1 itself (k_classify);
    abundances above and below the centre's, 30 % of the raws locked, greedy on and off."""
    rng = np.random.default_rng(101)
    c = _rs(rng, 100)
    seqs = [c] + [_mut(rng, c, int(k)) for k in rng.integers(0, 31, 220)] + [_indel(rng, _mut(rng, c, int(k))) for k in rng.integers(0, 12, 79)]
    reads = rng.integers(1, 200, len(seqs)).astype(np.int32)
    reads[0] = 100
    lock = (rng.random(len(seqs)) < 0.3).astype(np.uint8)
    ref = screen_ref.screen(seqs, 0, 0.42)
    occurring = np.unique(ref["minsum"])
    pick = occurring[np.linspace(0, len(occurring) - 1, 6).astype(int)]
    cut = []
    for ms in pick:
        kd = float(screen_ref.kdist_of(ms, 100, 100))
        cut += [kd, np.nextafter(kd, -1.0), np.nextafter(kd, 2.0)]
    cut += [0.42, 0.0, np.nextafter(1.0, 0.0), 1.0 - 1e-9, 1.0]
    calls = _calls([0], cut, greedy=(True, False), lock=lock)
    calls += _calls([0], [0.42], greedy=(True,), lock=lock, centre_reads=50)
    calls += _calls([0], [0.42, 0.2], opts=({"SSE": 0}, {"SSE": 1}, {"gapless": False}, {"band_size": 0}, {"use_kmers": False}))
    return dict(label="kdist cutoff on the boundary, greedy", seqs=seqs, reads=reads, calls=calls, worlds=(1,), max_sms=(0, 1))


def bound_case():
    """Raws whose presence bound is inconclusive while the exact min-sum shrouds them (the centre's 5-mers repeated in the raw), and
    raws the exact min-sum keeps, interleaved over consecutive tiles so that the hand-over of a pending raw (resolve()) runs in every
    iteration; the centre holds repeated 5-mers itself, so min(count_raw, count_centre) > 1 matters.  Every shard of worlds 1, 2, 3, 8."""
    rng = np.random.default_rng(202)
    a, b, x = _rs(rng, 40), _rs(rng, 40), _rs(rng, 40)
    c = a + a + b                                              # 120 nt, the 5-mers of a twice
    kinds = [lambda: a + a + a, lambda: b + b + b, lambda: a + b + b, lambda: a + b + x, lambda: c, lambda: x + x + a,
             lambda: (a + b)[:60] * 2, lambda: a + a + a[:20] + b[:20]]
    seqs = [c]
    for i in range(1100):
        s = kinds[i % len(kinds)]()
        seqs.append(_mut(rng, s, int(rng.integers(0, 6))))
    reads = rng.integers(1, 50, len(seqs)).astype(np.int32)
    calls = _calls([0], [0.42, 0.3, 0.5, 0.6])
    return dict(label="presence bound and exact min-sum disagree", seqs=seqs, reads=reads, calls=calls, worlds=(1, 2, 3, 8), max_sms=(0, 1))


def _with_repeats(rng, d, flank=20):
    """A raw with exactly d distinct repeated 5-mers, each twice, and no other repeated 5-mer."""
    while True:
        seg = _rs(rng, d + 4) if d else ""
        s = _rs(rng, flank) + seg + _rs(rng, flank) + seg + _rs(rng, flank)
        km = screen_ref.kmers(s)
        cnt = np.bincount(km, minlength=screen_ref.NK)
        if (cnt >= 2).sum() == d and cnt.max() <= 2:
            return s, seg


def repeat_case():
    """The repeated-5-mer list: raw counts of AAAAA 2 / 63 / 64 / 65 (65 overflows) against centres holding it 1 / 2 / 260 times
    (the shared count table caps at 255), and raws with 0, 1, 7, 8, 9, 15, 16, 47, 48, 49 distinct repeated 5-mers (the 8-entry blocks
    of the list; 49 overflows) against a centre that holds those 5-mers once or twice."""
    rng = np.random.default_rng(303)
    f1, f2 = _rs(rng, 40), _rs(rng, 40)
    f1, f2 = "C" + f1[1:-1] + "C", "G" + f2[1:-1] + "T"        # the runs of A stay exactly as long as written
    seqs, cen = [], []
    for run in (5, 6, 264):
        cen.append(len(seqs)); seqs.append(f1 + "A" * run + f2)
    for cnt in (2, 63, 64, 65):
        for k in range(6):
            seqs.append(_mut(rng, f1, k % 3) + "A" * (cnt + 4) + _mut(rng, f2, k // 3))
    segs = []
    for d in (0, 1, 7, 8, 9, 15, 16, 47, 48, 49):
        s, seg = _with_repeats(rng, d)
        segs.append(seg)
        seqs.append(s)
        for k in range(3):
            seqs.append(_mut(rng, s, k))
    cen.append(len(seqs))
    seqs.append("".join(g + "T" for g in segs) + "".join(g + "C" for g in segs[::2]))
    reads = np.full(len(seqs), 5, np.int32)
    calls = _calls(cen, [0.42, 0.1, 0.8])
    return dict(label="repeat-list boundaries", seqs=seqs, reads=reads, calls=calls, worlds=(1,), max_sms=(0,))


def length_case():
    """Lengths 6, 19 / 20 / 21 (k_kord's 16-base words: nko 15, 16, 17), 250, 251 and 1500 in one set, raws longer and shorter than
    the centre, SSE 0 / 1 / 2 (kord_dist is -1 for unequal lengths only when SSE is 0)."""
    rng = np.random.default_rng(404)
    seqs, cen = [], []
    for L in (6, 19, 20, 21, 250, 251, 1500):
        c = _rs(rng, L + 10)
        cen.append(len(seqs)); seqs.append(c[:L])
        for dl in (-3, -1, 0, 0, 1, 3, 10):
            l2 = L + dl
            if l2 <= 5:
                continue
            base = c[:l2] if l2 <= len(c) else c + _rs(rng, l2 - len(c))
            for k in (0, 1, 3):
                seqs.append(_mut(rng, base, k))
    reads = np.full(len(seqs), 5, np.int32)
    calls = _calls(cen, [0.42, 0.05], opts=({"SSE": 0}, {"SSE": 1}, {"SSE": 2}))
    return dict(label="lengths 6 .. 1500", seqs=seqs, reads=reads, calls=calls, worlds=(1,), max_sms=(0,))


MAXLEN = 9998                  # upload rejects 9999 and longer (Rmain.cpp); setup_params accepts it when the lengths spread by little


def long_case():
    """The longest raws a context takes: 9990 .. 9998 nt, and a homopolymer of 9998 nt whose list slack (14 bits of the meta word)
    is the largest possible: against a homopolymer centre its presence bound is 1 + 9993."""
    rng = np.random.default_rng(505)
    c = _rs(rng, MAXLEN)
    seqs = [c, "A" * MAXLEN]
    for L in (9990, 9994, 9997, 9998):
        for k in (0, 2, 40):
            seqs.append(_mut(rng, c[:L], k))
    seqs.append("A" * (MAXLEN - 1) + "C")
    seqs.append("A" * 9990)
    reads = np.full(len(seqs), 5, np.int32)
    calls = _calls([0, 1], [0.42, 0.001])
    return dict(label="longest raws", seqs=seqs, reads=reads, calls=calls, worlds=(1,), max_sms=(0,))


def size_cases():
    """nraw 1, 127, 128, 129 (a partial / full / one-past-full tile)."""
    out = []
    for n in (1, 127, 128, 129):
        rng = np.random.default_rng(600 + n)
        c = _rs(rng, 150)
        seqs = [c] + [_mut(rng, c, int(k)) for k in rng.integers(0, 40, n - 1)]
        out.append(dict(label="nraw %d" % n, seqs=seqs, reads=np.full(n, 3, np.int32), calls=_calls([0], [0.42, 0.15]), worlds=(1, 2),
                        max_sms=(0,)))
    return out


def ring_case():
    """4613 raws of 250 nt with max_sms = 1: 37 tiles over 3 CTAs, about 12 tiles per CTA, so the 4-stage ring wraps 3 times."""
    rng = np.random.default_rng(707)
    c = _rs(rng, 250)
    seqs = [c] + [_mut(rng, c, int(k)) for k in rng.integers(0, 50, 4612)]
    reads = rng.integers(1, 30, len(seqs)).astype(np.int32)
    return dict(label="ring wraps at max_sms=1", seqs=seqs, reads=reads, calls=_calls([0], [0.42, 0.25]), worlds=(1,), max_sms=(1,),
                wrap=True)


def full_grid_case(sms):
    """More than 4 * 3 * SMs * 128 raws of 40 to 60 nt at the device's full SM count: every CTA of the grid reuses every stage."""
    rng = np.random.default_rng(808)
    n = max(250000, PS_STAGES * PS_CTAS_PER_SM * sms * PS_TILE + 20 * PS_TILE)
    c = _rs(rng, 60)
    lens = rng.integers(40, 61, n - 1)
    subs = rng.integers(0, 20, n - 1)
    root = np.frombuffer(c.encode(), np.uint8)
    alt = np.frombuffer(b"ACGT", np.uint8)
    seqs = [c]
    for L, k in zip(lens, subs):
        s = root[:L].copy()
        p = rng.choice(L, int(k), replace=False)
        s[p] = alt[(np.searchsorted(alt, s[p]) + rng.integers(1, 4, len(p))) % 4]
        seqs.append(s.tobytes().decode())
    reads = rng.integers(1, 1000, n).astype(np.int32)
    return dict(label="full grid, ring wraps", seqs=seqs, reads=reads, calls=_calls([0], [0.42]), worlds=(1,), max_sms=(0,), wrap=True)


def small_cases():
    return [boundary_case(), bound_case(), repeat_case(), length_case(), long_case()] + size_cases() + [ring_case()]


def prescreen_grid(nown, sms):
    ntiles = (nown + PS_TILE - 1) // PS_TILE
    return ntiles, max(1, min(ntiles, PS_CTAS_PER_SM * sms))


def check_call(res, seqs, reads, call, path, rank, world, max_sms, label=""):
    """One hook call against the reference; -> the hook's result."""
    o = dict(call["opts"])
    greedy = call["greedy"]
    got = res.test_screen(call["centre"], kdist_cutoff=call["kdist_cutoff"], centre_reads=call["centre_reads"] if call["centre_reads"] is not None
                          else int(reads[call["centre"]]), lock=call["lock"], rank=rank, world=world, max_sms=max_sms, path=path,
                          greedy=greedy, **o)
    want = screen_ref.screen(seqs, call["centre"], call["kdist_cutoff"], reads=reads, centre_reads=call["centre_reads"],
                             lock=call["lock"], greedy=greedy, rank=rank, world=world, **o)
    tag = "%s: centre %d cutoff %r greedy %d opts %s path %d shard %d/%d max_sms %d" % (label, call["centre"], call["kdist_cutoff"], greedy, o,
                                                                                       path, rank, world, max_sms)
    bad = np.flatnonzero(got["kind"] != want["kind"])
    assert len(bad) == 0, "%s: kind differs at raws %s: got %s want %s (minsum %s, kdist %s)" % (
        tag, bad[:10], got["kind"][bad[:10]], want["kind"][bad[:10]], want["minsum"][bad[:10]], want["kdist"][bad[:10]])
    c = got["counters"]
    assert c["align"] == want["align"] and c["shroud"] == want["shroud"], (tag, c, want["align"], want["shroud"])
    assert c["gapless"] == int((want["kind"] == 1).sum()) and c["nw"] == int((want["kind"] == 2).sum()), (tag, c)
    ms = got["minsum"]
    streaming = path == 0 and o.get("use_kmers", True) and call["kdist_cutoff"] < 1.0
    if not streaming:
        assert (ms == -1).all(), tag
        return got
    act = want["owned"] & ~want["skipped"]
    cand = act & (want["kind"] > 0)
    lb = screen_ref.kdist_of(want["bound"], len(seqs[call["centre"]]), np.array([len(s) for s in seqs]))
    ovf_cand = act & want["overflow"] & ~(lb > call["kdist_cutoff"])           # overflowed lists go on whenever the bound cannot shroud
    expect = np.where(ovf_cand, 0xFFFF, np.where(cand & ~want["overflow"], want["minsum"], -1))
    bad = np.flatnonzero(ms != expect)
    assert len(bad) == 0, "%s: minsum differs at raws %s: got %s want %s" % (tag, bad[:10], ms[bad[:10]], expect[bad[:10]])
    return got


def run_case(make_resident, case, sms, paths=(0, 1)):
    """Every call of `case` on both paths, every shard of every world and every SM cap of the case; sms is the device's SM count
    (what max_sms = 0 means).  -> number of hook calls."""
    seqs, reads = case["seqs"], case["reads"]
    L = max(len(s) for s in seqs)
    q = np.full((len(seqs), L), np.nan)
    for i, s in enumerate(seqs):
        q[i, :len(s)] = 30.0
    res = make_resident(seqs, reads, None, q)
    calls = 0
    try:
        for max_sms in case["max_sms"]:
            eff = sms if max_sms == 0 else min(sms, max_sms)
            if case.get("wrap"):
                ntiles, grid = prescreen_grid(len(seqs), eff)
                assert ntiles > PS_STAGES * grid, (case["label"], ntiles, grid)      # each CTA streams more tiles than the ring has stages
            for call in case["calls"]:
                for path in paths:
                    union = None
                    for world in case["worlds"]:
                        kinds = np.full(len(seqs), -2, np.int32)
                        for rank in range(world):
                            got = check_call(res, seqs, reads, call, path, rank, world, max_sms, case["label"])
                            mine = got["kind"] >= 0
                            assert (np.flatnonzero(mine) % world == rank).all()
                            kinds[mine] = got["kind"][mine]
                            calls += 1
                        assert (kinds >= 0).all()
                        if union is None:
                            union = kinds
                        assert np.array_equal(kinds, union), (case["label"], world)    # the shards' union is the world = 1 result
    finally:
        res.close()
    return calls
