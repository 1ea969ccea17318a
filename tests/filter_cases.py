"""Seeded read sets and option sets at the edges of the read filter (R/filter.R stages 1-12), shared by the golden
generator (tools/make_golden_filter.py -> tests/golden/filter.npz), the emulator tests and the H100 tests."""
import math
import os

import numpy as np

from tests import filter_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "filter.npz")
PHIX_FA = os.path.join(HERE, "golden", "phix_genome.fa")
INF = math.inf


def phix():
    with open(PHIX_FA) as f:
        return "".join(ln.strip() for ln in f if not ln.startswith(">"))


def _rand(rng, n):
    return "".join("ACGT"[i] for i in rng.integers(0, 4, n))


def _quals(rng, n, lo=20, hi=41, tail=0):
    q = rng.integers(lo, hi, n)
    if tail and n:
        q[n - tail:] = rng.integers(0, 12, min(tail, n))
    return [int(x) for x in q]


def _differs_from_tree(q):
    return R.matrix_ee(q) != R.tree_ee(q)


def single_pool(seed=11):
    """Reads (seq, quals) covering every stage's edge; the comments name the edge."""
    rng = np.random.default_rng(seed)
    ph = phix()
    prc = R.rc(ph)
    reads = []
    add = lambda s, q=None: reads.append((s, q if q is not None else _quals(rng, len(s))))
    for _ in range(24):                                            # ordinary reads with low-quality tails
        L = int(rng.integers(150, 260))
        add(_rand(rng, L), _quals(rng, L, tail=int(rng.integers(0, 30))))
    s = _rand(rng, 120)
    add(s, [2] + _quals(rng, 119))                                 # truncQ hit at base 0
    add(s, _quals(rng, 119) + [2])                                 # ... at the last base
    add(s, [0] * 120)                                              # q 0 everywhere
    add(s, [93] * 120)                                             # q 93 everywhere
    for k in (1, 2, 3):                                            # maxN at the count and count + 1, N and IUPAC codes
        t = list(_rand(rng, 100))
        for j, c in zip(rng.choice(100, k, replace=False), "NRY"):
            t[j] = c
        add("".join(t))
    add("ACGTNRYSWKMBDHV" * 8)                                     # every IUPAC letter
    for w in (15, 16, 17, 18, 19):                                 # 100, 107, 114, 121, 128 nt
        add(_rand(rng, w * 7 - 5))
    for w in (19, 20, 21):                                         # raw width start - 1, start, start + 1 at trimLeft=19 ("trims")
        add(_rand(rng, w))
    # phiX: fragments from both strands, across the circular junction, two hits 15..18 apart, one hit, an N in a window
    for st in (100, 2000, 5000):
        add(ph[st:st + 150])
        add(prc[st:st + 150])
    add(ph[-60:] + ph[:90])
    bg = _rand(rng, 200)
    for gap in (15, 16, 17, 18):
        a, b = ph[300:316], ph[900:916]
        add(bg[:40] + a + bg[40:40 + gap] + b + bg[100:160])
    add(bg[:50] + ph[1200:1216] + bg[50:150])                      # exactly one hit
    add(bg[:50] + ph[1200:1232] + bg[50:150])                      # exactly two hits (16 + 16, adjacent)
    f = list(ph[2500:2650])
    f[8] = "N"
    f[140] = "N"
    add("".join(f))
    add(ph[3000:3015])                                             # length 15 and 16
    add(ph[3000:3016])
    # complexity: homopolymer (exactly 1.0), low complexity, reads with N; lengths 0 / 1
    add("A" * 120)
    add(("TC" * 30 + "TTC" * 20)[:110])
    add(_rand(rng, 60) + "N" + _rand(rng, 60))
    add("", [])
    add("G", [30])
    # EE: sequential vs tree sum differ in the last bits
    n_diff = 0
    while n_diff < 4:
        q = _quals(rng, 230, lo=2, hi=41)
        if _differs_from_tree(q):
            add(_rand(rng, 230), q)
            n_diff += 1
    # orient.fwd: forward, reverse complement, both, neither, IUPAC in the prefix
    pr = "GTGCCAGCAGCCGCGGTAA"
    add(pr + _rand(rng, 200))
    add(R.rc(pr + _rand(rng, 200)))
    add(pr + _rand(rng, 180) + R.rc(pr))
    add(_rand(rng, 220))
    add("GTGCCAGCRGCCGCGGTAA" + _rand(rng, 200))
    add(_rand(rng, 20000), _quals(rng, 20000, lo=25))               # 20 000 nt
    return reads, pr


def option_sets(reads):
    """(name, Opts) for single-end runs; maxEE edges are taken from one read's exact EE."""
    ee0 = R.matrix_ee(reads[0][1][:100])
    return [
        ("defaults", R.Opts()),
        ("vignette", R.Opts(trimLeft=10, truncLen=240, maxN=0, maxEE=2)),
        ("trims", R.Opts(trimLeft=19, trimRight=101, truncLen=119, minLen=0, truncQ=0, maxN=3)),
        ("trunclen_lt_start", R.Opts(trimLeft=30, truncLen=20, minLen=0, maxN=1, rm_phix=False)),
        ("maxlen", R.Opts(maxLen=120, minLen=0, truncQ=0, maxN=2)),
        ("maxn_minq", R.Opts(maxN=2, minQ=20, truncQ=1, minLen=0)),
        ("minq_le_truncq", R.Opts(minQ=2, truncQ=2, minLen=0)),
        ("truncq93", R.Opts(truncQ=93, minLen=0)),
        ("ee_equal", R.Opts(truncLen=100, truncQ=0, minLen=0, maxN=20, maxEE=ee0)),
        ("ee_below", R.Opts(truncLen=100, truncQ=0, minLen=0, maxN=20, maxEE=float(np.nextafter(ee0, 0.0)))),
        ("lowc", R.Opts(minLen=2, truncQ=0, maxN=0, rm_lowcomplex=8)),
        ("lowc_high", R.Opts(minLen=2, truncQ=0, maxN=0, rm_lowcomplex=15.2, rm_phix=False)),
    ]


def single_cases():
    """-> list of dict(name, reads, opts, orient, n)."""
    reads, pr = single_pool()
    plain = [r for r in reads if len(r[0]) >= len(pr)]
    out = [dict(name=nm, reads=reads, opts=[o], orient=None, n=100000) for nm, o in option_sets(reads)]
    for n in (1, 7, 1000):
        out.append(dict(name="orient_n%d" % n, reads=plain, opts=[R.Opts(minLen=0, truncQ=0, maxN=20)], orient=pr, n=n))
    for cnt in (0, 1, 31, 32, 33):
        out.append(dict(name="count%d" % cnt, reads=reads[:cnt], opts=[R.Opts()], orient=None, n=100000))
    return out


def paired_cases():
    rng = np.random.default_rng(23)
    reads, pr = single_pool()
    ph = phix()
    pool = [r for r in reads if len(r[0]) >= 20]
    pairs = []
    for k in range(len(pool)):
        pairs.append((pool[k], pool[(k * 7 + 3) % len(pool)]))
    # phiX on one mate only; each mate alone fails a stage
    pairs.append(((ph[10:260], _quals(rng, 250)), (_rand(rng, 250), _quals(rng, 250))))
    pairs.append(((_rand(rng, 250), _quals(rng, 250)), (R.rc(ph)[40:290], _quals(rng, 250))))
    # orientation: primer on F, on R, on both, on neither
    for a, b in ((True, False), (False, True), (True, True), (False, False)):
        fa = (pr if a else "") + _rand(rng, 230 - (len(pr) if a else 0))
        fb = (pr if b else "") + _rand(rng, 230 - (len(pr) if b else 0))
        pairs.append(((fa, _quals(rng, 230)), (fb, _quals(rng, 230))))
    mk = lambda **kw: [R.Opts(**{k: v[0] for k, v in kw.items()}), R.Opts(**{k: v[1] for k, v in kw.items()})]
    out = [
        dict(name="p_defaults", reads=pairs, opts=[R.Opts(), R.Opts()], orient=None, n=100000),
        dict(name="p_vignette", reads=pairs, opts=mk(trimLeft=(10, 10), truncLen=(240, 160), maxN=(0, 0), maxEE=(2, 2)), orient=None, n=100000),
        dict(name="p_permate", reads=pairs, opts=mk(truncQ=(2, 11), trimRight=(0, 30), minLen=(50, 100), maxN=(1, 0), minQ=(0, 8),
                                                    maxLen=(INF, 240), rm_phix=(True, False)), orient=None, n=100000),
        dict(name="p_phix_rev_only", reads=pairs, opts=mk(rm_phix=(False, True), truncQ=(0, 0)), orient=None, n=100000),
        dict(name="p_lowc", reads=pairs, opts=mk(rm_lowcomplex=(0, 9), minLen=(2, 2), truncQ=(0, 0), rm_phix=(False, False)), orient=None,
             n=100000),
    ]
    op = [p for p in pairs if len(p[0][0]) >= len(pr) and len(p[1][0]) >= len(pr)]
    for n in (1, 7):
        out.append(dict(name="p_orient_n%d" % n, reads=op, opts=[R.Opts(minLen=0, truncQ=0, maxN=30), R.Opts(minLen=0, truncQ=0, maxN=30)],
                        orient=pr, n=n))
    return out


def all_cases():
    return single_cases() + paired_cases()


def restate(case):
    nm = len(case["opts"])
    rd = [tuple(r) if nm == 2 else (r,) for r in case["reads"]]
    return R.filter_chunks(rd, case["opts"], case["orient"], phix(), case["n"])


def run_product(case, filter_reads):
    """Runs a case through dada2_b200.filter.filter_reads -> (reason, flags, src, [(seqs, quals) per mate])."""
    nm = len(case["opts"])
    if nm == 1:
        seqs = [r[0] for r in case["reads"]]
        quals = [np.array(r[1], np.uint8) for r in case["reads"]]
        rev = None
    else:
        seqs = [r[0][0] for r in case["reads"]]
        quals = [np.array(r[0][1], np.uint8) for r in case["reads"]]
        rev = ([r[1][0] for r in case["reads"]], [np.array(r[1][1], np.uint8) for r in case["reads"]])
    if nm == 1:
        kw = case["opts"][0].kw()
    else:
        kw = {k: tuple(o.kw()[k] for o in case["opts"]) for k in case["opts"][0].kw()}
    got = filter_reads(seqs, quals, rev, orient_fwd=case["orient"], phix=PHIX_FA, n=case["n"], **kw)
    mates = [(r.strings(), [list(r.qual[r.off[i]:r.off[i + 1]]) for i in range(len(r))]) for r in got["reads"]]
    return got["reason"], got["flags"], got["src"], mates


def check_case(case, got, want):
    """got: run_product's result; want: (reason, flags, src, mates) from the golden file or the restatement."""
    reason, flags, src, mates = got
    wr, wf, ws, wm = want
    name = case["name"]
    assert np.array_equal(reason, wr), (name, np.nonzero(reason != wr)[0][:10], reason[reason != wr][:10], wr[reason != wr][:10])
    assert np.array_equal(flags, wf), (name, np.nonzero(flags != wf)[0][:10])
    assert np.array_equal(src, ws), name
    for m, (s, q) in enumerate(mates):
        assert s == wm[m][0], (name, m)
        assert [list(map(int, x)) for x in q] == [list(map(int, x)) for x in wm[m][1]], (name, m)


def want_from_restatement(case):
    reason, flags, out = restate(case)
    nm = len(case["opts"])
    src = np.array([o[0] for o in out], np.int32)
    mates = [([o[1][m][0] for o in out], [o[1][m][1] for o in out]) for m in range(nm)]
    return reason, flags, src, mates


def load_golden():
    return np.load(GOLDEN)


def want_from_golden(g, case):
    k = case["name"]
    nm = len(case["opts"])
    mates = []
    for m in range(nm):
        off = g[k + "/off%d" % m]
        s = bytes(g[k + "/seq%d" % m]).decode()
        q = g[k + "/qual%d" % m]
        mates.append(([s[off[i]:off[i + 1]] for i in range(len(off) - 1)], [list(q[off[i]:off[i + 1]]) for i in range(len(off) - 1)]))
    return g[k + "/reason"], g[k + "/flags"], g[k + "/src"], mates


def check_stages(case, hook):
    """The stage hook's per-read values against the restatement's: exact, EE bit for bit, complexity within 1e-13."""
    o = case["opts"][0]
    seqs = [r[0] for r in case["reads"]]
    quals = [np.array(r[1], np.uint8) for r in case["reads"]]
    got = hook(seqs, quals, orient_fwd=case["orient"], phix=PHIX_FA, n=case["n"], **{k: v for k, v in o.kw().items() if k != "rm_phix"})
    ph = phix()
    for i, (s, q) in enumerate(case["reads"]):
        w = R.stage_values(s, q, o, case["orient"], ph)
        g = got[i]
        ints = (g["trim_fail"], g["flipped"], g["start"], g["end"], g["n_other"], g["min_q"] if not w[0] else 0, g["hits_fwd"], g["hits_rc"])
        assert ints == (w[0], w[1], w[2], w[3], w[4], w[5], w[7], w[8]), (case["name"], i, ints, w)
        assert float(g["ee"]).hex() == float(w[6]).hex(), (case["name"], i, g["ee"], w[6])
        if w[0]:
            continue
        if math.isnan(w[9]):
            assert math.isnan(g["complexity"]), (case["name"], i)
        else:
            assert abs(g["complexity"] - w[9]) <= 1e-13 * w[9], (case["name"], i, g["complexity"], w[9])


def check_errors_and_helpers():
    import ctypes
    import pytest
    from dada2_b200 import Dada2bError
    from dada2_b200 import filter as fl
    reads, pr = single_pool()
    seqs = [r[0] for r in reads]
    quals = [np.array(r[1], np.uint8) for r in reads]
    ph = phix()
    with pytest.raises(Dada2bError, match="shorter than orient.fwd"):
        fl.filter_reads(seqs, quals, orient_fwd=pr, phix=ph)
    with pytest.raises(Dada2bError, match="Mismatched forward and reverse"):
        fl.filter_reads(seqs[:5], quals[:5], (seqs[:4], quals[:4]), phix=ph)
    with pytest.raises(Dada2bError, match="Encoding for this truncQ"):
        fl.filter_reads(seqs[:5], quals[:5], truncQ=94, phix=ph)
    with pytest.raises(Dada2bError, match="upper-case IUPAC"):
        fl.filter_reads(["ACGTacgt" * 5], [np.full(40, 30, np.uint8)], phix=ph)
    with pytest.raises(Dada2bError, match="NA"):
        fl.filter_reads(["AN" + "A" * 30, "A"], [np.full(32, 30, np.uint8), np.full(1, 30, np.uint8)], minLen=0, maxN=5,
                        rm_lowcomplex=2, rm_phix=False)
    bad_q = [np.full(40, 30, np.uint8), np.full(40, 30, np.uint8)]
    bad_q[1][17] = 200                                             # rejected before any kernel indexes the EE table with it
    with pytest.raises(Dada2bError, match="quality values must be 0..93"):
        fl.filter_reads(["ACGT" * 10] * 2, bad_q, phix=ph)
    with pytest.raises(Dada2bError, match="quality values must be 0..93"):
        fl.test_filter_stages(["ACGT" * 10] * 2, bad_q, phix=ph)
    with pytest.raises(Dada2bError, match="quality values must be 0..93"):
        fl.filter_reads(["ACGT" * 10] * 2, bad_q, (["ACGT" * 10] * 2, [np.full(40, 30, np.uint8)] * 2), phix=ph)
    with pytest.raises(Dada2bError, match="maxLen must be >= 0"):
        fl.filter_reads(seqs[:3], quals[:3], maxLen=-5, phix=ph)
    for fn in (lambda: fl._lib().dada2b_match_ref(-1, b"", np.zeros(1, np.int64).ctypes.data, ph.encode(), 16, 1, 0, None, eb),
               lambda: fl._lib().dada2b_seq_complexity(-1, b"", np.zeros(1, np.int64).ctypes.data, 2, 0, 0, None, eb)):
        eb = ctypes.create_string_buffer(256)
        assert fn() != 0 and b"negative sequence count" in eb.value
    with pytest.raises(Dada2bError, match="phiX genome"):
        fl.filter_reads(seqs[:3], quals[:3])
    with pytest.raises(Dada2bError, match="window"):
        fl.seqComplexity(seqs[:3], window=25)
    # C_matchRef at word sizes 1 / 8 / 15 / 16, both non_overlapping values, against the restatement
    for w in (1, 8, 15, 16):
        for nov in (True, False):
            assert np.array_equal(fl.C_matchRef(seqs, ph, w, nov), R.match_ref(seqs, ph, w, nov)), (w, nov)
    assert np.array_equal(fl.isPhiX(seqs, PHIX_FA), np.array([R.is_phix(s, ph) for s in seqs]))
    for k in (1, 2, 3, 4):
        got = fl.seqComplexity(seqs, kmerSize=k)
        want = np.array([R.complexity(s, k) for s in seqs])
        nan = np.isnan(want)
        assert np.array_equal(nan, np.isnan(got)), k
        assert np.all(np.abs(got[~nan] - want[~nan]) <= 1e-13 * want[~nan]), k
    assert fl.seqComplexity(["A" * 120])[0] == 1.0


def read_at(reads, i):
    a, b = reads.off[i], reads.off[i + 1]
    return reads.seq[a:b].decode(), [int(x) for x in reads.qual[a:b]]


def synthetic_reads(N, L, seed=1, primer=None):
    """N reads of L nt (a dada2_b200.filter.Reads): Illumina-like qualities with low tails, ~2% with an N or an IUPAC
    code, ~3% spliced phiX fragments of either strand, ~2% low-complexity reads; with a primer, reads start with it, a
    third of them reverse-complemented."""
    from dada2_b200.filter import Reads
    rng = np.random.default_rng(seed)
    nt = np.frombuffer(b"ACGT", np.uint8)
    codes = rng.integers(0, 4, (N, L), dtype=np.uint8)
    seq = nt[codes]
    prof = np.clip(np.round(38 - 20 * (np.arange(L) / (L - 1)) ** 3), 2, 40)
    q = np.clip(np.round(prof[None, :] + rng.normal(0, 4, (N, L))), 0, 41).astype(np.uint8)
    tail = rng.random(N) < 0.2
    q[tail, L - 40:] = rng.integers(0, 12, (int(tail.sum()), 40), dtype=np.uint8)
    amb = np.nonzero(rng.random(N) < 0.02)[0]
    seq[amb, rng.integers(0, L, len(amb))] = np.frombuffer(b"NRYN", np.uint8)[rng.integers(0, 4, len(amb))]
    ph = np.frombuffer(phix().encode(), np.uint8)
    prc = np.frombuffer(R.rc(phix()).encode(), np.uint8)
    pk = np.nonzero(rng.random(N) < 0.03)[0]
    for i in pk:
        g = ph if rng.random() < 0.5 else prc
        ln = int(rng.integers(20, L))
        st = int(rng.integers(0, len(g) - ln))
        at = int(rng.integers(0, L - ln + 1))
        seq[i, at:at + ln] = g[st:st + ln]
    lc = np.nonzero(rng.random(N) < 0.02)[0]
    seq[lc] = np.frombuffer(b"TC", np.uint8)[rng.integers(0, 2, (len(lc), L))]
    if primer:
        p = np.frombuffer(primer.encode(), np.uint8)
        seq[:, :len(p)] = p
        fl = rng.random(N) < 1 / 3
        comp = np.zeros(256, np.uint8)
        for a, b in zip(b"ACGTNRY", b"TGCANYR"):
            comp[a] = b
        seq[fl] = comp[seq[fl][:, ::-1]]
    off = np.arange(N + 1, dtype=np.int64) * L
    return Reads(seq.tobytes(), off, q.ravel())


def vector_reasons(st, opts):
    """Stages 8-12 restated as vectorised predicates over the stage hook's values of each mate (no orient.fwd).
    -> (reason, flags) as dada2b_filter defines them."""
    nm = len(st)
    N = len(st[0])
    f = np.zeros((nm, N), np.int64)
    low = np.zeros((nm, N), np.int64)
    for m, o in enumerate(opts):
        s = st[m]
        fm = s["trim_fail"].astype(np.int64)
        live = fm == 0
        c = live & (s["n_other"] > o.maxN); fm[c] = 8; live &= ~c
        if o.minQ > o.truncQ:
            c = live & ~(s["min_q"] > o.minQ); fm[c] = 9; live &= ~c
        if o.maxEE < INF:
            c = live & (s["ee"] > o.maxEE); fm[c] = 10; live &= ~c
        if o.rm_phix:
            c = live & ((s["hits_fwd"] >= 2) | (s["hits_rc"] >= 2)); fm[c] = 11; live &= ~c
        if (o.rm_lowcomplex != 0) if nm == 2 else (o.rm_lowcomplex > 0):
            cx = s["complexity"]
            assert not np.any(live & np.isnan(cx))
            low[m] = live & (cx < o.rm_lowcomplex)
        f[m] = fm
    fz = np.where(f == 0, 99, f)
    why = fz.min(axis=0)
    why[why == 99] = 0
    flags = np.zeros(N, np.int64)
    for m in range(nm):
        flags |= np.where((why > 0) & (f[m] == why), 1 << m, 0)
    lowany = (why == 0) & low.any(axis=0)
    for m in range(nm):
        flags |= np.where(lowany & (low[m] == 1), 1 << m, 0)
    why[lowany] = 12
    return why.astype(np.uint8), flags.astype(np.uint8)
