"""Seeded reads and option sets at the edges of removePrimers' rules (tests/primer_ref.py), shared by the golden
generator (tools/make_golden_primer.py -> tests/golden/primer.npz), the emulator tests and the H100 tests."""
import os

import numpy as np

from tests import primer_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "primer.npz")
SAM_PB_PRIMERS = os.path.join(HERE, "golden", "samPBprimers.fastq.gz")
SAM_PB = os.path.join(HERE, "golden", "samPB.fastq.gz")
F27 = "AGRGTTYGATYMTGGCTCAG"                                        # the man page's primers
R1492 = "RGYTACCTTGTTACGACTT"
PF = "GTGCCAGCAGCCGCGGTAA"                                         # A/C/G/T only: fixed matching
PR = "ATTAGATACCCTGGTAGTCC"


def _rand(rng, n):
    return "".join("ACGT"[i] for i in rng.integers(0, 4, n))


def _q(rng, n):
    return [int(x) for x in rng.integers(0, 94, n)]


def mutate(p, pos, rng):
    """p with a base outside the letter's IUPAC set at each position in pos (a sure mismatch)."""
    s = list(p)
    for j in pos:
        s[j] = rng.choice([b for b in "ACGT" if not (R.MASK[b] & R.MASK[s[j]])])
    return "".join(s)


def pool(pf, pr, k, seed):
    """Reads around one primer pair; the comments name the edge."""
    rng = np.random.default_rng(seed)
    reads = []
    add = lambda s: reads.append((s, _q(rng, len(s))))
    body = lambda n=60: _rand(rng, n)
    P = len(pf)
    add(pf + body() + pr)                                          # hit at offset 0 and at the read's end
    add(body(30) + pf + body() + pr + body(25))                    # mid-read
    add(body(5) + mutate(pf, rng.choice(P, k, replace=False), rng) + body() + mutate(pr, [1, len(pr) - 2][:k], rng) + body(3))   # exactly k
    add(body(5) + mutate(pf, rng.choice(P, k + 1, replace=False), rng) + body() + pr)                                         # k + 1
    for d in range(1, k + 2):                                      # off the left / right end by 1..k (hit) and k + 1 (none)
        add(pf[d:] + body() + pr)
        add(pf + body() + pr[:-d])
    add(R.rc(pf + body() + pr))                                    # reverse complement only: flipped
    add(pf + body() + pr + R.rc(pf))                               # forward primer on both strands: not flipped
    add(body(120))                                                 # neither
    add(pf + body() + R.rc(pr))                                    # reverse primer on the wrong strand
    add(pf + pr)                                                   # window of 0 bases
    add(pf + "A" + pr)                                             # 1 base: dropped
    add(pf + "AC" + pr)                                            # 2 bases: kept
    add(pr + body(4) + pf + body(10))                              # reverse hit before the forward end
    add(pf + body(40) + pf + body() + pr + body(30) + pr)          # separated double hits: first fwd, last rev
    t = list(pf + body() + pr)
    t[3] = "N"                                                     # N / IUPAC letters in the primer sites
    t[-4] = "R"
    add("".join(t))
    add(pf[: P // 2])                                              # shorter than the primer
    add(pf[0])                                                     # 1 nt
    add("")                                                        # empty read
    return reads


def letters_pool(seed=5):
    """k = 0 reads that decide rule 1: N / R / Y in the read against F27 (IUPAC) and N against PF (fixed)."""
    rng = np.random.default_rng(seed)
    out = []
    for pf in (F27, PF):
        a = pf.index("A")
        for c in ("N", "R", "Y", "W", "A"):
            s = list(pf)
            s[a] = c
            r = "".join(s) + _rand(rng, 50)
            out.append((r, _q(rng, len(r))))
    return out


def multi_pool(seed=9):
    """Overlapping and separated multiple hits of a periodic primer."""
    rng = np.random.default_rng(seed)
    out = []
    for s in ("ACACACACAC" + "AC" * 3 + _rand(rng, 40) + "GGTTGGTTCC",
              _rand(rng, 10) + "ACACACACAC" + _rand(rng, 30) + "ACACACACAC" + _rand(rng, 20) + "GGTTGGTTCC" + _rand(rng, 5) + "GGTTGGTTCC",
              "GGAACCAACC" + _rand(rng, 30) + "GTGTGTGTGTGT"):
        out.append((s, _q(rng, len(s))))
    return out


def cases():
    """-> list of dict(name, reads, pf, pr, k, trim_fwd, trim_rev, orient)."""
    rng = np.random.default_rng(3)
    fixed = pool(PF, PR, 2, 1)
    iupac = pool(F27, R.rc(R1492), 2, 2)
    mk = lambda name, reads, pf, pr, k=2, tf=True, tr=True, o=True: dict(name=name, reads=reads, pf=pf, pr=pr, k=k, trim_fwd=tf,
                                                                         trim_rev=tr, orient=o)
    P64 = _rand(rng, 64)
    p64 = pool(P64, PR, 3, 4)
    short = [(s, _q(rng, len(s))) for s in ("ACGT", "TTACGTAA", "A", "GG", "ACGTACGTACGT", "CCCCCC")]
    out = [
        mk("fixed_k2", fixed, PF, PR),
        mk("iupac_k2", iupac, F27, R.rc(R1492)),
        mk("fixed_k0", fixed, PF, PR, k=0),
        mk("fixed_k1", fixed, PF, PR, k=1),
        mk("iupac_k3", iupac, F27, R.rc(R1492), k=3),
        mk("no_trim_fwd", fixed, PF, PR, tf=False),
        mk("no_trim_rev", fixed, PF, PR, tr=False),
        mk("no_orient", fixed, PF, PR, o=False),
        mk("no_rev", fixed, PF, None),
        mk("no_rev_no_trim", fixed, PF, None, tf=False),
        mk("k_ge_P", short, "ACGT", "TTA", k=5),
        mk("k_eq_P", short, "ACGT", "TTA", k=4),
        mk("k_eq_P1", short, "ACGT", "TTA", k=3),
        mk("letters_k0", letters_pool(), F27, None, k=0),
        mk("letters_k0_fixed", letters_pool(), PF, None, k=0),
        mk("multi", multi_pool(), "ACACACACAC", "GGTTGGTTCC", k=2),
        mk("multi_k0", multi_pool(), "ACACACACAC", "GGTTGGTTCC", k=0),
        mk("p64", p64, P64, PR, k=3),
        mk("all_rc", [(R.rc(s), q[::-1]) for s, q in fixed[:2]], PF, PR),                    # skipped: no forward hit as read
        mk("no_rev_hit", [(PF + _rand(rng, 50), _q(rng, 69))], PF, PR),                       # skipped: no reverse hit as read
        mk("empty_file", [], PF, PR),
        mk("zero_out", [(PF + "A" + PR, _q(rng, 40))] * 2, PF, PR),                          # not skipped, nothing kept
    ]
    return out


def restate(case):
    return R.remove_primers(case["reads"], case["pf"], case["pr"], case["k"], case["trim_fwd"], case["trim_rev"], case["orient"])


def restate_hits(case):
    h = np.zeros((len(case["reads"]), 4, 5), np.int32)
    for i, (s, _) in enumerate(case["reads"]):
        h[i] = R.scans(s, case["pf"], case["pr"], case["k"])
    return h


def run_product(case, fn):
    seqs = [r[0] for r in case["reads"]]
    quals = [np.array(r[1], np.uint8) for r in case["reads"]]
    return fn(seqs, quals, case["pf"], case["pr"], max_mismatch=case["k"], trim_fwd=case["trim_fwd"], trim_rev=case["trim_rev"],
              orient=case["orient"])


def check_case(case, got, want):
    """got: remove_primers_reads' result; want: dict(reason, flags, skipped, multi, src, seqs, quals)."""
    nm = case["name"]
    assert np.array_equal(got["reason"], want["reason"]), (nm, got["reason"], want["reason"])
    assert np.array_equal(got["flags"], want["flags"]), (nm, got["flags"], want["flags"])
    assert got["skipped"] == want["skipped"] and got["multi"] == want["multi"], nm
    assert np.array_equal(got["src"], want["src"]), nm
    r = got["reads"]
    assert r.strings() == list(want["seqs"]), nm
    assert [list(map(int, r.qual[r.off[i]:r.off[i + 1]])) for i in range(len(r))] == [list(map(int, q)) for q in want["quals"]], nm


def want_from_restatement(case):
    w = restate(case)
    return dict(reason=w["reason"], flags=w["flags"], skipped=w["skipped"], multi=w["multi"], src=np.array([o[0] for o in w["out"]], np.int32),
                seqs=[o[1] for o in w["out"]], quals=[o[2] for o in w["out"]])


def want_from_golden(g, case):
    k = case["name"]
    off = g[k + "/off"]
    s = bytes(g[k + "/seq"]).decode()
    q = g[k + "/qual"]
    n = len(off) - 1
    return dict(reason=g[k + "/reason"], flags=g[k + "/flags"], skipped=bool(g[k + "/skipped"]), multi=bool(g[k + "/multi"]), src=g[k + "/src"],
                seqs=[s[off[i]:off[i + 1]] for i in range(n)], quals=[list(q[off[i]:off[i + 1]]) for i in range(n)])


def load_golden():
    return np.load(GOLDEN)


def check_hits(case, hook, want):
    """hook: primer.test_primer_hits; want: [n, 4, 5] (count, first start / end, last start / end)."""
    if not case["reads"]:
        return
    seqs = [r[0] for r in case["reads"]]
    quals = [np.array(r[1], np.uint8) for r in case["reads"]]
    got = hook(seqs, quals, case["pf"], case["pr"], max_mismatch=case["k"], orient=case["orient"])
    g = np.stack([got[f] for f in ("count", "first_start", "first_end", "last_start", "last_end")], axis=-1)
    bad = np.nonzero((g != want).any(axis=(1, 2)))[0]
    assert len(bad) == 0, (case["name"], bad[:5], g[bad[:2]].tolist(), want[bad[:2]].tolist())


def write_fastq(path, ids, reads, gz=True):
    import gzip
    data = R.fastq_bytes(ids, [r[0] for r in reads], [r[1] for r in reads])
    with (gzip.open(path, "wb") if gz else open(path, "wb")) as f:
        f.write(data)


def check_files(tmpdir):
    """removePrimers over files: an ordinary file, one with no survivor, one skipped (no file written); then all files
    with 0 reads out (R's warning); an existing output file is replaced; the return matrix."""
    import warnings
    import pytest
    from dada2_b200 import Dada2bError, primer
    c = {x["name"]: x for x in cases()}
    names = ("fixed_k2", "zero_out", "all_rc")
    fn, fo = [], []
    for nm in names:
        p = os.path.join(tmpdir, nm + ".fastq.gz")
        write_fastq(p, [b"r%d" % i for i in range(len(c[nm]["reads"]))], c[nm]["reads"])
        fn.append(p)
        fo.append(os.path.join(tmpdir, "out", nm + ".fastq.gz"))
    os.makedirs(os.path.join(tmpdir, "out"))
    with open(fo[0], "wb") as f:
        f.write(b"stale")
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        m = primer.removePrimers(fn, fo, PF, PR, verbose=True)
    w = [want_from_restatement(c[nm]) for nm in names]
    assert m.tolist() == [[len(c[nm]["reads"]), len(x["src"])] for nm, x in zip(names, w)]
    import gzip
    ids = [b"r%d" % i for i in w[0]["src"]]
    assert gzip.open(fo[0]).read() == R.fastq_bytes(ids, w[0]["seqs"], w[0]["quals"])
    assert gzip.open(fo[1]).read() == b""                            # no survivor, not skipped: an empty file
    assert not os.path.exists(fo[2])                                 # skipped: no file
    with pytest.warns(UserWarning, match="No reads passed the primer detection"):
        m = primer.removePrimers(fn[1:], fo[1:], PF, PR, compress=False)
    assert m[:, 1].tolist() == [0, 0]
    with pytest.raises(Dada2bError, match="allow.indels"):
        primer.removePrimers(fn[:1], fo[:1], PF, PR, allow_indels=True)
    with pytest.raises(Dada2bError, match="distinct from the input"):
        primer.removePrimers(fn[:1], fn[:1], PF, PR)
    with pytest.raises(Dada2bError, match="corresponding output"):
        primer.removePrimers(fn, fo[:1], PF, PR)


def check_errors():
    import pytest
    from dada2_b200 import Dada2bError, primer
    s, q = ["ACGT" * 10], [np.full(40, 30, np.uint8)]
    for kw, msg in ((dict(primer_fwd=""), "empty"), (dict(primer_fwd="ACGU"), "upper-case IUPAC"), (dict(primer_fwd="acgt"), "upper-case IUPAC"),
                    (dict(primer_fwd="A" * 65), "longer than 64"), (dict(primer_fwd="ACGT", primer_rev="A-C"), "upper-case IUPAC"),
                    (dict(primer_fwd="ACGT", max_mismatch=-1), "max.mismatch"), (dict(primer_fwd="ACGT", allow_indels=True), "allow.indels")):
        with pytest.raises(Dada2bError, match=msg):
            primer.remove_primers_reads(s, q, **kw)
    with pytest.raises(Dada2bError, match="upper-case IUPAC"):
        primer.remove_primers_reads(["ACGTacgt" * 5], q, "ACGT")
    bad = np.full(40, 30, np.uint8)
    bad[7] = 120
    with pytest.raises(Dada2bError, match="quality values must be 0..93"):
        primer.remove_primers_reads(s, [bad], "ACGT")
    with pytest.raises(Dada2bError, match="quality values must be 0..93"):
        primer.test_primer_hits(s, [bad], "ACGT")
    r = primer.remove_primers_reads(["A" * 64 + "TTTT"], [np.full(68, 30, np.uint8)], "A" * 64, max_mismatch=0, trim_fwd=True)
    assert r["src"].tolist() == [0] and r["seqs"] == ["TTTT"]       # a 64-nt primer is accepted


def synthetic_ccs(N, seed=1):
    """N CCS-like reads of 1400-1600 nt with qualities up to 93: F27 at the start and rc(R1492) at the end with 0-3
    mismatches, some cut off at an end (out of limits), some doubled, half of the reads reverse-complemented.
    -> (filter.Reads, is_rc bool[N])."""
    from dada2_b200.filter import Reads
    rng = np.random.default_rng(seed)
    pf, pr = F27, R.rc(R1492)
    conc = lambda p: "".join(rng.choice(sorted(b for b in "ACGT" if R.MASK[b] & R.MASK[c])) for c in p)
    seqs = []
    is_rc = rng.random(N) < 0.5
    lens = rng.integers(1400, 1601, N)
    nt = np.frombuffer(b"ACGT", np.uint8)
    for i in range(N):
        a = conc(pf)
        b = conc(pr)
        a = mutate(a, rng.choice(len(a), int(rng.integers(0, 4)), replace=False), rng) if rng.random() < 0.5 else a
        b = mutate(b, rng.choice(len(b), int(rng.integers(0, 4)), replace=False), rng) if rng.random() < 0.5 else b
        u = rng.random()
        if u < 0.03:
            a = a[int(rng.integers(1, 4)):]                      # cut at the left end
        elif u < 0.06:
            b = b[:-int(rng.integers(1, 4))]                     # cut at the right end
        mid = nt[rng.integers(0, 4, int(lens[i]) - len(a) - len(b))].tobytes().decode()
        if rng.random() < 0.02:
            j = int(rng.integers(0, len(mid) - 30))
            mid = mid[:j] + conc(pf if rng.random() < 0.5 else pr) + mid[j + 20:]   # a second hit inside
        s = a + mid + b
        seqs.append(R.rc(s) if is_rc[i] else s)
    L = np.fromiter(map(len, seqs), np.int64, N)
    off = np.zeros(N + 1, np.int64)
    np.cumsum(L, out=off[1:])
    q = rng.integers(0, 94, int(off[-1]), dtype=np.uint8)
    q[rng.random(int(off[-1])) < 0.6] = 93
    return Reads("".join(seqs).encode(), off, q), is_rc
