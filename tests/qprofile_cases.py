"""Cases of plotQualityProfile / plotComplexity and the per-cycle quality tally (dd_qprofile.cu), shared by
tests/test_emu_qprofile.py (host SIMT emulator) and tests/test_gpu_zz_qprofile.py (H100).  Every case is checked against
tests/qprofile_ref.py: tallies equal as int64 arrays, every frame column equal (float64 columns bit for bit)."""
import gzip
import os

import numpy as np
import pytest

from tests import qprofile_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TILE = 128                                  # cycles per work item of k_qp_tally
ACGT = np.frombuffer(b"ACGT", np.uint8)


def gold(name):
    return os.path.join(GOLD, name + ".fastq.gz")


def write_fastq(path, seqs, quals):
    recs = "".join("@r%d\n%s\n+\n%s\n" % (i, s, "".join(chr(33 + int(x)) for x in q)) for i, (s, q) in enumerate(zip(seqs, quals)))
    op = gzip.open if path.endswith(".gz") else open
    with op(path, "wt") as f:
        f.write(recs)
    return path


def random_reads(rng, lens, qual_fn):
    seqs = [ACGT[rng.integers(0, 4, k)].tobytes().decode() for k in lens]
    return seqs, [qual_fn(k) for k in lens] if qual_fn else None


def synthetic_files(d):
    """name -> path of the synthetic fastq files, written under d."""
    rng = np.random.default_rng(11)
    out = {}
    q = np.zeros((94, 3), np.uint8)                         # every score 0..93 at cycle 1
    q[:, 0] = np.arange(94)
    q[:, 1:] = rng.integers(0, 94, (94, 2))
    out["allscores"] = write_fastq(os.path.join(d, "allscores.fastq"), random_reads(rng, [3] * 94, None)[0], list(q))
    bins = np.array([2, 12, 23, 37], np.uint8)              # NovaSeq-like binned qualities, most bases at 37
    s, ql = random_reads(rng, [151] * 2000, lambda k: bins[rng.choice(4, k, p=[0.02, 0.05, 0.13, 0.8])])
    out["binned"] = write_fastq(os.path.join(d, "binned.fastq.gz"), s, ql)
    lens = np.concatenate([rng.integers(1, 601, 700), [0] * 12, [600, 1]])   # ragged 1..600, zero-length reads among them
    rng.shuffle(lens)
    s, ql = random_reads(rng, lens, lambda k: rng.integers(0, 42, k).astype(np.uint8))
    out["ragged"] = write_fastq(os.path.join(d, "ragged.fastq"), s, ql)
    out["single"] = write_fastq(os.path.join(d, "single.fastq"), ["ACGTN"], [np.array([40, 3, 93, 0, 17], np.uint8)])
    lens = [TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1] * 20
    s, ql = random_reads(rng, lens, lambda k: rng.integers(0, 94, k).astype(np.uint8))
    out["tiles"] = write_fastq(os.path.join(d, "tiles.fastq.gz"), s, ql)
    s, ql = random_reads(rng, rng.integers(200, 260, 3000), lambda k: rng.integers(10, 41, k).astype(np.uint8))
    out["large"] = write_fastq(os.path.join(d, "large.fastq.gz"), s, ql)   # above the small n of the sampled cases
    lowc = ["A" * 80, "ACACACACAC" * 8, "NNNNNNNNNN", "", "ANANANANAN", "G", "ACGTN" * 30]
    s = random_reads(rng, [250] * 40, None)[0] + lowc
    out["cplx"] = write_fastq(os.path.join(d, "cplx.fastq"), s, [np.full(len(x), 30, np.uint8) for x in s])
    open(os.path.join(d, "empty.fastq"), "w").close()
    out["empty"] = os.path.join(d, "empty.fastq")
    return out


def profile_cases(files):
    """(label, fl, kwargs) of plotQualityProfile."""
    g = {k: gold(k) for k in ("sam1F", "sam1R", "sam2F", "sam2R", "samPB", "samPBprimers")}
    return [
        ("sam1F", g["sam1F"], {}),
        ("sam1R+sam2R", [g["sam1R"], g["sam2R"]], {}),
        ("sam1F+sam2F aggregate", [g["sam1F"], g["sam2F"]], {"aggregate": True}),
        ("three files with None", [g["sam1F"], None, g["sam2F"], g["sam1R"], None], {}),
        ("three files with None aggregate", [None, g["sam1F"], g["sam2F"], None, g["sam1R"]], {"aggregate": True}),
        ("samPB", g["samPB"], {"n": None}),
        ("samPBprimers", g["samPBprimers"], {}),
        ("allscores", files["allscores"], {}),
        ("binned", files["binned"], {"n": 1000, "seed": 2}),
        ("ragged", files["ragged"], {"n": None}),
        ("single", files["single"], {"n": 1}),
        ("tiles", [files["tiles"], files["allscores"]], {"aggregate": True}),
        ("large sampled", files["large"], {"n": 1000, "seed": 5}),
        ("large sampled aggregate", [files["large"], files["binned"], files["large"]], {"n": 1500, "seed": 9, "aggregate": True}),
    ]


def complexity_cases(files):
    return [
        ("sam1F sampled", gold("sam1F"), {"n": 300, "seed": 3}),
        ("cplx + samPBprimers", [files["cplx"], None, gold("samPBprimers")], {}),
        ("aggregate", [files["cplx"], files["large"]], {"n": 100, "seed": 4, "aggregate": True, "kmerSize": 3}),
    ]


def same_float(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def check_frames(label, got, want):
    for frame in ("plotdf", "statdf", "anndf"):
        g, w = got[frame], want[frame]
        assert sorted(g) == sorted(w), (label, frame, sorted(g), sorted(w))
        for col in w:
            if col in ("Mean", "Cum", "minScore"):
                assert same_float(g[col], w[col]), (label, frame, col)
            elif col in ("file", "label", "rclabel"):
                assert list(g[col]) == list(w[col]), (label, frame, col)
            else:
                assert np.array_equal(np.asarray(g[col], np.int64), np.asarray(w[col], np.int64)), (label, frame, col)
    assert np.array_equal(got["nreads"], want["nreads"]), label


def check_profiles(d):
    """Every plotQualityProfile case and its per-file tallies against the restatement."""
    import dada2_b200
    from dada2_b200 import filter as fl, qc
    files = synthetic_files(d)
    for label, f, kw in profile_cases(files):
        want = R.plot_quality_profile(f, **kw)
        check_frames(label, dada2_b200.plotQualityProfile(f, **kw), want)
        paths = [f] if isinstance(f, str) else [x for x in f if x is not None]
        rng = np.random.default_rng(kw.get("seed"))
        for path, counts in zip(paths, want["counts"]):
            _, reads = fl.read_fastq_records(path)
            idx = R.select(len(reads), kw.get("n", 500000), rng)
            sub = qc.gather(reads, idx)
            got, st = qc.quality_tally(sub.off, sub.qual)
            assert got.dtype == np.int64 and np.array_equal(got, counts), (label, path)
            assert st["nreads"] == len(idx) and st["nbases"] == int(counts.sum())


def check_complexity(d):
    import dada2_b200
    files = synthetic_files(d)
    for label, f, kw in complexity_cases(files):
        got = dada2_b200.plotComplexity(f, **kw)
        want = R.plot_complexity(f, **kw)
        assert got["file"] == want["file"], label
        g, w = got["complexity"], np.array(want["complexity"], np.float64)
        assert g.dtype == np.float64 and len(g) == len(w), label
        assert np.array_equal(np.isnan(g), np.isnan(w)), label
        ok = ~np.isnan(w)
        assert np.all(np.abs(g[ok] - w[ok]) <= 1e-13 * w[ok]), label


def check_edges_and_refusals(d):
    """Zero reads and zero-length reads through the C entry, the labels, and every refusal."""
    import dada2_b200
    from dada2_b200 import Dada2bError, qc
    files = synthetic_files(d)
    c, st = qc.quality_tally(np.zeros(1, np.int64), np.zeros(0, np.uint8))
    assert c.shape == (0, 94) and st["nreads"] == 0
    c, st = qc.quality_tally(np.zeros(4, np.int64), np.zeros(0, np.uint8))
    assert c.shape == (0, 94) and st["nreads"] == 3 and st["nbases"] == 0
    for bad in (94, 255):
        q = np.full(300, 30, np.uint8)
        q[257] = bad
        with pytest.raises(Dada2bError, match=r"quality values must be 0\.\.93"):
            qc.quality_tally(np.array([0, 10, 300], np.int64), q)
    for n, over, under in ((500000, "Reads >=  5e+05", "Reads:  499999"), (250000, "Reads >=  250000", "Reads:  1234"),
                           (100000, "Reads >=  1e+05", "Reads:  99999"), (1000, "Reads >=  1000", "Reads:  999")):
        assert qc.rclabel(n, n) == over and qc.rclabel(int(under.split()[-1]), n) == under
        assert R.paste("Reads >= ", R.as_character(n)) == over
    assert qc.rclabel(10 ** 7, None) == "Reads:  10000000"
    got = dada2_b200.plotQualityProfile(gold("sam1F"), n=None)
    assert got["anndf"]["rclabel"] == ["Reads:  1500"] and got["nreads"].tolist() == [1500]
    got = dada2_b200.plotQualityProfile(gold("sam1F"), n=1000, seed=1)
    assert got["anndf"]["rclabel"] == ["Reads >=  1000"] and got["anndf"]["rc"].tolist() == [1000]
    for n in (0, -3, 0.5):
        with pytest.raises(Dada2bError, match="n must be"):
            dada2_b200.plotQualityProfile(gold("sam1F"), n=n)
    with pytest.raises(Dada2bError, match="nosuch.fastq"):
        dada2_b200.plotQualityProfile([gold("sam1F"), os.path.join(d, "nosuch.fastq")])
    with pytest.raises(Dada2bError, match="empty.fastq"):
        dada2_b200.plotQualityProfile(files["empty"])
    with pytest.raises(Dada2bError, match="empty.fastq"):
        dada2_b200.plotComplexity(files["empty"])
    with pytest.raises(Dada2bError, match="window"):
        dada2_b200.plotComplexity(gold("sam1F"), window=20)
