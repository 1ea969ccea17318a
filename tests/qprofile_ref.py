"""Restatement of plotQualityProfile and plotComplexity (R/plot-methods.R:163-243, :293-309) up to their ggplot calls, for
the tests.  Independent of dada2_b200: its own fastq reader, the tally as np.bincount(cycle * 94 + q) over the selected
reads, and R's function bodies statement by statement (rowsum, by/get_quant in float64, aggregate, pmin, paste /
as.character).  Complexities through tests/filter_ref.complexity.

Sampling is the product's documented draw (one numpy.random.default_rng(seed) per call; for each file above n in order,
np.sort(rng.choice(nrec, n, replace=False))); a file with at most n reads is used whole, as R uses it."""
import gzip
import os

import numpy as np

from tests import filter_ref

NS = 94


def read_fastq(path):
    """-> (sequences list[str], qualities list[uint8 array]) of a Phred+33 four-line fastq(.gz)."""
    op = gzip.open if str(path).endswith(".gz") else open
    with op(path, "rt") as f:
        lines = f.read().split("\n")
    if lines and lines[-1] == "":
        lines.pop()
    seqs = lines[1::4]
    quals = [np.array([ord(c) - 33 for c in q], np.uint8) for q in lines[3::4]]
    return seqs, quals


def select(nrec, n, rng):
    """Indices of the reads used: all when n is None or nrec <= n."""
    if n is None or nrec <= n:
        return np.arange(nrec)
    return np.sort(rng.choice(nrec, n, replace=False))


def tally(quals):
    """int64[ncycles, 94]: bases with score s at 0-based cycle c."""
    lens = np.array([len(q) for q in quals], np.int64)
    nc = int(lens.max(initial=0))
    if nc == 0:
        return np.zeros((0, NS), np.int64)
    q = np.concatenate(quals).astype(np.int64)
    cyc = np.concatenate([np.arange(k, dtype=np.int64) for k in lens])
    return np.bincount(cyc * NS + q, minlength=nc * NS).astype(np.int64).reshape(nc, NS)


def tally_packed(off, qual, chunk=1 << 25):
    """tally() of reads in dada2b_derep_in's layout (off int64[n+1] into qual), in slices of about `chunk` bases."""
    lens = np.diff(off)
    nc = int(lens.max(initial=0))
    out = np.zeros(nc * NS, np.int64)
    r = 0
    while r < len(lens):
        e = int(np.searchsorted(off, off[r] + chunk, side="right"))
        e = max(e - 1, r + 1)
        a, b = int(off[r]), int(off[e])
        cyc = np.arange(b - a, dtype=np.int64) - np.repeat(off[r:e] - a, lens[r:e])
        out += np.bincount(cyc * NS + qual[a:b], minlength=nc * NS)
        r = e
    return out.reshape(nc, NS)


def per_cycle_quality(counts):
    """qa()$perCycle$quality as read from its use: rows (Cycle, Score, Count) with Count > 0, by cycle then score."""
    rows = [(c + 1, s, int(counts[c, s])) for c in range(counts.shape[0]) for s in range(NS) if counts[c, s] > 0]
    return {"Cycle": [r[0] for r in rows], "Score": [r[1] for r in rows], "Count": [r[2] for r in rows]}


def as_character(x):
    """R's as.character(<double>) for a whole number: fixed unless the scientific form (fewest digits that give x back)
    is narrower."""
    x = float(x)
    fixed = "%.0f" % x
    for sig in range(1, 16):
        sci = "%.*e" % (sig - 1, x)
        if float(sci) == x:
            break
    return fixed if len(fixed) <= len(sci) else sci


def paste(*args):
    return " ".join(str(a) for a in args)


def rowsum(x, g):
    """rowsum(x, g) -> (sorted unique groups, sums)."""
    keys = sorted(set(g))
    acc = {k: 0 for k in keys}
    for v, k in zip(x, g):
        acc[k] += v
    return keys, [acc[k] for k in keys]


def by(df, g, fun):
    """by(df, g, fun, simplify=TRUE): fun on each group's rows (in row order), groups in sorted order."""
    rows = {}
    for i, v in enumerate(g):
        rows.setdefault(v, []).append(i)
    return [fun({c: [df[c][i] for i in rows[k]] for c in df}) for k in sorted(rows)]


def get_quant(xx, yy, q):
    cs = np.cumsum(np.array(yy, np.int64)).astype(np.float64) / np.float64(sum(yy))
    return xx[int(np.nonzero(cs >= q)[0][0])]


def _stat(df, denom):
    keys, num = rowsum([s * c for s, c in zip(df["Score"], df["Count"])], df["Cycle"])
    _, den = rowsum(df["Count"], df["Cycle"])
    means = [np.float64(a) / np.float64(b) for a, b in zip(num, den)]
    q = [by(df, df["Cycle"], lambda foo, q=q: get_quant(foo["Score"], foo["Count"], q)) for q in (0.25, 0.5, 0.75)]
    cums = by(df, df["Cycle"], lambda foo: sum(foo["Count"]))
    return {"Cycle": keys, "Mean": means, "Q25": q[0], "Q50": q[1], "Q75": q[2],
            "Cum": [10.0 * np.float64(c) / np.float64(denom) for c in cums]}


def aggregate_count(plotdf):
    """aggregate(Count ~ Cycle + Score, plotdf, sum): one row per (Cycle, Score), ordered by Score, then Cycle."""
    acc = {}
    for c, s, k in zip(plotdf["Cycle"], plotdf["Score"], plotdf["Count"]):
        acc[(s, c)] = acc.get((s, c), 0) + k
    keys = sorted(acc)
    return {"Cycle": [k[1] for k in keys], "Score": [k[0] for k in keys], "Count": [acc[k] for k in keys]}


def plot_quality_profile(fl, n=500000, aggregate=False, seed=None):
    """The frames of plotQualityProfile as lists; plus counts (per file tallies) and nreads."""
    if isinstance(fl, str):
        fl = [fl]
    fl = [f for f in fl if f is not None]
    rng = np.random.default_rng(seed)
    statdf = {k: [] for k in ("Cycle", "Mean", "Q25", "Q50", "Q75", "Cum", "file")}
    anndf = {k: [] for k in ("minScore", "label", "rclabel", "rc", "file")}
    plotdf = {k: [] for k in ("Cycle", "Score", "Count", "file")}
    counts_all, nreads = [], []
    for f in fl:
        _, quals = read_fastq(f)
        nreads.append(len(quals))
        idx = select(len(quals), n, rng)
        counts = tally([quals[i] for i in idx])
        counts_all.append(counts)
        df = per_cycle_quality(counts)
        rc = len(idx)
        if n is not None and rc >= n:
            rclabel = paste("Reads >= ", as_character(n))
        else:
            rclabel = paste("Reads: ", rc)
        st = _stat(df, rc if n is None else min(rc, n))
        for c in ("Cycle", "Score", "Count"):
            plotdf[c] += df[c]
        plotdf["file"] += [os.path.basename(f)] * len(df["Cycle"])
        for c in st:
            statdf[c] += st[c]
        statdf["file"] += [os.path.basename(f)] * len(st["Cycle"])
        anndf["minScore"].append(float(min(df["Score"])) if df["Score"] else float("inf"))
        anndf["label"].append(os.path.basename(f)); anndf["rclabel"].append(rclabel); anndf["rc"].append(rc)
        anndf["file"].append(os.path.basename(f))
    anndf["minScore"] = [min(anndf["minScore"])] * len(anndf["minScore"])
    if aggregate:
        plotdf = aggregate_count(plotdf)
        plotdf["label"] = [paste(len(anndf["rc"]), "files (aggregated)")] * len(plotdf["Cycle"])
        denom = sum(rc if n is None else min(rc, n) for rc in anndf["rc"])     # sum(pmin(anndf$rc, n))
        statdf = _stat(plotdf, denom)
    return {"plotdf": plotdf, "statdf": statdf, "anndf": anndf, "nreads": nreads, "counts": counts_all}


def plot_complexity(fl, kmerSize=2, n=100000, aggregate=False, seed=None):
    if isinstance(fl, str):
        fl = [fl]
    fl = [f for f in fl if f is not None]
    rng = np.random.default_rng(seed)
    vals, files = [], []
    for f in fl:
        seqs, _ = read_fastq(f)
        idx = select(len(seqs), n, rng)
        vals += [filter_ref.complexity(seqs[i], kmerSize) for i in idx]
        files += [os.path.basename(f)] * len(idx)
    if aggregate:
        files = [paste(len(fl), "files (aggregated)")] * len(files)
    return {"complexity": vals, "file": files}
