"""Primer removal on the GPU at run scale: 10^6 synthetic CCS-like reads of 1400-1600 nt (tests/primer_cases.py's
generator: F27 / rc(R1492) with 0-3 mismatches, some cut at an end, some doubled, half reverse-complemented; a block of
--block reads tiled to --n), removePrimers' defaults.  Prints one JSON line with, per repetition: the kernels' CUDA-event
time and bases/s, H2D / D2H bytes and times, the kernels' compulsory bytes over 3.35 TB/s (the H100 SXM's HBM3 peak)
and which bound applies; the host fastq parse / write of the same reads (measured on --io-n reads, scaled by the read
count and labelled so); and, for scale only, the time of the Python restatement (tests/primer_ref.py) on 10^4 reads --
it is not the reference, whose matcher (Biostrings) is not available.  The card's name and power limit are read in the
same call.
Run:  python tools/primer_leg.py [--n 1000000] [--reps 3] [--io-n 100000]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import primer_cases as G       # noqa: E402
from tests import primer_ref as R         # noqa: E402
from tools.collapse_leg import gpu_info   # noqa: E402

PEAK = 3.35e12


def tile(r, n):
    """n reads: the block r repeated."""
    from dada2_b200.filter import Reads
    k = -(-n // len(r))
    lens = np.tile(np.diff(r.off), k)[:n]
    off = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return Reads((r.seq * k)[:off[-1]], off, np.tile(r.qual, k)[:off[-1]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--block", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--io-n", type=int, default=100000)
    a = ap.parse_args()
    from dada2_b200 import filter as fl, primer as pm
    res = {"gpu": gpu_info(), "n": a.n}
    blk, _ = G.synthetic_ccs(min(a.block, a.n), seed=11)
    rd = tile(blk, a.n)
    bases = int(rd.off[-1])
    res["bases"] = bases
    o = pm._opts(G.F27, R.rc(G.R1492), 2, False, True, True, True)
    pm._run(rd, o, 0)                                             # warm-up
    runs = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        r = pm._run(rd, o, 0)
        wall = (time.perf_counter() - t0) * 1e3
        st = r["stats"]
        at_peak = st["kernel_bytes"] / PEAK * 1e3
        runs.append({"wall_ms": round(wall, 1), "ms_kernels": round(st["ms_kernels"], 2), "ms_h2d": round(st["ms_h2d"], 2),
                     "ms_d2h": round(st["ms_d2h"], 2), "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                     "kernel_bases_per_s": round(bases / (st["ms_kernels"] / 1e3), 1), "kernel_bytes": st["kernel_bytes"],
                     "kernel_bytes_at_peak_ms": round(at_peak, 3), "kernel_fraction_of_peak": round(at_peak / max(st["ms_kernels"], 1e-9), 3),
                     "bound": "memory (compulsory bytes / 3.35 TB/s) -- no FLOP term: the kernels do integer work",
                     "nout": len(r["src"]), "launches": st["gpu_launches"]})
    res["runs"] = runs
    n_io = min(a.io_n, a.n)
    sub = tile(blk, n_io)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "r.fastq")
        ids = [b"r%d" % i for i in range(n_io)]
        t0 = time.perf_counter()
        with open(p, "wb") as f:
            f.write(fl.fastq_bytes(ids, sub))
        tw = time.perf_counter() - t0
        t0 = time.perf_counter()
        fl.read_fastq_records(p)
        tp = time.perf_counter() - t0
    scale = a.n / n_io
    res["host_io"] = {"measured_reads": n_io, "parse_s": round(tp, 2), "write_s": round(tw, 2), "scaled_parse_s": round(tp * scale, 1),
                      "scaled_write_s": round(tw * scale, 1),
                      "note": "uncompressed fastq, one host thread; scaled values are extrapolated by read count, not measured"}
    s = blk.strings()[:10000]
    recs = [(s[i], blk.qual[blk.off[i]:blk.off[i + 1]].tolist()) for i in range(len(s))]
    t0 = time.perf_counter()
    R.remove_primers(recs, G.F27, R.rc(G.R1492), 2)
    res["restatement_1e4_s"] = {"s": round(time.perf_counter() - t0, 2), "reads": len(recs),
                                "note": "tests/primer_ref.py (numpy, one thread), for scale only; not the reference"}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
