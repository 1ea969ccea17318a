"""The read filter on the GPU at run scale: 10^7 synthetic 250-nt single-end reads and 10^7 pairs (tests/filter_cases.py's
generator: low-quality tails, N / IUPAC codes, spliced phiX fragments, low-complexity reads), with the vignette's options
(trimLeft=10, truncLen=240 / 200, maxN=0, maxEE=2) plus rm_phix.  Prints one JSON line with, per run: the kernels' CUDA-event
time, H2D / D2H bytes and times, the kernels' compulsory bytes over 3.35 TB/s (the H100 SXM's HBM3 peak), and the host
fastq parse / write time of the same reads (measured on --io-n reads, scaled by the read count and labelled so).
The card's name and power limit are read in the same call.
Run:  python tools/filter_leg.py [--n 10000000] [--reps 2] [--io-n 1000000]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import filter_cases as G       # noqa: E402
from tools.collapse_leg import gpu_info   # noqa: E402

PEAK = 3.35e12


def tile(r, n):
    """n reads: the block r repeated (the generator's cost would otherwise dominate the leg)."""
    from dada2_b200.filter import Reads
    k = -(-n // len(r))
    L = int(r.off[1] - r.off[0])
    return Reads((r.seq * k)[:n * L], np.arange(n + 1, dtype=np.int64) * L, np.tile(r.qual, k)[:n * L])


def run(fl, opts, fwd, rev, reps):
    fl._run(fwd, rev, opts, 0)                                   # warm-up
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fl._run(fwd, rev, opts, 0)
        wall = (time.perf_counter() - t0) * 1e3
        st = r["stats"]
        out.append({"wall_ms": round(wall, 1), "ms_kernels": round(st["ms_kernels"], 2), "ms_h2d": round(st["ms_h2d"], 2),
                    "ms_d2h": round(st["ms_d2h"], 2), "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                    "kernel_bytes": st["kernel_bytes"], "kernel_bytes_at_peak_ms": round(st["kernel_bytes"] / PEAK * 1e3, 2),
                    "kernel_fraction_of_peak": round(st["kernel_bytes"] / PEAK * 1e3 / max(st["ms_kernels"], 1e-9), 3),
                    "nout": len(r["src"]), "launches": st["gpu_launches"]})
    return out


def host_io(fl, reads, n_total):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "r.fastq")
        ids = [b"r%d" % i for i in range(len(reads))]
        t0 = time.perf_counter()
        data = fl.fastq_bytes(ids, reads)
        with open(p, "wb") as f:
            f.write(data)
        tw = time.perf_counter() - t0
        t0 = time.perf_counter()
        fl.read_fastq_records(p)
        tp = time.perf_counter() - t0
    scale = n_total / len(reads)
    return {"measured_reads": len(reads), "parse_s": round(tp, 2), "write_s": round(tw, 2),
            "scaled_parse_s": round(tp * scale, 1), "scaled_write_s": round(tw * scale, 1),
            "note": "uncompressed fastq, one host thread; scaled values are extrapolated by read count, not measured"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--io-n", type=int, default=1000000)
    a = ap.parse_args()
    from dada2_b200 import filter as fl
    res = {"gpu": gpu_info(), "n": a.n}
    blk = [G.synthetic_reads(min(a.n, 1000000), 250, seed=s) for s in (1, 2)]
    fwd, rev = tile(blk[0], a.n), tile(blk[1], a.n)
    kw = dict(trimLeft=10, maxN=0, maxEE=2, rm_phix=True, rm_lowcomplex=0, phix=G.PHIX_FA, n=100000)
    o1 = fl._opts(False, truncLen=240, truncQ=2, trimRight=0, maxLen=float("inf"), minLen=20, minQ=0, orient_fwd=None, **kw)
    o2 = fl._opts(True, truncLen=(240, 200), truncQ=2, trimRight=0, maxLen=float("inf"), minLen=20, minQ=0, orient_fwd=None, **kw)
    res["single"] = run(fl, o1, fwd, None, a.reps)
    res["paired"] = run(fl, o2, fwd, rev, a.reps)
    res["host_io_single"] = host_io(fl, tile(blk[0], min(a.io_n, a.n)), a.n)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
