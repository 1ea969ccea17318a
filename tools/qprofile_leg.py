"""plotQualityProfile on the GPU at run scale: where the time of one call goes.  Writes three synthetic fastq.gz files
(5e5 x 250-nt reads with uniform scores 2..41, the same with NovaSeq's binned 2/12/23/37, and 5e4 PacBio-like reads of
1000-2500 nt with scores 0..93), then per file: the host fastq parse time, the device tally's H2D / kernel / D2H CUDA-event
times, the kernels' compulsory bytes over their time against 3.35 TB/s (the H100 SXM's HBM3 peak), and the whole
plotQualityProfile call.  Also plotQualityProfile(aggregate=True) over 8 copies of the first file, end to end.  The card's
name and power limit are read in the same call.  Prints one JSON line.
Run:  python tools/qprofile_leg.py [--reps 3]"""
import argparse
import gzip
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.collapse_leg import gpu_info   # noqa: E402

PEAK = 3.35e12


def write(path, lens, qual_fn, rng):
    from dada2_b200 import filter as fl
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(off[-1]))].tobytes()
    reads = fl.Reads(seq, off, qual_fn(int(off[-1])))
    with open(path, "wb") as raw, gzip.GzipFile(filename="", mode="wb", fileobj=raw, mtime=0, compresslevel=6) as f:
        f.write(fl.fastq_bytes([b"r%d" % i for i in range(len(lens))], reads))
    return path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import dada2_b200
    from dada2_b200 import filter as fl, qc
    rng = np.random.default_rng(1)
    lut = np.array([2] * 2 + [12] * 5 + [23] * 13 + [37] * 80, np.uint8)
    res = {"gpu": gpu_info(), "files": {}}
    with tempfile.TemporaryDirectory() as d:
        files = {
            "illumina_5e5x250_q2-41": write(os.path.join(d, "full.fastq.gz"), np.full(500000, 250),
                                            lambda k: rng.integers(2, 42, k, dtype=np.uint8), rng),
            "novaseq_binned_5e5x250": write(os.path.join(d, "binned.fastq.gz"), np.full(500000, 250),
                                            lambda k: lut[rng.integers(0, 100, k)], rng),
            "pacbio_5e4x1000-2500_q0-93": write(os.path.join(d, "pb.fastq.gz"), rng.integers(1000, 2501, 50000),
                                                lambda k: rng.integers(0, 94, k, dtype=np.uint8), rng),
        }
        dada2_b200.plotQualityProfile(files["pacbio_5e4x1000-2500_q0-93"], n=1000, seed=0)      # warm-up
        for name, path in files.items():
            rows = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                _, reads = fl.read_fastq_records(path)
                parse = (time.perf_counter() - t0) * 1e3
                t0 = time.perf_counter()
                counts, st = qc.quality_tally(reads.off, reads.qual)
                call = (time.perf_counter() - t0) * 1e3
                t0 = time.perf_counter()
                dada2_b200.plotQualityProfile(path, n=None)
                whole = (time.perf_counter() - t0) * 1e3
                rows.append({"parse_ms": round(parse, 1), "tally_call_ms": round(call, 2), "ms_h2d": round(st["ms_h2d"], 3),
                             "ms_kernels": round(st["ms_kernels"], 3), "ms_d2h": round(st["ms_d2h"], 3),
                             "ms_total": round(st["ms_total"], 2), "h2d_bytes": st["h2d_bytes"], "kernel_bytes": st["kernel_bytes"],
                             "kernel_GBps": round(st["kernel_bytes"] / st["ms_kernels"] / 1e6, 1),
                             "kernel_fraction_of_peak": round(st["kernel_bytes"] / PEAK * 1e3 / st["ms_kernels"], 3),
                             "plotQualityProfile_all_reads_ms": round(whole, 1)})
            res["files"][name] = {"nreads": int(st["nreads"]), "nbases": int(st["nbases"]), "runs": rows}
            print(name, rows[-1], flush=True)
        agg = [os.path.join(d, "agg%d.fastq.gz" % k) for k in range(8)]
        for p in agg:
            shutil.copy(files["illumina_5e5x250_q2-41"], p)
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            dada2_b200.plotQualityProfile(agg, aggregate=True)
            times.append(round((time.perf_counter() - t0) * 1e3, 1))
        res["aggregate_8_files_ms"] = times
    print(json.dumps(res))


if __name__ == "__main__":
    main()
