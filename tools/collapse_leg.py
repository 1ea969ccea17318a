"""collapseNoMismatch on the GPU against the reference's C++ on the host, on the seeded ~20 000 ASV x 96 sample table of
tests/test_gpu_zz_collapse.py.  Prints one JSON line.

GPU: the whole library call (screen, filter, alignments, greedy resolution), after one warm-up call, --reps times; plus
the candidate / filtered / aligned counts, DP cells and the alignment kernel's GCUPS.
Reference: the R loop of R/multiSample.R:125-144 restated in Python (tests/collapse_ref.py) over the reference's compiled
nwhamming, on the first --ref-n query-ordered sequences only; the time of the native calls and of the whole loop are
reported for that subset and extrapolated to the full table by the ratio of candidate pairs (labelled as such).
Run:  python tools/collapse_leg.py [--reps 3] [--ref-n 1500]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import collapse_cases as G      # noqa: E402
from tests import collapse_ref as R        # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-n", type=int, default=1500)
    a = ap.parse_args()
    from dada2_b200 import seqtab
    mat, cols = G.large_table()
    seqs = R.query_order(mat, cols)
    res = {"gpu": gpu_info(), "nproc": os.cpu_count(), "nseq": len(seqs), "nsamples": int(mat.shape[0])}
    seqtab.collapse_reps(seqs)
    runs = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        rep, st = seqtab.collapse_reps(seqs, return_stats=True)
        runs.append((time.perf_counter() - t0) * 1e3)
    res.update({"gpu_call_ms": [round(x, 2) for x in runs], "stats": st, "n_out": int(np.count_nonzero(rep == np.arange(len(rep)))),
                "align_gcups": st["n_cells"] / 1e6 / max(st["ms_k_align"], 1e-9)})
    from oracle import ref
    if ref.available():
        sub = seqs[:a.ref_n]
        tn = [0.0]

        def timed(*x, **k):
            t = time.perf_counter()
            h = R.ref_nwhamming(*x, **k)
            tn[0] += time.perf_counter() - t
            return h
        t0 = time.perf_counter()
        R.collapse(np.ones((1, len(sub)), np.int32) * np.arange(len(sub), 0, -1), sub, nwhamming=timed)
        loop_s = time.perf_counter() - t0
        nsub = len(G.screen_pairs(sub, 20)[0])
        scale = res["stats"]["n_candidates"] / max(nsub, 1)
        res["reference"] = {"subset_nseq": len(sub), "subset_candidates": nsub, "subset_loop_s": round(loop_s, 2),
                            "subset_native_s": round(tn[0], 2),
                            "extrapolated_full_native_s": round(tn[0] * scale, 1), "extrapolated_full_loop_s": round(loop_s * scale, 1),
                            "note": "host, one thread; full-table values are extrapolated by the candidate-pair ratio, not measured"}
    else:
        res["reference"] = "not measured (reference library not built)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
