"""nwalign's throughput on the GPU: --pairs random pairs (one a shifted copy of the other with a few substitutions) at
each length of --lengths, ends-free and global, after one warm-up call, --reps times.  Prints one JSON line with pairs
per second for the whole call (rows copied back to the host) and the alignment kernel's cells per second.
Run:  python tools/nwalign_leg.py [--pairs 20000] [--lengths 250,1500] [--reps 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.collapse_leg import gpu_info    # noqa: E402


def pairs(n, L, rng):
    A, B = [], []
    for _ in range(n):
        a = "".join("ACGT"[i] for i in rng.integers(0, 4, L))
        b = list(a[int(rng.integers(0, 5)):] + "".join("ACGT"[i] for i in rng.integers(0, 4, int(rng.integers(0, 5)))))
        for p in rng.choice(len(b), 3, replace=False):
            b[p] = "ACGT"[("ACGT".index(b[p]) + 1) % 4]
        A.append(a); B.append("".join(b))
    return A, B


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=20000)
    ap.add_argument("--lengths", default="250,1500")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from dada2_b200 import align
    rng = np.random.default_rng(1)
    res = {"gpu": gpu_info(), "runs": []}
    for L in (int(x) for x in a.lengths.split(",")):
        A, B = pairs(a.pairs, L, rng)
        for endsfree in (True, False):
            align.align_pairs(A[:1000], B[:1000], endsfree=endsfree)
            ms, st = [], None
            for _ in range(a.reps):
                t0 = time.perf_counter()
                r = align.align_pairs(A, B, endsfree=endsfree, return_stats=True)
                ms.append((time.perf_counter() - t0) * 1e3)
                st = r["stats"]
            res["runs"].append({"len": L, "endsfree": endsfree, "pairs": len(A), "call_ms": [round(x, 1) for x in ms],
                                "pairs_per_s": round(len(A) / (min(ms) / 1e3)), "ms_k_align": round(st["ms_k_align"], 2),
                                "ms_device": round(st["ms_device"], 2), "kernel_gcups": round(st["n_cells"] / 1e6 / st["ms_k_align"], 2),
                                "n_blocks": st["n_blocks"]})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
