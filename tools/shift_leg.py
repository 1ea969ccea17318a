"""isShiftDenovo on the GPU against the reference's loop on the host, on the seeded ~19 000 ASV table of
tests/collapse_cases.large_table() with column sums as abundances.  Prints one JSON line.

GPU: the whole library call (screen, direction, filter, alignments), after one warm-up call, --reps times, with the
screened / candidate / filtered / aligned counts, DP cells and the alignment kernel's cells per second.
Reference: R/chimeras.R:384-400 restated in Python (tests/shift_ref.py) over the reference's compiled nwalign_endsfree, on
the --ref-n most abundant sequences (cut at an abundance boundary, so the subset is closed under "more abundant"), with
the device's flags on that subset compared.
Run:  python tools/shift_leg.py [--reps 3] [--ref-n 300]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import collapse_cases as G      # noqa: E402
from tests import shift_ref as S           # noqa: E402
from tools.collapse_leg import gpu_info    # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-n", type=int, default=300)
    a = ap.parse_args()
    from dada2_b200 import bimera
    mat, seqs = G.large_table()
    ab = mat.sum(axis=0, dtype=np.int64)
    res = {"gpu": gpu_info(), "nproc": os.cpu_count(), "nseq": len(seqs)}
    bimera.shift_flags(seqs, ab)
    runs = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        flag, st = bimera.shift_flags(seqs, ab, return_stats=True)
        runs.append((time.perf_counter() - t0) * 1e3)
    res.update({"gpu_call_ms": [round(x, 2) for x in runs], "stats": st, "n_flagged": int(flag.sum()),
                "align_gcups": st["n_cells"] / 1e6 / max(st["ms_k_align"], 1e-9)})
    from oracle import ref
    if ref.available():
        o = np.argsort(-ab, kind="stable")
        k = a.ref_n
        while k < len(o) and ab[o[k - 1]] == ab[o[k]]:
            k += 1
        top = {seqs[i]: int(ab[i]) for i in o[:k]}
        t0 = time.perf_counter()
        f = S.is_shift_denovo(top, minOverlap=20)
        t_ref = time.perf_counter() - t0
        sub = [seqs[i] for i in o[:k]]
        t0 = time.perf_counter()
        fg = bimera.shift_flags(sub, ab[o[:k]])
        t_gpu = time.perf_counter() - t0
        res["ref_subset"] = {"n": k, "pairs_aligned": sum(int(np.count_nonzero(ab[o[:k]] > ab[i])) for i in o[:k]),
                             "ref_loop_s": round(t_ref, 3), "gpu_call_ms": round(t_gpu * 1e3, 2),
                             "same_flags": [f[s] for s in sub] == fg.astype(bool).tolist(),
                             "same_as_full_run": [f[s] for s in sub] == flag[o[:k]].astype(bool).tolist()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
