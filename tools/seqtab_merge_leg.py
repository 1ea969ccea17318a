"""mergeSequenceTables on the GPU at study scale: where the time of one call goes.  Builds the seeded 12-run merge of
tests/test_gpu_zz_seqtab_merge.py (12 runs x 96 samples over a pool of 2e5 ASVs, 20 000 columns per run, a quarter of
each run's sample names shared with the previous run, every third run in reverse orientation), then for tryRC off and
on: dada2b_merge_seqtabs after a warm-up over --reps calls (wall time, and the H2D / kernel / D2H CUDA-event times from
its stats), the whole mergeSequenceTables call, and the Python restatement of the R function at the same size.  The
card's name and power limit are read in the same call.  Prints one JSON line.
Run:  python tools/seqtab_merge_leg.py [--reps 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.collapse_leg import gpu_info   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import dada2_b200
    from dada2_b200 import seqtab
    from tests import seqtab_merge_cases as G
    from tests import seqtab_merge_ref as R
    runs = G.make_runs(7, nruns=12, nsamp=96, pool=200000, per_run=20000, shared_frac=0.25)
    res = {"gpu": gpu_info(), "ntables": len(runs), "input_columns": sum(len(r[1]) for r in runs),
           "input_cells": int(sum(r[0].size for r in runs)), "arms": {}}
    tables, rownames, row_out = seqtab._merge_inputs(None, None, (), runs, "sum")
    mats = [seqtab._int32_entries(t[0]) for t in tables]
    cols = [list(t[1]) for t in tables]
    ro = np.concatenate(row_out)
    for try_rc in (False, True):
        seqtab.merge_columns(mats, cols, ro, len(rownames), try_rc, 1)                 # warm-up
        rows = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            mat, src, st = seqtab.merge_columns(mats, cols, ro, len(rownames), try_rc, 1)
            wall = (time.perf_counter() - t0) * 1e3
            rows.append({"call_ms": round(wall, 1), **{k: (round(v, 3) if isinstance(v, float) else int(v)) for k, v in st.items()}})
            print("tryRC=%s" % try_rc, rows[-1], flush=True)
        t0 = time.perf_counter()
        got = dada2_b200.mergeSequenceTables(tables=runs, repeats="sum", tryRC=try_rc)
        whole = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        want = R.merge(runs, repeats="sum", tryRC=try_rc)
        ref = (time.perf_counter() - t0) * 1e3
        same = bool(np.array_equal(got[0], want[0]) and got[1] == want[1] and got[2] == want[2])
        res["arms"]["tryRC" if try_rc else "plain"] = {
            "nrow_out": int(mat.shape[0]), "ncol_out": int(mat.shape[1]), "n_rc": int(st["n_rc"]), "native": rows,
            "mergeSequenceTables_ms": round(whole, 1), "restatement_ms": round(ref, 1), "equal_to_restatement": same}
        print("tryRC=%s whole %.1f ms, restatement %.1f ms, equal %s" % (try_rc, whole, ref, same), flush=True)
        del got, want
    print(json.dumps(res))


if __name__ == "__main__":
    main()
