"""De novo bimera detection (removeBimeraDenovo's "per-sample" and "pooled" methods) through the C-ABI
dada2b_denovo_bimera on two synthetic tables (tools/synth.py bimera_table, 250 nt): 2000 sequences x 16 samples per
sample (zero-count cells are not queries), and the column sums of a 10^4-sequence table pooled (every sequence a query).
The timed call includes packing, H2D, the need / align / flag kernels and D2H (median of 3 after a warm-up); the kernel and
alignment milliseconds and pair counts come from dada2b_bimera_stats.  The reference is R's loop restated over the
compiled C_is_bimera (tests/removebim_ref.py; oracle/_ref, or the CPU restatement when it is absent) on all host cores:
every row of the per-sample table, and every 10th query of the pooled one (its flags are diffed on those queries).
Also printed: what the parent-list path that isBimeraDenovo used before would have built on the host for the same
inputs (one list per query with two or more parents; int32 indices, int64 offsets, and the C-ABI's two uint32 job
vectors), with its Python loop timed on a sample of queries and scaled.  The card's name, power limit and max SM clock
are read in the same run.  Prints one line `REMOVEBIMLEG {json}`.  Run:  python tools/removebim_leg.py"""
import json
import multiprocessing
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _ref_rows(args):
    from tests import removebim_ref as R
    seqs, ab, queries = args
    return R.is_bimera_denovo(seqs, ab, queries)


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def old_parent_lists(ab_rows, fold=2.0, mpa=8.0, sample=200, seed=0):
    """Size of the host parent lists the previous isBimeraDenovo built (one call per row), and its loop's time scaled
    from a sample of queries."""
    npairs, nq, t, ns = 0, 0, 0.0, 0
    rng = np.random.default_rng(seed)
    for ab in ab_rows:
        ab = np.asarray(ab, np.int64)
        s = np.sort(ab)
        thr = np.maximum(fold * ab, mpa)
        cnt = len(ab) - np.searchsorted(s, thr, side="right")              # #{k : ab[k] > fold * ab[i] and ab[k] > mpa}
        npairs += int(cnt[cnt >= 2].sum()); nq += int((cnt >= 2).sum())
        idx = rng.choice(len(ab), min(sample, len(ab)), replace=False)
        t0 = time.perf_counter()
        for i in idx:
            pars = np.nonzero((ab > fold * ab[i]) & (ab > mpa))[0]
            if len(pars) >= 2:
                pars.astype(np.int32)
        t += (time.perf_counter() - t0) * len(ab) / len(idx); ns += len(ab)
    host_bytes = 4 * npairs + 8 * (nq + len(ab_rows)) + 8 * npairs
    return {"queries": nq, "parent_indices": npairs, "host_bytes": host_bytes, "h2d_bytes": 8 * npairs + 12 * nq,
            "python_loop_s_est": round(t, 3)}


def run_case(tag, mat, seqs, zero_queries, ref_queries):
    from dada2_b200 import bimera
    bimera.denovo_bimera(mat, seqs, zero_queries=zero_queries)                  # warm-up (context, module load)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        flags, st = bimera.denovo_bimera(mat, seqs, zero_queries=zero_queries, return_stats=True)
        ts.append((time.perf_counter() - t0) * 1e3)
    out = {"shape": list(mat.shape), "e2e_ms": round(float(np.median(ts)), 2), "device_ms": round(st["ms_device"], 2),
           "k_align_ms": round(st["ms_k_align"], 2), "pairs": int(st["n_pairs"]), "cells": int(st["n_cells"]),
           "gpu_launches": int(st["gpu_launches"]), "h2d_bytes": int(st["h2d_bytes"]), "d2h_bytes": int(st["d2h_bytes"]),
           "flagged": int(flags.sum())}
    jobs = [(seqs, row, q) for row, q in zip(*ref_queries)]
    t0 = time.perf_counter()
    with ProcessPoolExecutor(max_workers=os.cpu_count(), mp_context=multiprocessing.get_context("spawn")) as ex:   # no fork of a CUDA process
        parts = list(ex.map(_ref_rows, jobs))
    dt = time.perf_counter() - t0
    want = np.array(parts)
    asked = np.array([q for q in ref_queries[1]])
    if len(parts) != mat.shape[0]:                                               # query chunks of one row
        want, asked = np.logical_or.reduce(want)[None, :], np.logical_or.reduce(asked)[None, :]
    out["cpu_reference"] = {"cores": os.cpu_count(), "s": round(dt, 3), "queries": int(asked.sum()),
                            "flags_identical": bool(np.array_equal(flags & asked, want & asked))}
    out["old_parent_lists"] = old_parent_lists(mat)
    print(tag, out, file=sys.stderr, flush=True)
    return out


def main():
    from oracle import ref
    from tools import synth
    info = _gpu_info()
    res = {"gpu": info, "reference": "compiled C_is_bimera" if ref.available() else "CPU restatement"}
    seqs, mat = synth.bimera_table(2000, 16, seed=21)
    res["per_sample_2000x16"] = run_case("per-sample", mat, seqs, False, (list(mat), [row > 0 for row in mat]))
    seqs, mat = synth.bimera_table(10000, 16, seed=22)
    cs = mat.sum(axis=0, dtype=np.int64)[None, :]
    n = cs.shape[1]
    chunks = [(np.arange(n) % 10 == 0) & (np.arange(n) % 80 == 10 * c) for c in range(8)]
    res["pooled_10000"] = run_case("pooled", cs, seqs, True, ([cs[0]] * len(chunks), chunks))
    res["gpu_after"] = _gpu_info()
    print("REMOVEBIMLEG " + json.dumps(res))


if __name__ == "__main__":
    main()
