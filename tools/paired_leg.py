"""Timing of mergePairs over S samples x N read pairs (dd_pairs.cu + dd_merge.cu) against the numpy / reference-C++
restatement of R's per-sample loop (tests/paired_ref.py).  Prints the native call's ms_k_tab (tabulation kernels),
ms_k_merge (the one alignment launch), n_aligned (distinct alignments across samples) against the pairings they stand for,
and the restatement's wall time.  Synthetic 2 x 250 nt reads over 253..480 nt amplicons (tests/paired_cases.synth_set).

    python tools/paired_leg.py --samples 50 --reads 200000 [--batch READS] [--reps 3]
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=50)
    ap.add_argument("--reads", type=int, default=200000)
    ap.add_argument("--batch", type=int, default=None, help="DADA2B_PAIRS_BATCH (reads per batch of whole samples)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=3)
    ap.add_argument("--no-host", action="store_true", help="skip the restatement")
    a = ap.parse_args()
    if a.batch:
        os.environ["DADA2B_PAIRS_BATCH"] = str(a.batch)
    import dada2_b200
    from tests import paired_cases as P, paired_ref as R
    sets = P.synth_set(a.samples, a.reads, seed=a.seed, namp=16)
    args = [list(x) for x in zip(*sets)]
    dada2_b200.mergePairs(*args[:4], returnRejects=True)                     # warm-up: context, module load
    for rep in range(a.reps):
        t0 = time.perf_counter()
        _, st = dada2_b200.mergePairs(*args, returnRejects=True, return_stats=True)
        t1 = time.perf_counter()
        print("rep %d: %d samples, %d reads, %d pairings, n_aligned %d, %d batches, %d launches | ms_k_tab %.2f  ms_k_merge %.2f  "
              "native %.1f ms  mergePairs %.1f ms  (H2D %.1f MB, D2H %.1f MB)" % (
                  rep, a.samples, st["n_reads"], st["n_pairings"], st["n_aligned"], st["n_batches"], st["gpu_launches"], st["ms_k_tab"],
                  st["ms_k_merge"], st["ms_total"], 1e3 * (t1 - t0), st["h2d_bytes"] / 1e6, st["d2h_bytes"] / 1e6), flush=True)
    if not a.no_host:
        R._CACHE.clear()
        t0 = time.perf_counter()
        for c in sets:
            R.merge_sample(*c, returnRejects=True)
        print("host restatement (numpy tabulation + one reference alignment per distinct pair): %.1f ms" % (1e3 * (time.perf_counter() - t0)))


if __name__ == "__main__":
    main()
