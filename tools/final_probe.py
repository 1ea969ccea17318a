"""Where the time of a dada() pass's final pass goes: resident passes of the bench workload (1e6 synthetic 250 nt uniques, seed
12345, tperr1, default options) with DADA2B_VERBOSE set.  Per timed pass it prints the final pass's kernel split (the row sweep,
the diagonal-list tally, the gapped list), the loop's exact NW pass, round 0's host time and the host phases of the finish; then
the medians.  The card's name, power limit and largest SM clock are printed first: they belong to every number below.
  python tools/final_probe.py [n_uniques] [passes]"""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["DADA2B_VERBOSE"] = "1"

import numpy as np

import dada2_b200
from tests import cases
from tools import synth

KEYS = ["ms_final", "ms_k_align_final", "ms_k_final_row", "ms_k_final_diag", "ms_k_final_gapped", "ms_k_nw_exact", "ms_k_nw_bound",
        "ms_loop", "ms_total"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "unknown (%s)" % e


def run_captured(res, err):
    """One pass with the library's stderr (fd 2) captured: (stats, verbose lines)."""
    sys.stderr.flush()
    with tempfile.TemporaryFile(mode="w+b") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            out = res.run(err)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        txt = f.read().decode(errors="replace")
    return out["stats"], txt


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
    passes = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    print("card: %s" % card(), flush=True)
    seqs, ab, q, _ = synth.illumina(n, seed=12345)
    err = cases.tperr1()
    res = dada2_b200.Resident(seqs, ab, None, q)
    for _ in range(2):
        run_captured(res, err)
    rows = []
    for k in range(passes):
        st, txt = run_captured(res, err)
        r0 = re.search(r"round 0 done: ([0-9.]+) ms", txt)
        st["round0_host_ms"] = float(r0.group(1)) if r0 else float("nan")
        rows.append(st)
        print("pass %d: %s | launches row %d diag %d gapped %d | round 0 %.2f ms" % (
            k, " ".join("%s %.2f" % (x, st[x]) for x in KEYS), st["n_k_final_row"], st["n_k_final_diag"], st["n_k_final_gapped"],
            st["round0_host_ms"]), flush=True)
        for line in txt.splitlines():
            if "final pass lists" in line or "finish host ms" in line or "loop NW:" in line:
                print("    " + line, flush=True)
    print("median over %d passes: %s" % (passes, " ".join("%s %.2f" % (x, float(np.median([r[x] for r in rows])))
                                                       for x in KEYS + ["round0_host_ms"])), flush=True)


if __name__ == "__main__":
    main()
