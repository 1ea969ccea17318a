"""Writes tests/golden/primer.npz: for every case of tests/primer_cases.py, the restated reason codes, flags, skip and
multiple-hit flags, source indices, output reads and the four scans' hit records of tests/primer_ref.py.  Before it
writes anything it checks the vectorised matcher against the per-shift definition on every read of every case.

    python tools/make_golden_primer.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import primer_cases as G  # noqa: E402
from tests import primer_ref as R  # noqa: E402


def main():
    out = {}
    for case in G.cases():
        k = case["name"]
        for s, _ in case["reads"]:
            for p in (case["pf"], case["pr"]):
                if p is not None:
                    for t in (s, R.rc(s)):
                        assert R.match_vec(p, t, case["k"]) == R.match_literal(p, t, case["k"]), (k, p, t)
        w = G.want_from_restatement(case)
        off = np.zeros(len(w["seqs"]) + 1, np.int64)
        np.cumsum([len(x) for x in w["seqs"]], out=off[1:])
        out[k + "/reason"], out[k + "/flags"], out[k + "/src"] = w["reason"], w["flags"], w["src"]
        out[k + "/skipped"], out[k + "/multi"] = np.array(w["skipped"]), np.array(w["multi"])
        out[k + "/off"] = off
        out[k + "/seq"] = np.frombuffer("".join(w["seqs"]).encode(), np.uint8)
        out[k + "/qual"] = np.array([x for y in w["quals"] for x in y], np.uint8)
        out[k + "/hits"] = G.restate_hits(case)
        print(k, len(w["reason"]), "->", len(w["src"]), np.bincount(w["reason"], minlength=5).tolist(), "skipped" if w["skipped"] else "",
              "multi" if w["multi"] else "")
    np.savez_compressed(G.GOLDEN, **out)
    print("wrote", G.GOLDEN)


if __name__ == "__main__":
    main()
