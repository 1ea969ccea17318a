"""Generates tests/golden/collapse.npz: seeded sequence tables, collapseNoMismatch's output for several option sets, and the
pair-level (screen, nwhamming) of every pair of every table.

The loop is tests/collapse_ref.py's restatement of R/multiSample.R:104-160; nwhamming is the reference's own C++
(oracle/_ref/libdada2ref.so, compiled unmodified; needs the reference sources at build time).
Run:  python tools/make_golden_collapse.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import collapse_ref as R      # noqa: E402

CASES = [("families", {}), ("families", {"minOverlap": 0}), ("families", {"minOverlap": 1}), ("families", {"minOverlap": 33}),
         ("families", {"minOverlap": 64}), ("families", {"orderBy": "nsamples"}), ("families", {"orderBy": None}),
         ("families", {"identicalOnly": True}), ("families", {"vec": False}), ("families", {"band": 0}), ("families", {"band": 16}),
         ("families", {"vec": False, "band": 16}), ("repeats", {}), ("repeats", {"vec": False}), ("repeats", {"band": 16}),
         ("repeats", {"minOverlap": 5}), ("repeats", {"minOverlap": 0, "orderBy": "nsamples"})]


def tables(seed=16):
    rng = np.random.default_rng(seed)

    def rs(n):
        return "".join("ACGT"[i] for i in rng.integers(0, 4, n))

    def snp(s, p):
        return s[:p] + "ACGT"[("ACGT".index(s[p]) + 1 + int(rng.integers(0, 3))) % 4] + s[p + 1:]

    out = {}
    # V4-like families: one conserved 24-nt start shared by all families, then a family backbone
    cons = rs(24)
    seqs = []
    for f in range(3):
        B = cons + rs(int(rng.integers(90, 130)))
        fam = [B, B[3:], B[:-5], B[4:] + rs(4), B[10:-10], snp(B, 60), snp(B, 2), snp(B, len(B) - 2),
               B[:50] + rs(1) + B[50:], B[:70] + B[71:], B + "AAAAAA", B[:-3] + "TTTTTTT", B[5:20], B[30:45]]
        seqs += fam
    seqs += [rs(12), rs(140), cons + rs(30)]
    seqs = list(dict.fromkeys(seqs))
    out["families"] = seqs
    # tandem repeats (alignments with several best paths, some exact, some not) and homopolymer-rich ends
    seqs = []
    for per in ("ACG", "AACGT", "ACGTTGA"):
        u = per * (90 // len(per))
        seqs += [u, u[1:], u[len(per):] + per[:2], snp(u, 40), u[:45] + per + u[45:], u[:30] + u[31:]]
    H = "A" * 9 + rs(80) + "T" * 9
    seqs += [H, "A" * 6 + H[9:], H[:-9] + "T" * 12, "A" * 12 + H[9:-2], "C" + H, H[:40] + "A" + H[40:]]
    seqs = list(dict.fromkeys(seqs))
    out["repeats"] = seqs
    res = {}
    for name, sq in out.items():
        ns = 5
        mat = rng.integers(0, 40, (ns, len(sq))) * (rng.random((ns, len(sq))) < 0.7)
        mat[:, 1] = mat[:, 0]                       # tied column sums
        mat[:, 4] = mat[:, 2]
        mat[:, 7] = mat[:, 3]
        mat[0, :] += 1
        cols = list(sq)
        cols.append(sq[2]); mat = np.concatenate([mat, rng.integers(0, 5, (ns, 1))], axis=1)          # duplicate column
        res[name] = (mat.astype(np.int32), cols, ["s%d" % i for i in range(ns)])
    return res


def main():
    tabs = tables()
    out = {}
    meta = {"cases": [], "tables": {}}
    for name, (mat, cols, rows) in tabs.items():
        out[name + "_mat"], out[name + "_cols"], out[name + "_rows"] = mat, np.array(cols), np.array(rows)
        seqs = R.query_order(mat, cols)
        n = len(seqs)
        pq, pr = np.array([(j, i) for j in range(n) for i in range(j)], np.int32).T
        out[name + "_seqs"], out[name + "_pq"], out[name + "_pr"] = np.array(seqs), pq, pr
        mos = sorted({o.get("minOverlap", 20) for t, o in CASES if t == name})
        alns = sorted({(int(o.get("vec", True)), o.get("band", -1)) for t, o in CASES if t == name})
        for m in mos:
            out["%s_scr_m%d" % (name, m)] = np.array([R.screen(seqs[j], seqs[i], m) for j, i in zip(pq, pr)], np.int32)
        for v, b in alns:
            out["%s_ham_v%d_b%d" % (name, v, b)] = np.array([R.ref_nwhamming(seqs[j], seqs[i], vec=bool(v), band=b) for j, i in zip(pq, pr)],
                                                            np.int32)
        meta["tables"][name] = {"minOverlap": mos, "aligners": alns}
    for k, (name, o) in enumerate(CASES):
        mat, cols, rows = tabs[name]
        m, c = R.collapse(mat, cols, **o)
        out["c%d_mat" % k], out["c%d_cols" % k] = m, np.array(c)
        meta["cases"].append([name, o])
        print(k, name, o, "->", m.shape[1], "of", len(set(cols)), "columns")
    out["meta"] = np.array(json.dumps(meta))
    path = os.path.join(ROOT, "tests", "golden", "collapse.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
