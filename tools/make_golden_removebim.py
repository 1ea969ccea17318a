"""Generates tests/golden/removebim.npz from the REFERENCE's own chimera.cpp (oracle/_ref, compiled unmodified; build
container only), through the R loops restated in tests/removebim_ref.py: for each table, the per-sample flag matrix of
removeBimeraDenovo(method = "per-sample") (every cell evaluated, zero counts included) and the pooled flags (isBimeraDenovo
on the column sums), under an option grid of isBimeraDenovo's arguments.  Tables: those of bimera.npz, plus "s_edge" (an
all-zero column, zero cells, a query with exactly one parent in one sample) and "s_dup" (duplicated column names).
Run:  python tools/make_golden_removebim.py"""
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OPTS = [dict(), dict(allowOneOff=True), dict(allowOneOff=True, minOneOffParentDistance=2),
        dict(minFoldParentOverAbundance=1.0, minParentAbundance=1), dict(minFoldParentOverAbundance=0.5),
        dict(minParentAbundance=2.5), dict(maxShift=4)]


def edge_table():
    from tools import synth
    seqs, mat = synth.bimera_table(24, 4, seed=5, L=80)
    mat = mat.copy()
    mat[:, 5] = 0                                          # all-zero column
    j, p = 17, 2                                           # sample 3: query j has exactly one parent (p) under the defaults
    mat[3] = np.minimum(mat[3], 8)
    mat[3, j], mat[3, p] = 4, 40
    return seqs, mat


def dup_table():
    from tools import synth
    seqs, mat = synth.bimera_table(16, 3, seed=6, L=80)
    rng = np.random.default_rng(6)
    extra = rng.integers(0, 30, (mat.shape[0], 2)).astype(np.int32)
    return seqs + [seqs[2], seqs[9]], np.concatenate([mat, extra], axis=1)


def tables():
    z = np.load(os.path.join(ROOT, "tests", "golden", "bimera.npz"), allow_pickle=False)
    meta = json.loads(str(z["meta"]))
    out = {n: (z[n + "_seqs"].tolist(), z[n + "_mat"]) for n in meta["tables"]}
    out["s_edge"] = edge_table()
    out["s_dup"] = dup_table()
    return out


def _job(args):
    name, oi, seqs, mat = args
    from tests import removebim_ref as R
    o = OPTS[oi]
    return name, oi, R.per_sample_flags(mat, seqs, "ref", **o), R.pooled_flags(mat, seqs, "ref", **o)


def main():
    from oracle import ref
    from tests import removebim_ref as R
    assert ref.available(), "needs the compiled reference (oracle/_ref/libdada2ref.so)"
    T = tables()
    seqs, mat = T["s_edge"]
    row = mat[3]
    npar = int(((row > 2 * row[17]) & (row > 8)).sum())
    assert npar == 1 and not (mat[:, 5] > 0).any(), "s_edge lost its corner cases"
    assert not R.per_sample_flags(mat[3:4], seqs, "ref")[0, 17]
    out = {}
    for name, (sq, m) in T.items():
        out[name + "_seqs"] = np.array(sq)
        out[name + "_mat"] = np.asarray(m, np.int32)
    jobs = [(name, oi, sq, m) for name, (sq, m) in T.items() for oi in range(len(OPTS))]
    with ProcessPoolExecutor(max_workers=os.cpu_count()) as ex:
        for name, oi, ps, po in ex.map(_job, jobs):
            out["%s_o%d_persample" % (name, oi)] = ps.astype(np.uint8)
            out["%s_o%d_pooled" % (name, oi)] = po.astype(np.uint8)
            print(name, oi, "per-sample flagged", int(ps.sum()), "of which nonzero", int((ps & (T[name][1] > 0)).sum()), "pooled", int(po.sum()),
                  flush=True)
    out["meta"] = np.array(json.dumps({"opts": OPTS, "tables": list(T)}))
    path = os.path.join(ROOT, "tests", "golden", "removebim.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
