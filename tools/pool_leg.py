"""dada(pool = TRUE) with selfConsist error learning at BASELINE.json configs[2]'s shape: --n pooled 250-nt uniques
(tools/synth.illumina) dealt with overlap to 8 samples (each unique to 1-3 samples, its reads split between them), pooled
on the device into a resident context, then learnErrors' loop (initializeErr, loessErrfun) on that context and the
expansion into per-sample objects.  Prints one JSON line: the card's name and power limit, the host combineDereps2 time,
the device pool's kernel / H2D / D2H times and bytes, each pass's time, the expansion time and the number of passes.
Exits 1 when the device pool differs from combineDereps2 or the first pass from dada_uniques on the host-pooled derep.
Run:  python tools/pool_leg.py [--n 1000000] [--samples 8]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools import synth                   # noqa: E402
from tools.collapse_leg import gpu_info   # noqa: E402


def split(seqs, ab, quals, nsamp, seed=3):
    rng = np.random.default_rng(seed)
    n = len(seqs)
    k = rng.integers(1, 4, n)
    ds = [[] for _ in range(nsamp)]
    for i in range(n):
        who = rng.choice(nsamp, int(k[i]), replace=False)
        parts = np.maximum(1, np.round(ab[i] * rng.dirichlet(np.ones(len(who))))).astype(np.int64)
        for s, a in zip(who, parts):
            ds[s].append((i, int(a)))
    out = []
    for lst in ds:
        idx = np.array([i for i, _ in lst]); a = np.array([x for _, x in lst], np.int32)
        o = np.argsort(-a, kind="stable")
        idx, a = idx[o], a[o]
        out.append({"uniques": [seqs[i] for i in idx], "abundances": a, "quals": quals[idx],
                    "map": np.repeat(np.arange(1, len(idx) + 1, dtype=np.int32), np.minimum(a, 4))})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--samples", type=int, default=8)
    a = ap.parse_args()
    import dada2_b200
    from dada2_b200 import errmodel
    from dada2_b200.derep import combineDereps2, pool_dereps
    from dada2_b200.denoise import _expand_pooled, _qmax, initial_err
    from tests import pool_cases as P
    res = {"gpu": gpu_info(), "n": a.n, "samples": a.samples}
    seqs, ab, quals, _ = synth.illumina(a.n)
    ds = split(seqs, ab, quals, a.samples)
    res["sample_uniques"] = sum(len(d["uniques"]) for d in ds)
    t0 = time.perf_counter()
    want = combineDereps2(ds)
    res["host_combineDereps2_s"] = round(time.perf_counter() - t0, 3)
    pool_dereps(ds[:2], want_quals=False)                          # warm-up (module load, allocator)
    got = pool_dereps(ds, return_stats=True)
    st = got["stats"]
    res["pool"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in st.items()}
    res["npool"] = len(got["uniques"])
    try:
        P.assert_same(got, P.expected(ds), "device pool")
        res["pool_equals_host"] = True
    except AssertionError as e:
        res["pool_equals_host"] = False
        res["error"] = str(e)
        print(json.dumps(res))
        sys.exit(1)
    del got
    t0 = time.perf_counter()
    pd, rs = pool_dereps(ds, want_quals=False, resident=True)
    res["pool_resident_wall_s"] = round(time.perf_counter() - t0, 3)
    qmax = _qmax(pd["qmax"], 1)
    e0 = initial_err(qmax)
    first = rs.run(e0, max_clust=1)
    ref = dada2_b200.dada_uniques(want["uniques"], want["abundances"], None, e0, want["quals"], max_clust=1)
    from tests import cases
    try:
        cases.assert_same(first, ref, rtol=0, label="first pass")
        res["first_pass_equals_host_pooled"] = True
    except AssertionError as e:
        res["first_pass_equals_host_pooled"] = False
        res["error"] = str(e)
        print(json.dumps(res))
        sys.exit(1)
    passes = []

    def run(e, mc):
        t = time.perf_counter()
        r = rs.run(initial_err(qmax) if e is None else e, max_clust=mc)
        passes.append(round((time.perf_counter() - t) * 1e3, 1))
        return r
    results, err, errs, npass = errmodel.consist_loop([run], err=None, selfConsist=True)
    res["pass_ms"] = passes
    res["passes"] = npass
    pres = dict(results[0], quality=np.asarray(results[0]["clusterquals"]).T)
    t0 = time.perf_counter()
    k0 = 0
    for d in ds:
        k1 = k0 + len(d["uniques"])
        _expand_pooled(pres, pd["index"][k0:k1], d["abundances"], len(pres["clustering"]["sequence"]))
        k0 = k1
    res["expansion_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    rs.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
