"""Generates the goldens of the differential fuzz tests and of the 1e5-unique GPU check from the REFERENCE's own C++
(oracle/_ref/libdada2ref.so, compiled unmodified by `make -C oracle ref`):
    fuzz_pairs.npz        ref.pair() on tests/test_oracle_fuzz.py's pair cases
    e2e_fuzz<i>.npz       ref.dada_uniques() on its end-to-end cases
    bimera_fuzz.npz       ref.table_bimera() / ref.bimera_pair() on tests/test_bimera_oracle.py's fuzz cases
    e2e_fullsize_1e5.npz  ref.dada_uniques() on tests/test_gpu_fullsize.py's 1e5 uniques; map and pval at its seeded
                          sample of raws (sample_raws), so that the file stays small
    e2e_fullsize_1e5_counts.json  the k-mer screen's totals on the same 1e5 uniques (n_align, n_shroud) from the CPU
                          oracle (oracle/port.cpp), which counts them with the reference's serial semantics
Run:  python tools/make_golden_fuzz.py  (--counts-only: the counts fixture alone)"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref                               # noqa: E402
from tests import cases, test_bimera_oracle as TB, test_oracle_fuzz as TF, test_gpu_fullsize as TG   # noqa: E402
from tools.make_golden import save_res               # noqa: E402


def fullsize_counts():
    from oracle import port
    seqs, ab, q, err, _ = TG.workload()
    st = port.dada_uniques(seqs, ab, None, err, q, homo_gap=-8)["stats"]
    path = os.path.join(cases.GOLDEN, "e2e_fullsize_1e5_counts.json")
    with open(path, "w") as f:
        json.dump({"n_align": int(st["n_align"]), "n_shroud": int(st["n_shroud"])}, f)
        f.write("\n")
    print(path, open(path).read().strip())


def main():
    fullsize_counts()
    if "--counts-only" in sys.argv:
        return
    G = cases.GOLDEN
    err = cases.tperr1()
    cols = {k: [] for k in ("shrouded", "lam", "nsubs", "al0", "al1") + TF.PAIR_ARRAYS}
    for a, qa, b, qb, o in TF.pair_cases():
        r = ref.pair(a, qa, b, qb, err, **o)
        for k in ("shrouded", "lam", "nsubs", "al0", "al1"):
            cols[k].append(r[k])
        for k, v in TF.pair_arrays(r).items():
            cols[k].append(v)
    out = {k: (np.concatenate(v) if k in TF.PAIR_ARRAYS else np.array(v)) for k, v in cols.items()}
    np.savez_compressed(os.path.join(G, "fuzz_pairs.npz"), **out)
    for it, (seqs, ab, pri, q, o) in enumerate(TF.e2e_cases()):
        save_res(os.path.join(G, "e2e_fuzz%d.npz" % it), ref.dada_uniques(seqs, ab, pri, err, q, **o))
    out = {}
    for n, (seqs, mat, o, pairs) in enumerate(TB.fuzz_cases()):
        out["t%d_nflag" % n], out["t%d_nsam" % n] = ref.table_bimera(mat, seqs, **o)
        rs = [ref.bimera_pair(seqs[j], seqs[k], **{x: o[x] for x in ("allow_one_off", "max_shift")}) for j, k in pairs]
        out["t%d_pairs" % n] = np.array([[r[x] for x in TB.FUZZ_PAIR_KEYS] for r in rs], np.int32)
        out["t%d_al0" % n] = np.array([r["al0"] for r in rs])
        out["t%d_al1" % n] = np.array([r["al1"] for r in rs])
    np.savez_compressed(os.path.join(G, "bimera_fuzz.npz"), **out)
    seqs, ab, q, err, _ = TG.workload()
    ref.set_threads(min(16, os.cpu_count() or 1))
    res = ref.dada_uniques(seqs, ab, None, err, q, multithread=True)
    idx = TG.sample_raws(len(seqs))
    res["map"], res["pval"] = res["map"][idx], res["pval"][idx]
    save_res(os.path.join(G, "e2e_fullsize_1e5.npz"), res)
    for f in sorted(os.listdir(G)):
        if "fuzz" in f or "fullsize" in f:
            print(f, os.path.getsize(os.path.join(G, f)), "bytes")


if __name__ == "__main__":
    main()
