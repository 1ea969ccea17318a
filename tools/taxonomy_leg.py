"""Measures assignTaxonomy's native core at Silva scale on one GPU: a synthetic database of 1.5*10^5 references
(1 400-1 600 nt) in 10^4 genera, classified with 10^4 and 10^5 250-nt queries (half reverse-complemented, tryRC).
Reports the table build, classify phases, table bytes and the kernels' compulsory traffic; then the reference's
C_assign_taxonomy2 (oracle/_ref/libdada2ref_taxonomy.so) on host threads for a few queries, scaled up and labelled so.
Prints one JSON object."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dada2_b200 import taxonomy as tx  # noqa: E402
from tests import taxonomy_ref as T  # noqa: E402
from tests import taxonomy_synth as S  # noqa: E402


def main():
    nref, ngenus = int(os.environ.get("TAX_NREF", 150000)), int(os.environ.get("TAX_NGENUS", 10000))
    t = time.time()
    refs, r2g, gm, gseq = S.database(nref, ngenus, seed=21, copy_every=0)
    res = {"nref": nref, "ngenus": ngenus, "gen_s": time.time() - t}
    t = time.time()
    db = tx.TaxDB.from_arrays(refs, r2g, gm)
    res["build"] = dict(db.info, wall_s=time.time() - t)
    for nq in (10000, 100000):
        qs = S.queries(gseq, nq, seed=22)
        db.raw(qs[:256], True, None, 1)                                   # warm-up
        t = time.time()
        r = db.raw(qs, True, None, 1)
        res["classify_%d" % nq] = dict(r["stats"], wall_s=time.time() - t)
    nref_q = int(os.environ.get("TAX_REF_QUERIES", 0))
    if nref_q and T.ref_lib() is not None:
        qs = S.queries(gseq, nref_q, seed=22)
        u = T.unifs_buffer(qs, 1)
        th = os.cpu_count()
        t = time.time()
        T.ref_assign(qs, refs, r2g, gm, True, u, nthreads=th)
        dt = time.time() - t
        res["reference_host"] = {"queries": nref_q, "threads": th, "s": dt,
                                 "s_per_query_per_thread_incl_build": dt * th / nref_q}
    print(json.dumps(res, default=float))


if __name__ == "__main__":
    main()
