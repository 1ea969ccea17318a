"""Writes tests/golden/taxonomy.npz: the reference's C_assign_taxonomy2 (oracle/_ref/libdada2ref_taxonomy.so) on the man
page's example (example_seqs.fa against example_train_set.fa.gz, forward, and with tryRC on the reverse complements),
with the uniforms of the seeded draws (seed 42).  Stored: tax, boot, boot_tax, and the restatement's masks of strict
arg-maxes (the reference draws its ties at random).  The GPU machine then needs no reference sources."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dada2_b200 import taxonomy as tx  # noqa: E402
from tests import taxonomy_ref as T  # noqa: E402

SEED = 42


def main():
    if T.ref_lib() is None:
        sys.exit("oracle/_ref/libdada2ref_taxonomy.so is not built (python __graft_entry__.py)")
    ids, refs = tx.read_fasta(os.path.join(T.GOLDEN, "example_train_set.fa.gz"))
    refs, gu, r2g, gm, td = tx.parse_training(ids, refs)
    seqs = T.read_fasta(os.path.join(T.GOLDEN, "example_seqs.fa"))[1]
    lgk = T.table(refs, r2g, gm.shape[0])
    out = {}
    for name, qs, rc in (("fwd", seqs, False), ("rc", [T.revcomp(s) for s in seqs], True)):
        u = T.unifs_buffer(qs, SEED)
        got = T.ref_assign(qs, refs, r2g, gm, rc, u)
        want = T.classify(lgk, gm, qs, rc, SEED, u)
        for k in ("tax", "boot", "boot_tax"):
            out[name + "/" + k] = got[k]
        out[name + "/strict"] = want["strict"]
        out[name + "/boot_strict"] = want["boot_strict"]
    out["seed"] = np.array(SEED)
    np.savez_compressed(os.path.join(T.GOLDEN, "taxonomy.npz"), **out)
    print("wrote tests/golden/taxonomy.npz")


if __name__ == "__main__":
    main()
