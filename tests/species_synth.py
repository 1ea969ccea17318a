"""Seeded synthetic species databases and queries for the H100 test and tools/species_leg.py.  The references come from
taxonomy_synth's mutation tree (root -> genus -> reference, some genera copying another's references exactly), so
queries hit several references, genera and species; a few references carry N runs, and some genus names are
Escherichia or Shigella."""
import numpy as np

from tests import taxonomy_synth as TS

COMP = str.maketrans("ACGT", "TGCA")


def revcomp(s):
    return s.translate(COMP)[::-1]


def database(nref, ngenus, seed=1):
    """-> (ids, refs, gseq): ids '>id Genus species', three species per genus (one in seven of them NA)."""
    refs, r2g, _, gseq = TS.database(nref, ngenus, seed=seed)
    rng = np.random.default_rng(seed + 1)
    ids = []
    for i, (r, g) in enumerate(zip(refs, r2g)):
        gname = "Escherichia" if g % 97 == 1 else "Shigella" if g % 97 == 2 else "G%d" % g
        sp = int(rng.integers(0, 3))
        ids.append("r%d %s %s" % (i, gname, "s%d_%d" % (g, sp)) if (g + sp) % 7 else "r%d %s" % (i, gname))
        if i % 100 == 17:                                                   # an N run inside the reference
            a = int(rng.integers(0, len(r) - 5))
            refs[i] = r[:a] + "NNN" + r[a + 3:]
    return ids, refs, gseq


def queries(refs, gseq, n, seed=2, length=250, full=0):
    """n queries of `length` nt: even ones planted substrings of references (every fourth reverse-complemented), odd ones
    genus windows with 2 % mutations; then `full` full-length ones (every other one a whole reference)."""
    rng = np.random.default_rng(seed)
    out = []
    mut = TS.queries(gseq, n // 2 + 1, seed=seed + 1, length=length)
    for k in range(n):
        if k % 2:
            out.append(mut[k // 2])
            continue
        r = refs[int(rng.integers(0, len(refs)))]
        a = int(rng.integers(0, len(r) - length + 1))
        q = r[a:a + length]
        if "N" in q:
            q = r[:length] if "N" not in r[:length] else r[-length:]
        out.append(revcomp(q) if k % 4 == 2 else q)
    for k in range(full):
        r = refs[int(rng.integers(0, len(refs)))]
        q = r if k % 2 == 0 else r[int(rng.integers(0, 40)):len(r) - int(rng.integers(0, 40))]
        if "N" in q:
            q = q.split("N")[0] or q.replace("N", "A")
        out.append(q)
    return out


def shared_prefix(refs, n, seed=3, length=250):
    """Worst case for the anchors: n queries sharing their first 64 nt (those of the first reference); the first one is
    that reference's first `length` nt, the others have random tails."""
    rng = np.random.default_rng(seed)
    base = refs[0][:64]
    out = []
    for k in range(n):
        tail = "".join("ACGT"[i] for i in rng.integers(0, 4, length - 64))
        out.append(refs[0][:length] if k == 0 else base + tail)
    return out
