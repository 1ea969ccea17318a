"""Seeded synthetic training sets and queries for the H100 test and tools/taxonomy_leg.py: a mutation tree (root ->
genus -> reference), so that k-mers are shared across genera, with some genera copying another genus's references
exactly, so that their scores tie exactly."""
import numpy as np

ACGT = np.frombuffer(b"ACGT", np.uint8)


def _mutate(rng, a, rate):
    a = a.copy()
    m = rng.random(a.size) < rate
    a[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
    return a


def database(nref, ngenus, seed=1, lo=1400, hi=1600, copy_every=50):
    """-> (refs list[str], ref_to_genus int32 1-based, genusmat [ngenus, 6], genus sequences as uint8 arrays)."""
    rng = np.random.default_rng(seed)
    root = ACGT[rng.integers(0, 4, hi)]
    nphy = max(1, ngenus // 100)
    phyla = [_mutate(rng, root, 0.12) for _ in range(nphy)]
    gseq = []
    for g in range(ngenus):
        gseq.append(_mutate(rng, phyla[g % nphy], 0.06))
    per = np.full(ngenus, nref // ngenus)
    per[: nref - per.sum()] += 1
    refs, r2g = [], []
    base = {}
    for g in range(ngenus):
        src = g - 1 if (copy_every and g % copy_every == copy_every - 1) else g
        for i in range(per[g]):
            if src != g and (src, i) in base:
                s = base[(src, i)]
            else:
                L = int(rng.integers(lo, hi + 1))
                a0 = int(rng.integers(0, hi - L + 1))
                s = _mutate(rng, gseq[src][a0:a0 + L], 0.01).tobytes().decode()
            base[(g, i)] = s
            refs.append(s)
            r2g.append(g + 1)
    gm = np.zeros((ngenus, 6), np.int32)
    for g in range(ngenus):
        gm[g] = [1, g % nphy + 1, g % nphy + 1, (g // 10) + 1, (g // 3) + 1, g + 1]
    return refs, np.array(r2g, np.int32), gm, gseq


def queries(gseq, n, seed=2, length=250, full=False, rc_half=True):
    rng = np.random.default_rng(seed)
    comp = np.zeros(256, np.uint8)
    comp[list(b"ACGT")] = list(b"TGCA")
    out = []
    for k in range(n):
        g = gseq[int(rng.integers(0, len(gseq)))]
        if full:
            a = _mutate(rng, g[: int(rng.integers(1400, len(g) + 1))], 0.02)
        else:
            a0 = int(rng.integers(500, 540))
            a = _mutate(rng, g[a0:a0 + length], 0.02)
        if rc_half and k % 2:
            a = comp[a[::-1]]
        out.append(a.tobytes().decode())
    return out
