"""Species assignment (dd_species.cu) on the H100: every check of the emulator file, and a seeded synthetic database of
5*10^4 references of 1 400-1 600 nt with 2*10^4 250-nt queries (half planted, some reverse-complemented, half mutated)
and 500 full-length ones, tryRC: hit lists restated exactly for a sample of 500 queries, assignments consistent with the
hit lists for every query."""
import time

import numpy as np
import pytest

from tests import species_cases as G
from tests import species_ref as S
from tests import species_synth as Y

pytestmark = pytest.mark.gpu


def test_gpu_species_example():
    G.run_example()


def test_gpu_species_synthetic(monkeypatch):
    G.run_synthetic(monkeypatch)


def test_gpu_species_refusals():
    G.check_refusals()


def test_gpu_species_synthetic_scale():
    from dada2_b200.species import SpeciesDB
    ids, refs, gseq = Y.database(50000, 2000, seed=31)
    db = SpeciesDB((ids, refs))
    print("build:", {k: db.info[k] for k in ("nbases", "device_bytes", "ms_h2d", "ms_kernels", "ms_total")})
    qs = Y.queries(refs, gseq, 20000, seed=32, full=500)
    hits, st = db.hits(qs, True)
    print("hits: %d queries, %d records, %d distinct, scan %.2f ms, reduce %.2f ms, max group %d" % (
        len(qs), st["hit_records"], st["distinct_hits"], st["ms_scan"], st["ms_reduce"], st["max_group"]))
    nhit = np.array([len(h) for h in hits])
    assert (nhit[:20000:2] > 0).all() and (nhit[20000:] > 0).all()          # every planted query hits
    assert nhit.max() > 1 and (nhit[1:20000:2] == 0).any()
    R = S.Refs(refs)
    only = np.sort(np.random.default_rng(4).choice(len(qs), 500, replace=False))
    t = time.time()
    want = R.hits([qs[j] for j in only], True)
    print("restatement: %d queries in %.1f s" % (len(only), time.time() - t))
    for j, w in zip(only, want):
        assert list(hits[j]) == w, j
    genus, species = S.labels(ids)
    for am in (False, True, 3):
        out, _ = db.assign(qs, allowMultiple=am, tryRC=True, n=len(qs))
        exp = S.assign(hits, genus, species, am)
        assert [tuple(r) for r in out] == exp, am
        print("allowMultiple=%s: %d genus, %d species assigned" % (am, sum(e[0] is not None for e in exp), sum(e[1] is not None for e in exp)))
    db.close()
