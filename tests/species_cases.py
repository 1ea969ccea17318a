"""Species cases shared by the emulator and the H100 files: the product (dd_species.cu behind dada2_b200/species.py)
against the restatement (tests/species_ref.py), hit lists exactly and assignments row by row, on the man page's
example and on a small synthetic set built to sit on every edge of the scan; then the same answers with a one-record
hit buffer, with every anchor at offset 0, with small batches and from a reused database; and every refusal."""
import random

import numpy as np
import pytest

from tests import species_ref as S
from tests.taxonomy_ref import revcomp

ACGT = "ACGT"


def _rand(rng, n):
    return "".join(rng.choice(ACGT) for _ in range(n))


def synthetic(seed=5):
    """-> (ids, refs, queries): references with N / IUPAC runs inside and right next to planted queries; queries of 1, 2,
    31, 32, 33 and 64 nt; a query equal to a whole reference and one a base longer; a query occurring twice in one
    reference; a palindrome; reverse-complement-only hits; a query across a reference boundary and one across an N; and
    50 queries sharing their first 64 nt."""
    rng = random.Random(seed)
    refs = [_rand(rng, rng.randint(150, 400)) for _ in range(30)]
    qs = []
    for L in (1, 2, 31, 32, 33, 64, 100, 250):                                # planted substrings of several lengths
        r = rng.randrange(len(refs))
        if len(refs[r]) < L:
            continue
        a = rng.randint(0, len(refs[r]) - L)
        qs.append(refs[r][a:a + L])
    qs += ["A", "T", "ACG", "GGGGGGGGGGGGGGGGGGGGGGGGGGGGGGGGGG"]
    qs += [refs[4], refs[4] + "A", "C" + refs[6], refs[6][1:]]                 # whole reference, one base longer
    q2 = _rand(rng, 40)                                                        # twice in one reference
    refs.append(_rand(rng, 50) + q2 + _rand(rng, 30) + q2 + _rand(rng, 20))
    qs.append(q2)
    half = _rand(rng, 20)                                                      # palindrome (its own reverse complement)
    pal = half + revcomp(half)
    refs.append(_rand(rng, 60) + pal + _rand(rng, 60))
    qs.append(pal)
    for L in (12, 33, 70):                                                     # reverse-complement-only hits
        q = _rand(rng, L)
        refs.append(_rand(rng, 40) + revcomp(q) + _rand(rng, 40))
        qs.append(q)
    for run in ("N", "NNNN", "RYKM", "-", "W"):                                # non-ACGT runs right next to and inside queries
        q = _rand(rng, 45)
        refs.append(_rand(rng, 30) + run + q + run + _rand(rng, 30))
        qs.append(q)
        q = _rand(rng, 45)
        refs.append(_rand(rng, 30) + q[:20] + run + q[20 + len(run):] + _rand(rng, 30))
        qs.append(q)
        qs.append(q[:20])
        qs.append(q[20 + len(run):])
    qs.append(refs[10][-20:] + refs[11][:20])                                  # across a reference boundary: no hit
    qs.append(refs[10][-1:] + refs[11][:1])
    prefix = _rand(rng, 64)                                                    # 50 queries sharing their first 64 nt
    shared = [prefix + _rand(rng, 100) for _ in range(50)]
    for k in range(0, 50, 5):
        refs.append(_rand(rng, 25) + shared[k] + _rand(rng, 25))
    refs.append(_rand(rng, 10) + prefix + _rand(rng, 10))
    qs += shared + [prefix]
    refs.append(_rand(rng, 100).lower())                                       # lower case matches nothing
    qs.append(refs[-1][10:40].upper())
    refs.append("N" * 50)
    qs += [_rand(rng, L) for L in (1, 2, 31, 32, 33, 64)]                      # unplanted
    genus = ["Lactobacillus", "Escherichia", "Shigella", "Bacillus", "Clostridium", "Escherichia-Shigella", "Bacillus"]
    species = ["salivarius", "coli", "flexneri", "subtilis", "similis", "coli", "cereus"]
    ids = []
    for i in range(len(refs)):
        g, s = genus[i % len(genus)], species[(i * 3) % len(species)]
        if i == 0:
            ids.append("r0 %s %s" % (g, s))
        elif i % 11 == 3:
            ids.append("r%d %s" % (i, g))                                      # species NA
        elif i % 11 == 5:
            ids.append("r%d  %s %s" % (i, g, s))                               # double space: genus "", species = g
        elif i % 11 == 7:
            ids.append("r%d" % i)                                              # both NA
        else:
            ids.append("r%d %s %s extra" % (i, g, s))
    return ids, refs, qs


def check(db, ids, refs, qs, try_rc, label="", n=2000):
    """Hit hook and assign (allowMultiple FALSE, TRUE, 2) against the restatement."""
    R = S.Refs(refs)
    want = R.hits(qs, try_rc)
    got, st = db.hits(qs, try_rc)
    assert len(got) == len(qs)
    for j, (g, w) in enumerate(zip(got, want)):
        assert list(g) == w, (label, j, qs[j][:40], list(g), w)
    genus, species = S.labels(ids)
    for am in (False, True, 2):
        out, names = db.assign(qs, allowMultiple=am, tryRC=try_rc, n=n)
        assert names == ["Genus", "Species"] and out.shape == (len(qs), 2)
        exp = S.assign(want, genus, species, am)
        for j, (row, e) in enumerate(zip(out, exp)):
            assert tuple(row) == e, (label, am, j, tuple(row), e)
    return got, st


def example_db():
    from dada2_b200.species import SpeciesDB
    return SpeciesDB(S.SPECIES_FA)


def run_example():
    """The man page's example: hit lists, the table of DESIGN.md 22, and tryRC on reverse-complemented queries."""
    from dada2_b200 import species as sp
    (ids, refs), qs = S.example()
    db = example_db()
    for rc in (False, True):
        check(db, ids, refs, qs, rc, "example rc=%d" % rc)
    check(db, ids, refs, [revcomp(q) for q in qs], True, "example rc queries")
    single, _ = sp.assignSpecies(qs, S.SPECIES_FA)
    multi, _ = sp.assignSpecies(qs, S.SPECIES_FA, allowMultiple=True)
    rcm, _ = sp.assignSpecies([revcomp(q) for q in qs], S.SPECIES_FA, allowMultiple=True, tryRC=True)
    want = [("Lactobacillus", None, "mixtipabuli/odoratitofui/similis"), (None, None, None), ("Virgibacillus", "kekensis", "kekensis"),
            (None, None, None), ("Clostridium", "hydrogeniformans", "hydrogeniformans"), (None, None, None)]
    for j, (g, s1, sm) in enumerate(want):
        assert tuple(single[j]) == (g, s1) and tuple(multi[j]) == (g, sm) and tuple(rcm[j]) == (g, sm), j
    return db


def run_synthetic(monkeypatch, extra=()):
    """The synthetic set, then the hooks, batches and a reused database; the answers must not change."""
    from dada2_b200.species import SpeciesDB
    ids, refs, qs = synthetic()
    qs = qs + list(extra)
    db = SpeciesDB((ids, refs))
    base = {}
    for rc in (False, True):
        base[rc], st = check(db, ids, refs, qs, rc, "synthetic rc=%d" % rc)
        assert st["scans"] == 1 and st["hit_records"] > st["distinct_hits"] > 0
    monkeypatch.setenv("DADA2B_SPECIES_HITCAP", "1")
    _, st = check(db, ids, refs, qs, True, "hitcap=1")
    assert st["scans"] == 2 and st["hit_capacity"] == st["hit_records"]
    monkeypatch.delenv("DADA2B_SPECIES_HITCAP")
    monkeypatch.setenv("DADA2B_SPECIES_ANCHOR0", "1")
    _, st0 = check(db, ids, refs, qs, True, "anchor0")
    monkeypatch.delenv("DADA2B_SPECIES_ANCHOR0")
    _, st1 = db.hits(qs, True)
    assert st0["max_group"] >= 51 > st1["max_group"], (st0["max_group"], st1["max_group"])   # 50 shared prefixes + the prefix
    for n in (1, 7):
        check(db, ids, refs, qs, True, "n=%d" % n, n=n)
    again, _ = db.hits(qs, True)
    assert [list(x) for x in again] == [list(x) for x in base[True]]
    db.close()
    return db


def check_refusals():
    from dada2_b200 import Dada2bError, species as sp
    (ids, refs), qs = S.example()
    db = example_db()
    for bad in (["ACGTN"], ["acgt"], ["ACGT", "AC GT"]):
        with pytest.raises(Dada2bError, match="Non-ACGT characters present in the query sequences."):
            db.assign(bad)
        with pytest.raises(Dada2bError, match="Non-ACGT characters present in the query sequences."):
            db.raw(bad)                                                       # the native check, without the wrapper's
    with pytest.raises(Dada2bError, match="empty"):
        db.assign(["ACGT", ""])
    with pytest.raises(Dada2bError, match="empty"):
        db.raw([""])
    with pytest.raises(Dada2bError, match="n must be"):
        db.assign(qs, n=0)
    with pytest.raises(Dada2bError, match=r"looks like a file formatted for assignTaxonomy"):
        sp.SpeciesDB((["Bacteria;Firmicutes;Bacilli;Lactobacillales;"], ["ACGT" * 10]))
    with pytest.raises(Dada2bError, match=r"^Incorrect reference file format for assignSpecies\.$"):
        sp.SpeciesDB((["id Genus"], ["ACGT" * 10]))
    with pytest.raises(Dada2bError, match="Non-ACGT"):                          # the queries are checked before the format
        sp.assignSpecies(["ACGN"], (["id Genus"], ["ACGT" * 10]))
    db.close()
    with pytest.raises(Dada2bError, match="closed"):
        db.assign(qs)
    empty, names = example_db().assign([])
    assert empty.shape == (0, 2) and names == ["Genus", "Species"]
