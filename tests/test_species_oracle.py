"""assignSpecies / addSpecies' wrapper rules (dada2_b200/species.py) against the restatement (tests/species_ref.py),
on crafted fastas, and the man page's example through the restatement -- CPU only."""
import numpy as np
import pytest

from dada2_b200 import Dada2bError, species as sp
from tests import species_ref as S
from tests.taxonomy_ref import revcomp

IDS = ["r0 Lactobacillus salivarius", "r1 Escherichia coli", "r2 Shigella flexneri", "r3 Bacillus", "r4  Bacillus cereus",
       "r5", "r6 Escherichia-Shigella coli x", "r7 Bacillus subtilis", "r8 Bacillus cereus", "r9 Clostridium Escherichia_like"]


def product_assign(hits, ids, allowMultiple):
    """The wrapper's path from the device's answer (distinct label ids per query) to the two columns."""
    g, s = sp.parse_species(ids)
    gi, gn = sp.label_ids(g)
    si, sn = sp.label_ids(s)
    keep = sp.keep_of(allowMultiple)
    out = []
    for h in hits:
        dg = sorted(set(gi[h].tolist()))
        ds = sorted(set(si[h].tolist()))
        out.append((sp.map_hits(len(dg), [gn[x] for x in dg], 1), sp.map_hits(len(ds), [sn[x] for x in ds], keep)))
    return out


def test_species_fields():
    g, s = S.labels(IDS)
    assert g == sp.parse_species(IDS)[0] and s == sp.parse_species(IDS)[1]
    assert (g[3], s[3]) == ("Bacillus", None)                                 # species field missing: NA
    assert (g[4], s[4]) == ("", "Bacillus")                                   # double space: an empty genus field
    assert (g[5], s[5]) == (None, None)
    ids, names = sp.label_ids(g)
    assert names[0] is None and ids[5] == 0
    assert names[ids[1]] == names[ids[2]] == names[ids[6]] == "Escherichia/Shigella"
    sids, snames = sp.label_ids(s)
    assert snames[sids[9]] == "Escherichia/Shigella"                          # mapHits rewrites species labels too


@pytest.mark.parametrize("allowMultiple", [False, True, 1, 2, 3, 0, -1, 2.7])
def test_species_map_hits(allowMultiple):
    hits = [[], [0], [1, 2], [1, 6], [3, 7, 8], [7, 8], [4, 7], [5], [5, 0], [3], [9, 1], [0, 7, 8, 4], list(range(10))]
    g, s = S.labels(IDS)
    want = S.assign(hits, g, s, allowMultiple)
    assert product_assign([np.array(h, int) for h in hits], IDS, allowMultiple) == want
    if allowMultiple is False:
        assert want[2] == ("Escherichia/Shigella", None) and want[5] == ("Bacillus", None) and want[8] == (None, None)
        assert want[3] == ("Escherichia/Shigella", "coli") and want[9] == ("Bacillus", None)
    if allowMultiple is True:
        assert want[4][1] == "cereus/subtilis" and want[8] == (None, "salivarius")   # NA counted by unique, dropped by sort
        assert want[11] == (None, "Bacillus/cereus/salivarius/subtilis")


def test_species_keep():
    assert sp.keep_of(False) == 1 and sp.keep_of(True) == float("inf") and sp.keep_of(2) == 2 and sp.keep_of(2.7) == 2
    assert sp.keep_of(np.bool_(True)) == float("inf")


def test_species_format_errors():
    for ids, msg in ((["Bacteria;Firmicutes;Bacilli;Lactobacillales;"], "(this looks like a file formatted for assignTaxonomy)"),
                     (["a;b;c;"], "(this looks like a file formatted for assignTaxonomy)"), (["a;b;c"], None), (["id Genus"], None), (["a;b Genus"], None),
                     (["id Genus species"], "ok"), (["id  Genus"], "ok")):
        want = S.format_error(ids)
        if msg == "ok":
            assert want is None
            sp.parse_species(ids)
            continue
        assert want == ("Incorrect reference file format for assignSpecies " + msg + "." if msg else
                        "Incorrect reference file format for assignSpecies.")
        with pytest.raises(Dada2bError) as e:
            sp.parse_species(ids)
        assert str(e.value) == want


def test_species_query_refusals():
    with pytest.raises(Dada2bError, match="^Non-ACGT characters present in the query sequences.$"):
        sp._check_queries(["ACGT", "ACGN"])
    with pytest.raises(Dada2bError, match="^Non-ACGT characters present in the query sequences.$"):
        sp.assignSpecies(["acgt"], (IDS[:1], ["ACGT"]))
    with pytest.raises(Dada2bError, match="empty"):
        sp._check_queries(["ACGT", ""])


@pytest.mark.parametrize("tax,binom,want", [
    ("Escherichia/Shigella", "Escherichia/Shigella", True), ("Clostridium_sensu_stricto_1", "Clostridium", True),
    ("Clostridium sensu stricto", "Clostridium", True), ("Clostridium/Sarcina", "Clostridium", True),
    ("Sarcina/Clostridium", "Clostridium", True), ("Clostridiumx", "Clostridium", False), ("xClostridium", "Clostridium", False),
    ("Bacillus", "Bacillu.", False), ("Bacillus_1", "Bacill.s", True), ("a/Bacillus", "Bac.*", True), (None, "Bacillus", False),
    ("Bacillus", None, False), ("", "", False), ("Bacillus", "", False), ("Lactobacillus", "Bacillus", False)])
def test_species_match_genera(tax, binom, want):
    assert S.match_genera(tax, binom) is want
    assert sp.match_genera(tax, binom) is want


def test_species_add_merge():
    rows = [["Bacteria", "Firmicutes", "Clostridium_sensu_stricto_1"], ["Bacteria", "Firmicutes", "Bacillus"],
            ["Bacteria", None, None], ["Bacteria", "Proteobacteria", "Escherichia/Shigella"]]
    binom = np.array([["Clostridium", "butyricum"], ["Lactobacillus", "salivarius"], [None, None], ["Escherichia/Shigella", "coli"]],
                     dtype=object)
    for names in (["Kingdom", "Phylum", "Genus"], ["Kingdom", "Phylum", "Family"], ["Kingdom", "Genus", "Genus"]):
        got, gnames = sp.merge_species((np.array(rows, dtype=object), names), binom)
        want, wnames = S.add(rows, names, binom.tolist())
        assert gnames == wnames == names + ["Species"]
        assert got.tolist() == want
        if names == ["Kingdom", "Phylum", "Genus"]:
            assert got.tolist()[0][-1] == "butyricum" and got.tolist()[1][-1] is None and got.tolist()[3][-1] == "coli"


def test_species_add_duplicate_species_column():
    """A table that already ends in a Species level: R blanks the first column named Species, not the new one."""
    rows = [["Bacteria", "Bacillus", "old1"], ["Bacteria", "Clostridium", "old2"]]
    names = ["Kingdom", "Genus", "Species"]
    binom = np.array([["Lactobacillus", "new1"], ["Clostridium", "new2"]], dtype=object)
    got, gnames = sp.merge_species((np.array(rows, dtype=object), names), binom)
    want, wnames = S.add(rows, names, binom.tolist())
    assert gnames == wnames == ["Kingdom", "Genus", "Species", "Species"]
    assert got.tolist() == want == [["Bacteria", "Bacillus", None, "new1"], ["Bacteria", "Clostridium", "old2", "new2"]]


def test_species_man_page_example_restated():
    (ids, refs), qs = S.example()
    g, s = S.labels(ids)
    R = S.Refs(refs)
    want = {False: [("Lactobacillus", None), (None, None), ("Virgibacillus", "kekensis"), (None, None),
                    ("Clostridium", "hydrogeniformans"), (None, None)],
            True: [("Lactobacillus", "mixtipabuli/odoratitofui/similis"), (None, None), ("Virgibacillus", "kekensis"), (None, None),
                   ("Clostridium", "hydrogeniformans"), (None, None)]}
    for am in (False, True):
        assert S.assign(R.hits(qs, False), g, s, am) == want[am]
        assert S.assign(R.hits([revcomp(q) for q in qs], True), g, s, am) == want[am]
        assert product_assign([np.array(h, int) for h in R.hits(qs, False)], ids, am) == want[am]
    assert all(R.hits([revcomp(q) for q in qs], False)[j] == [] for j in (0, 2, 4))
