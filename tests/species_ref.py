"""Plain restatement of assignSpecies / addSpecies (R/taxonomy.R:162-360; DESIGN.md 22).

The search: every query is looked for with str.find, occurrence after occurrence, in the references joined with a
separator that is not A/C/G/T, and each occurrence is mapped back to its reference; with tryRC the reverse complement is
looked for too.  The wrapper rules (the label fields, mapHits, matchGenera and addSpecies' merge) are written out again
from R's code, independently of dada2_b200/species.py."""
import bisect
import os
import re

from tests.taxonomy_ref import GOLDEN, read_fasta, revcomp

SPECIES_FA = os.path.join(GOLDEN, "example_species_assignment.fa.gz")
EXAMPLE = os.path.join(GOLDEN, "example_seqs.fa")


class Refs:
    """The references joined once, for any number of searches."""

    def __init__(self, refs):
        self.refs = list(refs)
        self.text = "|".join(self.refs)
        self.starts = []
        p = 0
        for r in self.refs:
            self.starts.append(p)
            p += len(r) + 1

    def find(self, q):
        """Sorted distinct indices of the references holding q."""
        out, i = set(), self.text.find(q)
        while i >= 0:
            out.add(bisect.bisect_right(self.starts, i) - 1)
            i = self.text.find(q, i + 1)
        return out

    def hits(self, seqs, try_rc):
        res = []
        for q in seqs:
            h = self.find(q)
            if try_rc:
                h |= self.find(revcomp(q))
            res.append(sorted(h))
        return res


# ---- R's wrapper rules ----
def r_split_ws(s):
    """strsplit(s, "\\\\s")[[1]]: one field per whitespace character, a trailing empty field dropped."""
    f = re.split(r"\s", s, flags=re.ASCII)
    return f[:-1] if f and f[-1] == "" else f


def labels(ids):
    f = [r_split_ws(t) for t in ids]
    return [x[1] if len(x) > 1 else None for x in f], [x[2] if len(x) > 2 else None for x in f]


def format_error(ids):
    if len(r_split_ws(ids[0])) >= 3:
        return None
    if ids[0].count(";") >= 3:
        return "Incorrect reference file format for assignSpecies (this looks like a file formatted for assignTaxonomy)."
    return "Incorrect reference file format for assignSpecies."


def map_hits(x, refs, keep):
    hits = [refs[i] for i in x]
    hits = ["Escherichia/Shigella" if (h is not None and ("Escherichia" in h or "Shigella" in h)) else h for h in hits]
    uniq = list(dict.fromkeys(hits))
    if len(uniq) <= keep:
        rval = sorted(h for h in uniq if h is not None)
        return "/".join(rval) if rval else None
    return None


def keep_of(allowMultiple):
    if isinstance(allowMultiple, bool):
        return float("inf") if allowMultiple else 1
    return int(allowMultiple)


def assign(hits, genus, species, allowMultiple=False):
    keep = keep_of(allowMultiple)
    return [(map_hits(h, genus, 1), map_hits(h, species, keep)) for h in hits]


def match_genera(gen_tax, gen_binom, split_glyph="/"):
    if gen_tax is None or gen_binom is None:
        return False
    if len(gen_tax) == 0 or len(gen_binom) == 0:
        return False
    return bool(gen_tax == gen_binom or re.search("^%s[ _%s]" % (gen_binom, split_glyph), gen_tax)
                or re.search("%s%s$" % (split_glyph, gen_binom), gen_tax))


def add(rows, names, binom):
    """addSpecies on a table given as row lists: -> (rows, names)."""
    gcol = names.index("Genus") if "Genus" in names else len(names) - 1
    match = [match_genera(r[gcol], b[0]) for r, b in zip(rows, binom)]
    rows = [list(r) + [b[1]] for r, b in zip(rows, binom)]
    names = list(names) + ["Species"]
    scol = names.index("Species")
    for r, m in zip(rows, match):
        if not m:
            r[scol] = None
    return rows, names


def example():
    """(ids, refs) of the species fixture and the man page's query sequences."""
    return read_fasta(SPECIES_FA), read_fasta(EXAMPLE)[1]
