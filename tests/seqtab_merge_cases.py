"""mergeSequenceTables cases shared by the emulator and H100 tests: hand-built tables whose expected matrix, columns and
rows are written out literally (each is also checked against the restatement in seqtab_merge_ref.py), refusals, and a
seeded multi-run generator (runs of 96 samples over a shared ASV pool of 250-nt reads and 450-nt merged reads with N
runs, some runs in reverse orientation, about 1 % duplicate column names)."""
import contextlib
import io
import re
import warnings

import numpy as np

from tests import seqtab_merge_ref as R

S1, S3, S4 = "AAAC", "CCGA", "AAAA"           # rc: GTTT, TCGG, TTTT
S2 = "ACGT"                                    # a palindrome
IU = "ACGTNNNNRYKMBDHVSW"
IU_RC = "WSBDHVKMRYNNNNACGT"                   # rc(IU), written out


def t(mat, cols, rows):
    return (np.array(mat, np.int32), list(cols), list(rows))


# (id, positional tables, keyword arguments, expected (mat, cols, rows) or an error regex, expected messages)
HAND = [
    ("disjoint", [t([[1, 2]], [S1, S3], "a"), t([[5]], [S4], "b")], {"orderBy": None},
     ([[1, 2, 0], [0, 0, 5]], [S1, S3, S4], ["a", "b"]), []),
    ("disjoint_abundance", [t([[1, 2]], [S1, S3], "a"), t([[5]], [S4], "b")], {},
     ([[0, 2, 1], [5, 0, 0]], [S4, S3, S1], ["a", "b"]), []),
    ("overlap", [t([[1, 2], [3, 4]], [S1, S3], "ab"), t([[10, 0], [0, 7]], [S3, S4], "cd")], {},
     ([[2, 0, 1], [4, 0, 3], [10, 0, 0], [0, 7, 0]], [S3, S4, S1], ["a", "b", "c", "d"]), []),
    ("three_more", [t([[1]], [S1], "a"), t([[2]], [S1], "b"), t([[3, 1]], [S3, S1], "c")], {},
     ([[1, 0], [2, 0], [1, 3]], [S1, S3], ["a", "b", "c"]), []),
    ("unequal_rows", [t([[1], [2], [3]], [S1], "abc"), t([[4, 5]], [S1, S3], "d")], {},
     ([[1, 0], [2, 0], [3, 0], [4, 5]], [S1, S3], ["a", "b", "c", "d"]), []),
    ("repeats_error_across", [t([[1]], [S1], "a"), t([[2]], [S3], "a")], {},
     r"^Duplicated sample names detected in the sequence table row names: a$", []),
    ("repeats_error_within", [t([[1], [2]], [S1], "aa"), t([[2]], [S3], "b")], {},
     r"^Duplicated sample names detected in the sequence table row names: a$", ["Duplicated row (sample) names."]),
    ("repeats_sum_across", [t([[1, 2]], [S1, S3], "a"), t([[10, 20]], [S3, S4], "a")], {"repeats": "sum", "orderBy": None},
     ([[1, 12, 20]], [S1, S3, S4], ["a"]), ["Duplicated sample names detected in the sequence table row names."]),
    ("repeats_sum_row_last_wins", [t([[1, 2], [5, 6]], [S1, S3], "aa"), t([[7]], [S1], "b")], {"repeats": "sum", "orderBy": None},
     ([[5, 6], [7, 0]], [S1, S3], ["a", "b"]), ["Duplicated row (sample) names.", "Duplicated sample names detected"]),
    ("repeats_sum_row_last_wins_plus_table", [t([[1, 2], [5, 6]], [S1, S3], "aa"), t([[100, 9]], [S1, S4], "a")],
     {"repeats": "other", "orderBy": None}, ([[105, 6, 9]], [S1, S3, S4], ["a"]), ["Duplicated sample names detected"]),
    ("dup_col_last_wins", [t([[1, 2, 3]], [S1, S3, S1], "a"), t([[4]], [S4], "b")], {"orderBy": None},
     ([[3, 2, 0], [0, 0, 4]], [S1, S3, S4], ["a", "b"]), ["Duplicated column (sequences) names."]),
    ("dup_row_and_col_last_wins", [t([[1, 2], [3, 4]], [S1, S1], "aa"), t([[1]], [S3], "b")], {"repeats": "sum", "orderBy": None},
     ([[4, 0], [0, 1]], [S1, S3], ["a", "b"]), []),
    ("rc_other_table_collapsed", [t([[1]], [S1], "a"), t([[2, 3, 4]], ["GTTT", S3, S3], "b")], {"tryRC": True, "orderBy": None},
     ([[1, 0], [2, 7]], [S1, S3], ["a", "b"]), ["Reverse complemented sequences detected and re-oriented."]),
    ("rc_off_same_tables", [t([[1]], [S1], "a"), t([[2, 3, 4]], ["GTTT", S3, S3], "b")], {"orderBy": None},
     ([[1, 0, 0], [0, 2, 4]], [S1, "GTTT", S3], ["a", "b"]), []),
    ("rc_same_table", [t([[1, 2]], [S1, "GTTT"], "a"), t([[3]], [S3], "b")], {"tryRC": True, "orderBy": None},
     ([[3, 0], [0, 3]], [S1, S3], ["a", "b"]), ["Reverse complemented sequences detected and re-oriented."]),
    ("rc_first_seen_later_table", [t([[1]], [S3], "a"), t([[2, 5]], [S4, "TCGG"], "b"), t([[4, 6]], ["TTTT", S3], "c")],
     {"tryRC": True, "orderBy": None}, ([[1, 0], [5, 2], [6, 4]], [S3, S4], ["a", "b", "c"]),
     ["Reverse complemented sequences detected and re-oriented."]),
    ("palindrome", [t([[1, 2]], [S2, S1], "a"), t([[5]], [S2], "b")], {"tryRC": True, "orderBy": None},
     ([[1, 2], [5, 0]], [S2, S1], ["a", "b"]), []),
    ("iupac_n", [t([[4]], [IU], "a"), t([[6, 1]], [IU_RC, "NNNN"], "b")], {"tryRC": True},
     ([[4, 0], [6, 1]], [IU, "NNNN"], ["a", "b"]), ["Reverse complemented sequences detected and re-oriented."]),
    ("order_abundance_ties", [t([[2, 1, 3]], [S1, S3, S4], "a"), t([[1, 1]], [S3, S4], "b")], {},
     ([[3, 2, 1], [1, 0, 1]], [S4, S1, S3], ["a", "b"]), []),
    ("order_nsamples_ties", [t([[2, 1, 3]], [S1, S3, S4], "a"), t([[1, 1]], [S3, S4], "b")], {"orderBy": "nsamples"},
     ([[1, 3, 2], [1, 1, 0]], [S3, S4, S1], ["a", "b"]), []),
    ("order_none", [t([[2, 1, 3]], [S1, S3, S4], "a"), t([[1, 1]], [S3, S4], "b")], {"orderBy": None},
     ([[2, 1, 3], [0, 1, 1]], [S1, S3, S4], ["a", "b"]), []),
    ("order_unknown", [t([[2, 1, 3]], [S1, S3, S4], "a"), t([[1, 1]], [S3, S4], "b")], {"orderBy": "sequence"},
     ([[2, 1, 3], [0, 1, 1]], [S1, S3, S4], ["a", "b"]), []),
    ("float_entries", [(np.array([[1.0, 2.0]]), [S1, S3], ["a"]), t([[5]], [S4], "b")], {"orderBy": None},
     ([[1, 2, 0], [0, 0, 5]], [S1, S3, S4], ["a", "b"]), []),
    ("overflow_cell", [t([[2 ** 31 - 1]], [S1], "a"), t([[1]], [S1], "a")], {"repeats": "sum"}, r"int32 range \(R would return NA\)", []),
    ("overflow_colsum", [t([[2 ** 31 - 1]], [S1], "a"), t([[1]], [S1], "b")], {}, r"int32 range \(R would return NA\)", []),
    ("bad_letter", [t([[1]], ["ACGU"], "a"), t([[1]], [S1], "b")], {}, r"IUPAC.*found 'U'", []),
    ("bad_lower_case", [t([[1]], ["acgt"], "a"), t([[1]], [S1], "b")], {"tryRC": True}, r"IUPAC.*found 'a'", []),
]

GOOD = t([[1]], [S1], "a")
# refusals made on the host before any device work: (id, args, kwargs, error regex)
REFUSALS = [
    ("neither", [GOOD], {}, r"^Either 'tables' or 'table1' and 'table2' must be provided\.$"),
    ("one_table", [], {"tables": [GOOD]}, r"^At least two sequence tables are expected$"),
    ("not_a_list", [], {"tables": 5}, r"^'tables' must be a list or vector\.$"),
    ("rds_names", [], {"tables": ["a.rds", "b.rds"]}, r"RDS"),
    ("rds_name", [], {"tables": "a.rds"}, r"RDS"),
    ("negative_named", [], {"tables": {"x": GOOD, "y": t([[-1]], [S3], "b")}}, r"^Some sequence tables found invalid: y$"),
    ("negative_unnamed", [GOOD, t([[-1]], [S3], "b")], {}, r"^Some sequence tables found invalid$"),
    ("not_matrix", [], {"tables": {"x": (np.array([1, 2]), [S1, S3], ["a"]), "y": GOOD, "z": "seqtab"}}, r"RDS"),
    ("not_matrix_1d", [], {"tables": {"x": (np.array([1, 2]), [S1, S3], ["a"]), "y": GOOD}}, r"^Some sequence tables found invalid: x$"),
    ("no_colnames", [], {"tables": {"x": (np.array([[1]]), None, ["a"]), "y": GOOD}}, r"found invalid: x$"),
    ("no_rownames", [], {"tables": {"x": GOOD, "y": (np.array([[1]]), [S3], None)}}, r"found invalid: y$"),
    ("no_columns", [], {"tables": {"x": GOOD, "y": (np.zeros((1, 0), np.int32), [], ["b"])}}, r"found invalid: y$"),
    ("blank_col", [], {"tables": {"x": GOOD, "y": t([[1]], [""], "b"), "z": t([[1]], [S3], [""])}}, r"found invalid: y, z$"),
    ("non_integer", [GOOD, (np.array([[1.5]]), [S3], ["b"])], {}, r"whole numbers"),
]
WARNS = {"not_matrix_1d": "Not a matrix.", "negative_named": "Negative entries.", "no_colnames": "Column (sequence) names are missing.",
         "no_rownames": "Row (sample) names are missing.", "no_columns": "Column (sequence) names are missing.",
         "blank_col": "Some column (sequence) names are blank."}


def _call(fn, args, kw):
    err, out, got_w = io.StringIO(), None, []
    with warnings.catch_warnings(record=True) as w, contextlib.redirect_stderr(err):
        warnings.simplefilter("always")
        exc = None
        try:
            out = fn(*args, **kw)
        except Exception as e:                                      # noqa: BLE001 - compared by the caller
            exc = e
        got_w = [str(x.message) for x in w]
    return out, exc, err.getvalue() + "\n".join(got_w)


def _ref(*args, **kw):
    kw = dict(kw)
    tables = kw.pop("tables", None)
    names = None
    if isinstance(tables, dict):
        names, tables = list(tables), list(tables.values())
    tables = list(args) if tables is None else tables
    mat, cols, rows, msgs = R.merge(tables, names, **kw)
    return (mat, cols, rows), "\n".join(msgs)


def check_hand():
    import dada2_b200
    from dada2_b200 import Dada2bError
    for cid, args, kw, want, msgs in HAND:
        got, exc, text = _call(dada2_b200.mergeSequenceTables, args, kw)
        ref, rexc, rtext = _call(_ref, args, kw)
        if isinstance(want, str):
            assert isinstance(exc, Dada2bError) and re.search(want, str(exc)), (cid, exc)
            assert isinstance(rexc, R.RefError) and re.search(want, str(rexc)), (cid, rexc)
        else:
            assert exc is None, (cid, exc)
            assert rexc is None, (cid, rexc)
            for label, (mat, cols, rows) in (("product", got), ("restatement", ref[0])):
                assert mat.dtype == np.int32, (cid, label)
                assert np.array_equal(mat, np.array(want[0], np.int32)), (cid, label, mat)
                assert cols == want[1] and rows == want[2], (cid, label, cols, rows)
            for m in msgs:
                assert m in ref[1], (cid, "restatement", m, ref[1])
        for m in msgs:
            assert m in text, (cid, m, text)
        if "Reverse complemented" not in " ".join(msgs) and not isinstance(want, str):
            assert "Reverse complemented" not in text, cid
    # three or more tables through `tables=`, as a list and as a dict, equal the positional call
    three = HAND[3][1]
    a = dada2_b200.mergeSequenceTables(*three)
    for tables in (three, {"r%d" % i: x for i, x in enumerate(three)}):
        b = dada2_b200.mergeSequenceTables(tables=tables)
        assert np.array_equal(a[0], b[0]) and a[1:] == b[1:]


def check_refusals():
    """Every host-side refusal, with R's message and is.sequence.table's warning; no device is needed."""
    import dada2_b200
    from dada2_b200 import Dada2bError
    for cid, args, kw, want in REFUSALS:
        _, exc, text = _call(dada2_b200.mergeSequenceTables, args, kw)
        assert isinstance(exc, Dada2bError) and re.search(want, str(exc)), (cid, exc)
        if cid in WARNS:
            assert WARNS[cid] in text, (cid, text)
        if "RDS" not in want and cid != "not_a_list" and "Either" not in want:
            _, rexc, _ = _call(_ref, args, kw)
            assert isinstance(rexc, R.RefError) and re.search(want, str(rexc)), (cid, rexc)


# ---- seeded multi-run tables ------------------------------------------------------------------------------------------
def _random_seqs(rng, n, length):
    raw = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n * length)].tobytes()
    return [raw[i * length:(i + 1) * length].decode() for i in range(n)]


def make_runs(seed, nruns=4, nsamp=96, pool=3000, per_run=600, merged_frac=0.3, rc_every=3, dup_frac=0.01, shared_frac=0.0,
              density=0.08):
    """nruns tables of nsamp samples.  The ASV pool holds 250-nt reads and 450-nt merged reads (220 + ten N + 220);
    each run takes per_run of them, every rc_every-th run (1-based) in reverse orientation, and about dup_frac of its
    columns again under the same name.  With shared_frac, that share of a run's sample names repeats the previous
    run's (merge those with repeats="sum")."""
    rng = np.random.default_rng(seed)
    nmerged = int(pool * merged_frac)
    seqs = _random_seqs(rng, pool - nmerged, 250)
    halves = _random_seqs(rng, 2 * nmerged, 220)
    seqs += [halves[2 * i] + "N" * 10 + halves[2 * i + 1] for i in range(nmerged)]
    order = rng.permutation(pool)
    seqs = [seqs[k] for k in order]
    runs = []
    for r in range(nruns):
        pick = rng.choice(pool, per_run, replace=False)
        cols = [seqs[k] for k in pick]
        if rc_every and (r + 1) % rc_every == 0:
            cols = [R.rc(c) for c in cols]
        ndup = int(round(dup_frac * per_run))
        for k in rng.choice(per_run, ndup, replace=False):
            cols.insert(int(rng.integers(0, len(cols) + 1)), cols[k])
        mask = rng.random((nsamp, len(cols))) < density
        mat = np.where(mask, rng.integers(1, 2000, (nsamp, len(cols))), 0).astype(np.int32)
        rows = ["run%d_s%d" % (r, i) for i in range(nsamp)]
        if shared_frac and r > 0:
            for i in rng.choice(nsamp, int(shared_frac * nsamp), replace=False):
                rows[i] = "run%d_s%d" % (r - 1, i)
        runs.append((mat, cols, rows))
    return runs


def check_seeded(runs, **kw):
    """The product against the restatement on one merge; returns the product's result."""
    import dada2_b200
    got, exc, _ = _call(dada2_b200.mergeSequenceTables, [], dict(kw, tables=runs))
    assert exc is None, exc
    (mat, cols, rows), _ = _ref(tables=runs, **kw)
    assert got[1] == cols and got[2] == rows
    assert got[0].dtype == np.int32 and np.array_equal(got[0], mat)
    return got
