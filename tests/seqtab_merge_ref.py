"""Line-by-line restatement of mergeSequenceTables (R/multiSample.R:290-364) with is.sequence.table (:206-238), rc
(R/misc.R:272-280, Biostrings' IUPAC complement) and collapseNoMismatch(identicalOnly = TRUE) (:104-115), on tables
(mat, colnames, rownames).  Test infrastructure: no product code is used.

merge(...) -> (int32 mat, colnames, rownames, messages) or raises RefError with R's stop() message.  Conventions of the
product that R does not have are restated too: int32 overflow of a cell or column sum is an error, entries are whole
numbers, and column names are upper-case IUPAC."""
import numpy as np

IUPAC = "ACGTMRWSYKVHDBN"
COMP = str.maketrans(IUPAC, "TGCAKYWSRMBDHVN")
INT32_MAX = np.iinfo(np.int32).max


class RefError(Exception):
    pass


def rc(s):
    return s[::-1].translate(COMP)


def is_sequence_table(tab):
    """-> (valid, warnings) in R's order of checks."""
    mat, cols, rows = tab
    mat = np.asarray(mat)
    if mat.ndim != 2:
        return False, ["Not a matrix."]
    if not (mat >= 0).all():
        return False, ["Negative entries."]
    if cols is None or mat.shape[1] == 0:                         # zero-length dimnames are NULL in R
        return False, ["Column (sequence) names are missing."]
    if rows is None or mat.shape[0] == 0:
        return False, ["Row (sample) names are missing."]
    if not all(len(c) > 0 for c in cols):
        return False, ["Some column (sequence) names are blank."]
    if not all(len(r) > 0 for r in rows):
        return False, ["Some row (sample) names are blank."]
    w = []
    if len(set(cols)) < len(cols):
        w.append("Duplicated column (sequences) names.")
    if len(set(rows)) < len(rows):
        w.append("Duplicated row (sample) names.")
    return True, w


def collapse_identical(mat, cols):
    """collapseNoMismatch(seqtab, identicalOnly = TRUE): duplicated columns are added into the first of their name."""
    seen, dupes = set(), []
    for c in cols:
        dupes.append(c in seen)
        seen.add(c)
    if not any(dupes):
        return mat, cols
    keep = [k for k, d in enumerate(dupes) if not d]
    st = mat[:, keep].astype(np.int64)
    st_cols = [cols[k] for k in keep]
    pos = {c: k for k, c in reversed(list(enumerate(st_cols)))}   # st[, sq]: the first column named sq
    for i, d in enumerate(dupes):
        if d:
            st[:, pos[cols[i]]] += mat[:, i]
    return st, st_cols


def assign_colmajor(rval, ri, ci, new):
    """rval[ri, ci] <- new with R's semantics: the cells are written in column-major order, so where several (i, j)
    reach one target the last column, and within it the last row, wins.  Small tables are written cell by cell in that
    order; large ones keep only the last row and column of every name, which is the same set of final writes."""
    ri, ci = np.asarray(ri), np.asarray(ci)
    if len(ri) * len(ci) <= 20000:
        for j in range(len(ci)):
            for i in range(len(ri)):
                rval[ri[i], ci[j]] = new[i, j]
        return
    last_r = np.zeros(len(ri), bool)
    last_r[len(ri) - 1 - np.unique(ri[::-1], return_index=True)[1]] = True
    last_c = np.zeros(len(ci), bool)
    last_c[len(ci) - 1 - np.unique(ci[::-1], return_index=True)[1]] = True
    rval[np.ix_(ri[last_r], ci[last_c])] = new[np.ix_(last_r, last_c)]


def merge(tables, names=None, repeats="error", orderBy="abundance", tryRC=False):
    messages = []
    if len(tables) < 2:
        raise RefError("At least two sequence tables are expected")
    valid = []
    for t in tables:
        ok, w = is_sequence_table(t)
        messages += w
        valid.append(ok)
    if not all(valid):
        em = ", ".join(names[i] for i, v in enumerate(valid) if not v) if names else ""
        raise RefError("Some sequence tables found invalid" + (": " + em if em else ""))
    tables = [(np.asarray(m), list(c), list(r)) for m, c, r in tables]
    for m, _, _ in tables:
        if not np.issubdtype(m.dtype, np.integer) and (m != np.floor(m)).any():
            raise RefError("dada2b: sequence table entries must be whole numbers.")
    sample_names = [r for _, _, rows in tables for r in rows]
    seen, dup = set(), []
    for r in sample_names:
        if r in seen and r not in dup:
            dup.append(r)
        seen.add(r)
    if dup:
        if repeats == "error":
            raise RefError("Duplicated sample names detected in the sequence table row names: " + ", ".join(dup))
        sample_names = list(dict.fromkeys(sample_names))
        messages.append("Duplicated sample names detected in the sequence table row names.")
    seqs = list(dict.fromkeys(c for _, cols, _ in tables for c in cols))
    bad = set("".join(seqs)) - set(IUPAC)                          # the product packs names 4 bits per letter
    if bad:
        raise RefError("dada2b: column (sequence) names must be upper-case IUPAC letters (%s); found '%s'." % (IUPAC, min(bad)))
    if tryRC and len(seqs) > 1:
        earlier, before = [], set()
        for s in seqs:                                             # rc(seqs[[i]]) %in% seqs[1:(i-1)]
            earlier.append(rc(s) in before)
            before.add(s)
        rc_seqs = {s for s, e in zip(seqs, earlier) if e}
        if rc_seqs:
            messages.append("Reverse complemented sequences detected and re-oriented.")
            for i, (m, cols, rows) in enumerate(tables):
                do_rc = [c in rc_seqs for c in cols]
                if any(do_rc):
                    cols = [rc(c) if d else c for c, d in zip(cols, do_rc)]
                    m, cols = collapse_identical(m, cols)
                    tables[i] = (m, cols, rows)
            seqs = [s for s in seqs if s not in rc_seqs]
    rval = np.zeros((len(sample_names), len(seqs)), np.int64)
    rpos = {r: k for k, r in reversed(list(enumerate(sample_names)))}
    cpos = {c: k for k, c in enumerate(seqs)}
    for m, cols, rows in tables:
        ri = [rpos[r] for r in rows]
        ci = [cpos[c] for c in cols]
        new = rval[np.ix_(ri, ci)] + m.astype(np.int64)
        assign_colmajor(rval, ri, ci, new)
    cs = rval.sum(axis=0)
    if rval.size and (rval.max() > INT32_MAX or cs.max() > INT32_MAX):
        raise RefError("dada2b: a merged table entry or column sum exceeds the int32 range (R would return NA).")
    if orderBy is not None:
        o = None
        if orderBy == "abundance":
            o = np.argsort(-cs, kind="stable")
        elif orderBy == "nsamples":
            o = np.argsort(-(rval > 0).sum(axis=0), kind="stable")
        if o is not None:
            rval = rval[:, o]
            seqs = [seqs[k] for k in o]
    return rval.astype(np.int32), seqs, sample_names, messages
