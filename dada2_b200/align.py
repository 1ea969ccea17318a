"""nwalign (R/misc.R:179-191) batched over pairs of sequences.

The alignments run in libdada2b.so behind include/dada2b_align.h: one warp per pair on the GPU, in every mode of the
reference (ends-free, ends-free with homopolymer gap costs, global, and the vectorized aligner with either end rule).
This module restates R's argument rules and marshals.  No CPU fallback.
"""
import ctypes as C
import sys

import numpy as np

from . import api
from .bimera import _pack_seqs

ERRLEN = 256
_ACGT = frozenset("ACGT")


class NwalignOpts(C.Structure):
    _fields_ = [("match", C.c_int32), ("mismatch", C.c_int32), ("gap_p", C.c_int32), ("homo_gap_p", C.c_int32), ("band", C.c_int32),
                ("endsfree", C.c_int32), ("vec", C.c_int32)]


class NwalignStats(C.Structure):
    _fields_ = [("n_pairs", C.c_int64), ("n_cells", C.c_int64), ("n_blocks", C.c_int64), ("gpu_launches", C.c_int64),
                ("ms_device", C.c_double), ("ms_k_align", C.c_double), ("ms_total", C.c_double)]


_BOUND = None             # the library object the argtypes were set on (a test may swap api's library)


def _lib():
    global _BOUND
    L = api.lib()
    if _BOUND is not L:
        P = C.POINTER
        L.dada2b_nwalign_default_opts.argtypes = [P(NwalignOpts)]
        L.dada2b_nwalign.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, P(NwalignOpts), C.c_int32,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, P(NwalignStats), C.c_char_p]
        _BOUND = L
    return L


def _pairs(s1, s2, what):
    """R's recycling of a length-one side (Vectorize / C_nwvec's vectors): -> (list, list, scalar call)."""
    one = isinstance(s1, str) and isinstance(s2, str)
    a = [s1] if isinstance(s1, str) else list(s1)
    b = [s2] if isinstance(s2, str) else list(s2)
    if not all(isinstance(s, str) for s in a + b):
        raise api.Dada2bError("Can only align character sequences.")                                  # R/misc.R:180
    if len(a) == 1 and len(b) > 1:
        a = a * len(b)
    if len(b) == 1 and len(a) > 1:
        b = b * len(a)
    if len(a) != len(b):
        raise api.Dada2bError("dada2b: %s needs pairs of sequences." % what)
    return a, b, one


def _rules(a, b, gap, homo_gap, endsfree, vec):
    """R/misc.R:180-190 and evaluate.cpp:36-47 for one call over the pairs (a, b): -> the homopolymer gap to align with."""
    if homo_gap is None:
        homo_gap = gap
    if vec:
        if homo_gap != gap:
            raise api.Dada2bError("Homopolymer gap penalties are not implemented in the vectorized aligner.")   # :183
        if not all(_ACGT.issuperset(s) for s in a + b):
            raise api.Dada2bError("dada2b: the vectorized aligner here needs A/C/G/T sequences (2-bit packed on the device).")
    elif not all(_ACGT.issuperset(s) for s in a + b):
        raise api.Dada2bError("Sequences must contain only A/C/G/T characters.")                      # :187 (C_isACGT)
    if not vec and not endsfree and homo_gap != gap:
        # evaluate.cpp:49-51 prints this for every pair; one call prints it once
        print("Warning: A separate homopolymer gap penalty isn't implemented when endsfree=FALSE.\n\tAll gaps will be penalized by "
              "the regular gap penalty.", file=sys.stderr)
        homo_gap = gap
    return homo_gap


def align_pairs(a, b, match=5, mismatch=-4, gap=-8, homo_gap=None, band=-1, endsfree=True, vec=False, rows=True, counts=False,
                device=0, return_stats=False):
    """The device call for equal-length lists a, b of non-empty A/C/G/T sequences.  -> dict with "al1", "al2" (lists of
    str) when rows, "counts" (int32[n, 3]: C_eval_pair's match, mismatch, indel) when counts; "stats" with return_stats."""
    n = len(a)
    hg = gap if homo_gap is None else homo_gap
    uniq, idx = {}, np.zeros(2 * n, np.int32)
    for k, s in enumerate(a + b):
        idx[k] = uniq.setdefault(s, len(uniq))
    seqs = list(uniq)
    buf, off = _pack_seqs(seqs)
    s1, s2 = np.ascontiguousarray(idx[:n]), np.ascontiguousarray(idx[n:])
    o = NwalignOpts(int(match), int(mismatch), int(gap), int(hg), int(band), int(bool(endsfree)), int(bool(vec)))
    slot = np.fromiter((len(x) + len(y) for x, y in zip(a, b)), np.int64, count=n)
    sl_off = np.zeros(n + 1, np.int64)
    np.cumsum(slot, out=sl_off[1:])
    tot = int(sl_off[-1])
    r1 = np.zeros(max(tot, 1), np.uint8) if rows else None
    r2 = np.zeros(max(tot, 1), np.uint8) if rows else None
    al_len = np.zeros(max(n, 1), np.int32) if rows else None
    cnt = np.zeros((max(n, 1), 3), np.int32) if counts else None
    st = NwalignStats()
    eb = C.create_string_buffer(ERRLEN)
    ptr = lambda v: v.ctypes.data if v is not None else None                                             # noqa: E731
    rc = _lib().dada2b_nwalign(len(seqs), buf, off.ctypes.data, n, s1.ctypes.data, s2.ctypes.data, C.byref(o), int(device),
                               ptr(r1), ptr(r2), ptr(al_len), ptr(cnt), C.byref(st), eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    out = {}
    if rows:
        b1, b2 = r1.tobytes(), r2.tobytes()
        out["al1"] = [b1[sl_off[x]:sl_off[x] + al_len[x]].decode() for x in range(n)]
        out["al2"] = [b2[sl_off[x]:sl_off[x] + al_len[x]].decode() for x in range(n)]
    if counts:
        out["counts"] = cnt[:n]
    if return_stats:
        out["stats"] = {k: getattr(st, k) for k, _ in NwalignStats._fields_}
    return out


def nwalign(s1, s2, match=5, mismatch=-4, gap=-8, homo_gap=None, band=-1, endsfree=True, vec=False, device=0):
    """R/misc.R:179-191 on the GPU.  s1, s2: strings, or lists of strings (a one-element side is recycled).
    -> (al1, al2) for two strings, else a list of such tuples ([] for zero pairs).

    vec=False aligns with C_nwalign (evaluate.cpp:18-61): nwalign_endsfree, nwalign_endsfree_homo when homo_gap differs
    from gap, or the global nwalign with endsfree=False (which ignores homo_gap after R's warning).  vec=True aligns with
    nwalign_vectorized2 (C_nwvec) and is refused where the reference's int16 scores could overflow, and for sequences that
    are not A/C/G/T (the reference would compare raw characters there)."""
    a, b, one = _pairs(s1, s2, "nwalign")
    homo_gap = _rules(a, b, gap, homo_gap, endsfree, vec)
    out = [None] * len(a)
    work = []
    for x, (p, q) in enumerate(zip(a, b)):
        if p and q:
            work.append(x)
        else:                               # a zero-length side: the traceback walks the other along row or column 0
            out[x] = ("-" * len(q) + p, q + "-" * len(p))
    if work:
        r = align_pairs([a[x] for x in work], [b[x] for x in work], match, mismatch, gap, homo_gap, band, endsfree, vec, device=device)
        for k, x in enumerate(work):
            out[x] = (r["al1"][k], r["al2"][k])
    return out[0] if one else out


def eval_counts(a, b, match=5, mismatch=-4, gap=-8, homo_gap=None, band=-1, endsfree=True, vec=False, device=0):
    """nwalign then C_eval_pair for equal-length lists of sequences, under nwalign's rules: -> int32[n, 3] (match,
    mismatch, indel).  A pair with an empty side has no internal part: (0, 0, 0)."""
    homo_gap = _rules(a, b, gap, homo_gap, endsfree, vec)
    kw = dict(match=match, mismatch=mismatch, gap=gap, homo_gap=homo_gap, band=band, endsfree=endsfree, vec=vec)
    n = len(a)
    cnt = np.zeros((n, 3), np.int32)
    work = [x for x in range(n) if a[x] and b[x]]
    if work:
        cnt[work] = align_pairs([a[x] for x in work], [b[x] for x in work], rows=False, counts=True, device=device, **kw)["counts"]
    return cnt
