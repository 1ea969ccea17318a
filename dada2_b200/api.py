"""Host-side mirror of the reference's `dada_uniques` entry point for the GPU path.

`dada_uniques(...)` has the reference's name, argument order, meaning and error behaviour
(/root/reference/src/Rmain.cpp:30-47; called from R/dada.R:335-352) and returns a dict shaped
like the R list of Rmain.cpp:294.  All computation happens in libdada2b.so (hand-written
sm_90a CUDA behind the C-ABI of include/dada2b.h); this module only marshals.  There is no
CPU fallback: if the library is missing or no GPU is visible, calls raise.
"""
import ctypes as C
import os

import numpy as np

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.path.join(_HERE, "libdada2b.so")
_LIB = None


class Dada2bError(RuntimeError):
    """Raised where the reference would Rcpp::stop()."""


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_LIBPATH):
            raise Dada2bError("libdada2b.so is not built (run `python -m dada2_b200.build`); "
                              "there is no CPU fallback for the dada() core.")
        L = C.CDLL(_LIBPATH)
        P = C.POINTER
        L.dada2b_run.argtypes = [P(_abi.In), P(_abi.Opts), P(P(_abi.Out)), C.c_char_p]
        L.dada2b_free.argtypes = [P(_abi.Out)]
        L.dada2b_upload.argtypes = [P(_abi.In), C.c_int32, P(C.c_void_p), C.c_char_p]
        L.dada2b_run_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, P(_abi.Opts), P(P(_abi.Out)), C.c_char_p]
        L.dada2b_ctx_free.argtypes = [C.c_void_p]
        L.dada2b_reupload.argtypes = [C.c_void_p, P(_abi.In), C.c_char_p]
        L.dada2b_default_opts.argtypes = [P(_abi.Opts)]
        L.dada2b_nccl_unique_id.argtypes = [C.c_char_p, C.c_char_p]
        L.dada2b_comm_init.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_char_p, C.c_char_p]
        L.dada2b_test_calc_pA.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p]
        L.dada2b_test_pairs.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                        P(_abi.Opts), C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_int32, C.c_char_p]
        L.dada2b_test_loop_nw.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, P(_abi.Opts),
                                          C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p]
        L.dada2b_test_screen.argtypes = [C.c_void_p, C.c_uint32, P(_abi.Opts), C.c_double, C.c_uint32, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p]
        L.dada2b_test_raw_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_char_p]
        L.dada2b_test_bound.argtypes = [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int32, P(_abi.Opts), C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_char_p]
        _LIB = L
    return _LIB


def _check_err(err):
    e = np.asarray(err, dtype=np.float64)
    if e.ndim != 2 or e.shape[0] != 16:
        raise Dada2bError("Error matrix must have 16 rows.")          # Rmain.cpp:75-77
    return e


def _normalise_opts(kw):
    if kw.get("homo_gap") is None:
        kw["homo_gap"] = kw.get("gap", _abi.DEFAULT_OPTS["gap"])      # R/dada.R:224-226
    return kw


class Resident:
    """Uniques uploaded and packed once on the device; run() can then be called repeatedly with
    different error matrices / options (selfConsist loop, R/dada.R:256-391)."""

    def __init__(self, seqs, abundances, priors, quals, device=0):
        L = lib()
        if len(seqs) == 0:
            raise Dada2bError("Zero input sequences.")                 # Rmain.cpp:55
        self.nraw = len(seqs)
        try:
            self._pin = _abi.PackedIn(seqs, abundances, priors, None, quals)
        except ValueError as e:
            raise Dada2bError(str(e))
        self._ctx = C.c_void_p()
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = L.dada2b_upload(C.byref(self._pin.struct), int(device), C.byref(self._ctx), eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        self._pin = None  # host buffers are copied by the library

    def reupload(self, packed_in):
        """Replace this context's uniques from host buffers (`_abi.PackedIn`); keeps buffers and communicator."""
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = lib().dada2b_reupload(self._ctx, C.byref(packed_in.struct), eb)
        if rc:
            raise Dada2bError(eb.value.decode())

    def run_raw(self, ecm, Q, opts_struct):
        """run() without Python-side marshalling of the result (stats only) -- for timing."""
        L = lib()
        out = C.POINTER(_abi.Out)()
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = L.dada2b_run_resident(self._ctx, ecm.ctypes.data, int(Q), C.byref(opts_struct), C.byref(out), eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        try:
            return {k: getattr(out.contents, k) for k in _abi.STAT_FIELDS}
        finally:
            L.dada2b_free(out)

    def comm_init(self, rank, world, unique_id):
        """Join a sharded multi-GPU run (one process per GPU): raw r is aligned by rank r % world, one NCCL
        all-gather per split round.  `unique_id` comes from nccl_unique_id() on rank 0."""
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = lib().dada2b_comm_init(self._ctx, int(rank), int(world), bytes(unique_id), eb)
        if rc:
            raise Dada2bError(eb.value.decode())

    def run(self, err, **opts):
        L = lib()
        e = _check_err(err)
        ecm = np.asfortranarray(e)
        o = _abi.make_opts(**_normalise_opts(dict(opts)))
        out = C.POINTER(_abi.Out)()
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = L.dada2b_run_resident(self._ctx, ecm.ctypes.data, int(e.shape[1]), C.byref(o), C.byref(out), eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        try:
            return _abi.unpack_out(out.contents)
        finally:
            L.dada2b_free(out)

    def test_pairs(self, centre, raw, err, use_kmers=True, kdist_cutoff=0.42, opcap=None, subcap=None, maxlen=None, **opts):
        """Kernel-level hook (include/dada2b_test.h): classify + align the given index pairs."""
        L = lib()
        e = _check_err(err)
        ecm = np.asfortranarray(e)
        o = _abi.make_opts(**_normalise_opts(dict(opts)))
        centre = np.ascontiguousarray(centre, dtype=np.uint32)
        raw = np.ascontiguousarray(raw, dtype=np.uint32)
        n = len(centre)
        opcap = int(opcap or 2 * maxlen)
        subcap = int(subcap or maxlen)
        kind = np.zeros(n, np.int32); lam = np.zeros(n, np.float64); nsubs = np.zeros(n, np.int32)
        ops = np.zeros((n, opcap), np.uint8); nops = np.zeros(n, np.int32)
        pos = np.zeros((n, subcap), np.uint16); nt0 = np.zeros((n, subcap), np.uint8)
        nt1 = np.zeros((n, subcap), np.uint8); q1 = np.zeros((n, subcap), np.uint8)
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = L.dada2b_test_pairs(self._ctx, n, centre.ctypes.data, raw.ctypes.data, ecm.ctypes.data, int(e.shape[1]),
                                 C.byref(o), int(use_kmers), float(kdist_cutoff), kind.ctypes.data, lam.ctypes.data,
                                 nsubs.ctypes.data, ops.ctypes.data, nops.ctypes.data, opcap, pos.ctypes.data,
                                 nt0.ctypes.data, nt1.ctypes.data, q1.ctypes.data, subcap, eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        return dict(kind=kind, lam=lam, nsubs=nsubs, ops=ops, nops=nops, pos=pos, nt0=nt0, nt1=nt1, q1=q1)

    def test_loop_nw(self, which, centre, raw, err, njobs_hint=1, **opts):
        """Kernel-level hook (include/dada2b_test.h): each (centre, raw) pair alone through one loop aligner
        (0 k_nwrow<EXACT>, 1 k_nwlane, 2 k_nwfwd, 3 k_nwrow<BOUND>) -> lambda, nsubs, handled.  njobs_hint: the round size
        k_nwfwd picks its instantiation from (1: the small-round choice; above num_sms * 512 the G = 4 / ND = 10 kernel)."""
        e = _check_err(err)
        ecm = np.asfortranarray(e)
        o = _abi.make_opts(**_normalise_opts(dict(opts)))
        centre = np.ascontiguousarray(centre, dtype=np.uint32)
        raw = np.ascontiguousarray(raw, dtype=np.uint32)
        n = len(centre)
        lam = np.zeros(n, np.float64); nsubs = np.zeros(n, np.int32); handled = np.zeros(n, np.int32)
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = lib().dada2b_test_loop_nw(self._ctx, int(which), n, centre.ctypes.data, raw.ctypes.data, ecm.ctypes.data, int(e.shape[1]),
                                       C.byref(o), int(njobs_hint), lam.ctypes.data, nsubs.ctypes.data, handled.ctypes.data, eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        return dict(lam=lam, nsubs=nsubs, handled=handled)

    def test_screen(self, centre, kdist_cutoff=0.42, centre_reads=None, lock=None, rank=0, world=1, max_sms=0, path=0, **opts):
        """Kernel-level hook (include/dada2b_test.h): one round's k-mer screen of `centre` against the raws of shard (rank, world)
        -> kind (-1 other rank, 0 shrouded or skipped, 1 gapless, 2 NW), minsum (k_prescreen's, 0xFFFF overflowed, -1 no
        candidate), counters {align, shroud, gapless, nw}.  `greedy` goes in with the other options; centre_reads defaults to 0."""
        o = _abi.make_opts(**_normalise_opts(dict(opts)))
        n = self.nraw
        lk = None
        if lock is not None:
            lk = np.ascontiguousarray(lock, dtype=np.uint8)
            if len(lk) != n:
                raise ValueError("lock needs one entry per raw")
        kind = np.zeros(n, np.int32); minsum = np.zeros(n, np.int32); ctr = np.zeros(4, np.int64)
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = lib().dada2b_test_screen(self._ctx, int(centre), C.byref(o), float(kdist_cutoff), int(centre_reads or 0),
                                      lk.ctypes.data if lk is not None else None, int(rank), int(world), int(max_sms), int(path),
                                      kind.ctypes.data, minsum.ctypes.data, ctr.ctypes.data, eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        return dict(kind=kind, minsum=minsum, counters=dict(zip(("align", "shroud", "gapless", "nw"), ctr.tolist())))

    def test_raw_bounds(self, err, use_quals=True, rank=0, world=1):
        """Kernel-level hook (include/dada2b_test.h): k_raw_bounds' per-raw factors (S, rho) of the two-phase bound for the raws
        of shard (rank, world); NaN for the other raws."""
        e = _check_err(err)
        ecm = np.asfortranarray(e)
        S = np.zeros(self.nraw, np.float64); rho = np.zeros(self.nraw, np.float64)
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = lib().dada2b_test_raw_bounds(self._ctx, ecm.ctypes.data, int(e.shape[1]), int(bool(use_quals)), int(rank), int(world),
                                          S.ctypes.data, rho.ctypes.data, eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        return S, rho

    def test_bound(self, which, centre, cluster_i, jobs, e_minmax, err, njobs_hint=0, **opts):
        """Kernel-level hook (include/dada2b_test.h): one launch of a bound-testing loop kernel (0 k_nwrow<BOUND>, 1 k_nwlane,
        2 k_nwfwd's bound pass, 3 k_gapless_loop) over the job list -> outcome per job (0 dropped, 1 survivor list, 2 gapless
        list, 3 handed back, 4 stored, 5 passed the bound, not stored), nsubs, lambda (stored lambda, NaN otherwise), e_after
        (E_minmax after the launch) and counters {surv, gapless, back, stored}."""
        e = _check_err(err)
        ecm = np.asfortranarray(e)
        o = _abi.make_opts(**_normalise_opts(dict(opts)))
        jobs = np.ascontiguousarray(jobs, dtype=np.uint32)
        em = np.ascontiguousarray(e_minmax, dtype=np.float64)
        if len(em) != self.nraw:
            raise ValueError("e_minmax needs one entry per raw")
        n = len(jobs)
        outcome = np.zeros(n, np.int32); nsubs = np.zeros(n, np.int32); lam = np.zeros(n, np.float64)
        e_after = np.zeros(self.nraw, np.float64); ctr = np.zeros(4, np.int64)
        eb = C.create_string_buffer(_abi.ERRLEN)
        rc = lib().dada2b_test_bound(self._ctx, int(which), int(centre), int(cluster_i), n, jobs.ctypes.data, em.ctypes.data, ecm.ctypes.data,
                                     int(e.shape[1]), C.byref(o), int(njobs_hint), outcome.ctypes.data, nsubs.ctypes.data, lam.ctypes.data,
                                     e_after.ctypes.data, ctr.ctypes.data, eb)
        if rc:
            raise Dada2bError(eb.value.decode())
        return dict(outcome=outcome, nsubs=nsubs, lam=lam, e_after=e_after,
                    counters=dict(zip(("surv", "gapless", "back", "stored"), ctr.tolist())))

    def close(self):
        if getattr(self, "_ctx", None) and self._ctx.value:
            lib().dada2b_ctx_free(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def dada_uniques(seqs, abundances, priors, err, quals,
                 match=5, mismatch=-4, gap=-8, use_kmers=True, kdist_cutoff=0.42, band_size=16,
                 omegaA=1e-40, omegaP=1e-4, omegaC=1e-40, detect_singletons=False, max_clust=0,
                 min_fold=1.0, min_hamming=1, min_abund=1, use_quals=True, final_consensus=False,
                 vectorized_alignment=True, homo_gap=None, multithread=True, verbose=False, SSE=2,
                 gapless=True, greedy=True):
    """Drop-in for the reference's dada_uniques (same positional order as Rmain.cpp:30-47).

    seqs: list of A/C/G/T strings; abundances: ints; priors: bools or None; err: [16, Q] float64;
    quals: [nraw, maxlen] float64 per-position mean qualities (NaN beyond a read's length), i.e.
    `derep$quals`; returns {"clustering", "birth_subs", "subqual", "clusterquals", "map", "pval"}.
    One-shot path through dada2b_run(): host buffers in, host buffers out.
    """
    L = lib()
    e = _check_err(err)
    if len(seqs) == 0:
        raise Dada2bError("Zero input sequences.")
    try:
        pin = _abi.PackedIn(seqs, abundances, priors, e, quals)
    except ValueError as ex:
        raise Dada2bError(str(ex))
    o = _abi.make_opts(**_normalise_opts(dict(
        match=match, mismatch=mismatch, gap=gap, use_kmers=use_kmers, kdist_cutoff=kdist_cutoff, band_size=band_size,
        omegaA=omegaA, omegaP=omegaP, omegaC=omegaC, detect_singletons=detect_singletons, max_clust=max_clust,
        min_fold=min_fold, min_hamming=min_hamming, min_abund=min_abund, use_quals=use_quals,
        final_consensus=final_consensus, vectorized_alignment=vectorized_alignment, homo_gap=homo_gap,
        multithread=multithread, verbose=verbose, SSE=SSE, gapless=gapless, greedy=greedy)))
    out = C.POINTER(_abi.Out)()
    eb = C.create_string_buffer(_abi.ERRLEN)
    rc = L.dada2b_run(C.byref(pin.struct), C.byref(o), C.byref(out), eb)
    if rc:
        raise Dada2bError(eb.value.decode())
    try:
        return _abi.unpack_out(out.contents)
    finally:
        L.dada2b_free(out)


def nccl_unique_id():
    buf = C.create_string_buffer(128)
    eb = C.create_string_buffer(_abi.ERRLEN)
    if lib().dada2b_nccl_unique_id(buf, eb):
        raise Dada2bError(eb.value.decode())
    return buf.raw


class PackedCall:
    """Pre-marshalled one-shot call: `run()` is exactly one dada2b_run() C-ABI call on host buffers
    (what the Rcpp shim of INTEGRATION.md does), so benchmarks can time the ABI without Python's
    string joining."""

    def __init__(self, seqs, abundances, priors, err, quals, **opts):
        self.err = _check_err(err)
        self.pin = _abi.PackedIn(seqs, abundances, priors, self.err, quals)
        self.opts = _abi.make_opts(**_normalise_opts(dict(opts)))

    def run(self, unpack=True):
        import time
        L = lib()
        out = C.POINTER(_abi.Out)()
        eb = C.create_string_buffer(_abi.ERRLEN)
        t0 = time.perf_counter()
        rc = L.dada2b_run(C.byref(self.pin.struct), C.byref(self.opts), C.byref(out), eb)
        wall_ms = (time.perf_counter() - t0) * 1e3
        if rc:
            raise Dada2bError(eb.value.decode())
        try:
            res = _abi.unpack_out(out.contents) if unpack else {"stats": {k: getattr(out.contents, k) for k in _abi.STAT_FIELDS}}
        finally:
            L.dada2b_free(out)
        return res, wall_ms


def test_calc_pA(reads, E, prior):
    L = lib()
    reads = np.ascontiguousarray(reads, dtype=np.int32)
    E = np.ascontiguousarray(E, dtype=np.float64)
    prior = np.ascontiguousarray(prior, dtype=np.int32)
    out = np.zeros(len(reads), np.float64)
    eb = C.create_string_buffer(_abi.ERRLEN)
    rc = L.dada2b_test_calc_pA(len(reads), reads.ctypes.data, E.ctypes.data, prior.ctypes.data, out.ctypes.data, eb)
    if rc:
        raise Dada2bError(eb.value.decode())
    return out
