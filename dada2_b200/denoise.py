"""dada() over samples and learnErrors() over files: the R around dada_uniques (R/dada.R:144-488, R/errorModels.R:333-363).

Every dada_uniques pass runs in libdada2b.so; pooling (pool = TRUE) runs there too (dada2_b200.derep.pool_dereps,
include/dada2b_pool.h) and leaves the pooled uniques resident on the device, so every pass of the selfConsist loop is one
run() on that context.  This module restates the R line by line: options, validation, the err extension, the loop
(errmodel.consist_loop), the pseudo-pooling pass, the expansion of a pooled result into per-sample objects and the
return value.  A result is one dict per sample with dada_uniques' keys plus denoised, sequence, quality, trans, err_in,
err_out and opts, as R's dada-class object.  Not restated: verbose text, directory inputs and qualityType detection;
USE_QUALS = FALSE is refused.
"""
import math
import os
import warnings

import numpy as np

from . import api, errmodel
from .errmodel import loessErrfun

NA_INT = np.iinfo(np.int32).min

# R/dada.R:1-26
DADA_OPTS = dict(OMEGA_A=1e-40, OMEGA_P=1e-4, OMEGA_C=1e-40, DETECT_SINGLETONS=False, USE_KMERS=True, KDIST_CUTOFF=0.42,
                 MAX_CONSIST=10, MATCH=5, MISMATCH=-4, GAP_PENALTY=-8, BAND_SIZE=16, VECTORIZED_ALIGNMENT=True, MAX_CLUST=0,
                 MIN_FOLD=1, MIN_HAMMING=1, MIN_ABUNDANCE=1, USE_QUALS=True, HOMOPOLYMER_GAP_PENALTY=None, SSE=2, GAPLESS=True,
                 GREEDY=True, PSEUDO_PREVALENCE=2, PSEUDO_ABUNDANCE=math.inf)


def extend_err(err, qmax):
    """R/dada.R:303-313: repeat the last column until the matrix reaches quality score qmax."""
    err = np.asarray(err, dtype=np.float64)
    if err.shape[1] >= qmax + 1:
        return err
    return np.concatenate([err, np.repeat(err[:, -1:], qmax + 1 - err.shape[1], axis=1)], axis=1)


def initial_err(qmax):
    """initializeErr's matrix (R/dada.R:298): all ones, 16 x max(41, qmax + 1)."""
    return np.ones((16, max(41, qmax + 1)))


def _uniques_opts(o, max_clust, multithread):
    """dada()'s options -> dada_uniques' arguments (R/dada.R:335-352)."""
    return dict(match=o["MATCH"], mismatch=o["MISMATCH"], gap=o["GAP_PENALTY"], use_kmers=o["USE_KMERS"], kdist_cutoff=o["KDIST_CUTOFF"],
                band_size=o["BAND_SIZE"], omegaA=o["OMEGA_A"], omegaP=o["OMEGA_P"], omegaC=o["OMEGA_C"],
                detect_singletons=o["DETECT_SINGLETONS"], max_clust=max_clust, min_fold=o["MIN_FOLD"], min_hamming=o["MIN_HAMMING"],
                min_abund=o["MIN_ABUNDANCE"], use_quals=True, final_consensus=False, vectorized_alignment=o["VECTORIZED_ALIGNMENT"],
                homo_gap=o["HOMOPOLYMER_GAP_PENALTY"], multithread=bool(multithread), verbose=False, SSE=o["SSE"],
                gapless=o["GAPLESS"], greedy=o["GREEDY"])


def _validate(d):
    """Per-sample validation (R/dada.R:267-292) -> the largest mean quality (qmax is checked on its ceiling by _qmax)."""
    u = d["uniques"]
    if set("".join(u)) - set("ACGT"):
        raise ValueError("Invalid derep$uniques vector. Sequences must be made up only of A/C/G/T.")
    if d.get("quals") is None:
        raise ValueError("The input derep-class object(s) must include quals if USE_QUALS is TRUE.")
    q = np.asarray(d["quals"], dtype=np.float64)
    if q.ndim != 2 or q.shape[0] != len(u):
        raise ValueError("derep$quals matrices must have one row for each derep$unique sequence.")
    lens = np.fromiter((len(s) for s in u), dtype=np.int64, count=len(u))
    if len(u) and lens.max() > q.shape[1]:
        raise ValueError("derep$quals matrices must have as many columns as the length of the derep$unique sequences.")
    if np.isnan(q[np.arange(q.shape[1])[None, :] < lens[:, None]]).any():
        raise ValueError("NAs in derep$quals matrix. Check that all input sequences had valid associated qualities assigned.")
    if np.nanmin(q) < 0:
        raise ValueError("Invalid derep$quals matrix. Quality values must be positive integers.")
    return np.nanmax(q)


def _qmax(mx, i):
    qmax = int(math.ceil(mx))
    if qmax > 250:
        raise ValueError("Sample %d has an invalid maximum Phred Quality Scores of %d" % (i, qmax))
    return qmax


def _sample_inputs(derep, device):
    """-> (list of derep dicts, names or None, shape of the return value: 'one', 'list' or 'dict')."""
    from .derep import derepFastq
    if isinstance(derep, dict) and "uniques" in derep:
        return [derep], None, "one"
    if isinstance(derep, (str, os.PathLike)):
        derep, shape = [derep], "one"
    elif isinstance(derep, dict):
        names, vals = list(derep.keys()), list(derep.values())
        ds, _, _ = _sample_inputs(vals, device)
        return ds, names, "dict"
    elif isinstance(derep, (list, tuple)):
        shape = "list"
    else:
        shape = None
    ok = shape is not None and len(derep) > 0 and (all(isinstance(d, dict) and "uniques" in d for d in derep)
                                                   or all(isinstance(d, (str, os.PathLike)) for d in derep))
    if not ok:
        raise ValueError("The derep argument must be derep-class object, list of derep-class objects, or a character vector of "
                         "fastq files or a directory containing fastq files.")
    if isinstance(derep[0], dict):
        return list(derep), None, shape
    if not all(os.path.exists(f) for f in derep):
        raise ValueError("Some of the filenames provided do not exist. This may have happened because some samples had zero "
                         "reads after filtering.")
    return [derepFastq(f, device=device) for f in derep], [os.path.basename(str(f)) for f in derep], shape


def _denoised(res):
    cl = res["clustering"]
    return dict(zip(cl["sequence"], (int(a) for a in cl["abundance"])))


def _expand_pooled(pres, pooled_index, ab, nclust):
    """R/dada.R:443-475 for one sample: pres = the pooled dada result object, pooled_index = 1-based pooled position of
    each of the sample's uniques, ab = their abundances in the sample."""
    pmap = np.asarray(pres["map"])
    mi = pmap[pooled_index - 1]                                   # map[names(derep.in[[i]]$uniques)]
    ok = mi != NA_INT
    keep = np.zeros(nclust, bool)
    keep[mi[ok] - 1] = True                                       # unique(map[... %in% ...]); NA drops out of %in%
    newBi = np.cumsum(keep).astype(np.int32)
    out = dict(pres)
    cl = {k: ([v for v, kk in zip(col, keep) if kk] if isinstance(col, list) else np.asarray(col)[keep])
          for k, col in pres["clustering"].items()}
    bs = pres["birth_subs"]
    bclust = np.asarray(bs["clust"], dtype=np.int64)
    sel = keep[bclust - 1] if len(bclust) else np.zeros(0, bool)
    out["birth_subs"] = {k: ([v for v, kk in zip(col, sel) if kk] if isinstance(col, list) else np.asarray(col)[sel])
                         for k, col in bs.items()}
    out["birth_subs"]["clust"] = newBi[bclust[sel] - 1]
    m = np.full(len(mi), NA_INT, np.int32)
    m[ok] = newBi[mi[ok] - 1]
    out["map"] = m
    dn = np.bincount(m[ok] - 1, weights=np.asarray(ab, np.float64)[ok], minlength=int(keep.sum())).astype(np.int32)
    cl["abundance"] = dn                                         # tapply(derep.in[[i]]$uniques, map, sum)
    out["clustering"] = cl
    out["sequence"] = cl["sequence"]
    out["denoised"] = dict(zip(cl["sequence"], dn.tolist()))
    out["quality"] = np.asarray(pres["quality"])[keep]
    out["clusterquals"] = out["quality"].T.copy()
    return out


def dada(derep, err=None, errorEstimationFunction=loessErrfun, selfConsist=False, pool=False, priors=(), multithread=False,
         verbose=True, device=0, **opts):
    """dada() (R/dada.R:144-488).  derep: a derep dict, a list of them, a dict name -> derep, or fastq path(s) (dereplicated
    once).  pool: False, True (pooled on the device) or "pseudo".  priors: sequences.  Options take R's names
    (OMEGA_A, BAND_SIZE, MAX_CONSIST, PSEUDO_PREVALENCE, ...).  -> one dada-class dict per sample: a dict for one derep,
    a list for a list, a dict for a dict."""
    o = dict(DADA_OPTS)
    for k, v in opts.items():
        if k in o:
            o[k] = v
        else:
            warnings.warn("%s is not a valid DADA option." % k)
    dereps, names, shape = _sample_inputs(derep, device)
    priors = set(priors)
    pseudo = False
    if len(dereps) <= 1:
        pool = False
    if pool is True:
        pooled = True
    elif pool is False:
        pooled = False
    elif pool == "pseudo":
        pooled, pseudo = False, True
    else:
        raise ValueError("Invalid pool argument.")
    initializeErr = selfConsist and err is None
    if not initializeErr:
        err = errmodel.getErrors_enforce(err)
    if o["OMEGA_A"] < 0 or o["OMEGA_A"] >= 1:
        raise ValueError("OMEGA_A must be between zero and one.")
    if o["OMEGA_P"] < 0 or o["OMEGA_P"] >= 1:
        raise ValueError("OMEGA_P must be between zero and one.")
    if o["OMEGA_P"] < o["OMEGA_A"] and len(priors) > 0:
        warnings.warn("OMEGA_P should generally be larger than OMEGA_A.")
    if o["OMEGA_C"] > 1e-10 and selfConsist:
        warnings.warn("Strict error correction (OMEGA_C < 1e-10) is not recommended when learning error rates.")
    if o["OMEGA_C"] >= 1 and selfConsist:
        raise ValueError("Some error correction required when learning error rates.")
    if not o["USE_QUALS"]:
        raise ValueError("USE_QUALS = FALSE is not supported (noqualErrfun is not restated).")
    if not callable(errorEstimationFunction):
        raise ValueError("Must provide a function for errorEstimationFunction.")
    if o["GAP_PENALTY"] > 0:
        o["GAP_PENALTY"] = -o["GAP_PENALTY"]
    if o["HOMOPOLYMER_GAP_PENALTY"] is None:
        o["HOMOPOLYMER_GAP_PENALTY"] = o["GAP_PENALTY"]
    if o["HOMOPOLYMER_GAP_PENALTY"] > 0:
        o["HOMOPOLYMER_GAP_PENALTY"] = -o["HOMOPOLYMER_GAP_PENALTY"]
    if o["HOMOPOLYMER_GAP_PENALTY"] != o["GAP_PENALTY"]:
        o["VECTORIZED_ALIGNMENT"] = False
    if o["VECTORIZED_ALIGNMENT"] and o["BAND_SIZE"] == 0:
        o["VECTORIZED_ALIGNMENT"] = False

    state = {"pseudo": set()}

    def runner(run_fn, qmax):
        def run(e, mc):
            if e is None and mc != 1:
                raise ValueError("Error matrix is NULL.")
            erri = initial_err(qmax) if e is None else extend_err(e, qmax)
            return run_fn(erri, _uniques_opts(o, 1 if mc == 1 else o["MAX_CLUST"], multithread))
        return run

    if pooled:
        from .derep import pool_dereps
        for d in dereps:                                          # the pooled derep fails these exactly when a sample does
            _validate(d)
        pr = [np.fromiter((s in priors for s in d["uniques"]), bool, len(d["uniques"])) for d in dereps]
        pd, rs = pool_dereps(dereps, want_quals=False, device=device, priors=pr, resident=True)
        runners = [runner(lambda e, kw: rs.run(e, **kw), _qmax(pd["qmax"], 1))]
    else:
        runners = []
        for i, d in enumerate(dereps):
            qmax = _qmax(_validate(d), i + 1)

            def run_i(e, kw, d=d):
                pri = [s in priors or s in state["pseudo"] for s in d["uniques"]]
                return api.dada_uniques(d["uniques"], d["abundances"], pri, e, d["quals"], **kw)
            runners.append(runner(run_i, qmax))

    def pseudo_priors(results):
        from .seqtab import makeSequenceTable
        mat, cols, _ = makeSequenceTable([{"clustering": r["clustering"]} for r in results])
        sel = ((mat > 0).sum(axis=0) >= o["PSEUDO_PREVALENCE"]) | (mat.sum(axis=0) >= o["PSEUDO_ABUNDANCE"])
        state["pseudo"] = {c for c, k in zip(cols, sel) if k}

    try:
        results, err_out, errs, npass = errmodel.consist_loop(
            runners, err=None if initializeErr else err, errorEstimationFunction=errorEstimationFunction, MAX_CONSIST=o["MAX_CONSIST"],
            selfConsist=selfConsist, verbose=verbose, pseudo=pseudo_priors if pseudo else None)
    finally:
        if pooled:
            rs.close()
    rvals = []
    for res in results:
        r = dict(res)
        r["denoised"] = _denoised(res)
        r["sequence"] = list(res["clustering"]["sequence"])
        r["quality"] = np.asarray(res["clusterquals"]).T.copy()
        r["trans"] = res["subqual"]
        r["err_in"] = errs if selfConsist else errs[0]
        r["err_out"] = err_out
        r["opts"] = dict(o)
        r["passes"] = npass
        if pseudo:
            r["pseudo_priors"] = sorted(state["pseudo"])
        rvals.append(r)
    if pooled:
        pres = rvals[0]
        nclust = len(pres["sequence"])
        rvals, k0 = [], 0
        for d in dereps:
            k1 = k0 + len(d["uniques"])
            rvals.append(_expand_pooled(pres, pd["index"][k0:k1], d["abundances"], nclust))
            k0 = k1
    if shape == "one":
        return rvals[0]
    if shape == "dict":
        return dict(zip(names, rvals))
    return rvals


def getErrors_detailed(dds):
    """getErrors(dds, detailed = TRUE) (R/errorModels.R:390-423) for what dada() returns."""
    if isinstance(dds, dict) and "err_out" in dds:
        return {"err_out": dds["err_out"], "err_in": dds["err_in"], "trans": dds["trans"]}
    objs = list(dds.values()) if isinstance(dds, dict) else list(dds)
    if not all(np.array_equal(x["err_out"], objs[0]["err_out"]) for x in objs):
        raise ValueError("If list of dada-class objects provided, all must have the same output error rates.")
    return {"err_out": objs[0]["err_out"], "err_in": objs[0]["err_in"], "trans": errmodel.accumulateTrans([x["trans"] for x in objs])}


def learnErrors(fls, nbases=1e8, errorEstimationFunction=loessErrfun, randomize=False, MAX_CONSIST=10, OMEGA_C=0, verbose=False,
                device=0, seed=None, **opts):
    """learnErrors (R/errorModels.R:333-363): dereplicate samples (fastq paths, or take derep dicts as they are) until more
    than nbases bases have been read, then dada(selfConsist = TRUE) on them -> getErrors(detailed = TRUE): err_out, err_in
    and trans accumulated over the samples used (plus `nsamples`).  randomize shuffles the samples with numpy's generator
    (seeded by `seed`); R's sample() stream cannot be reproduced, so a randomized run picks other samples than R's."""
    from .derep import derepFastq
    if isinstance(fls, dict) and "uniques" in fls:
        fls = [fls]
    fls = list(fls)
    if randomize:
        fls = [fls[k] for k in np.random.default_rng(seed).permutation(len(fls))]
    drps, NBASES = [], 0
    for f in fls:
        d = f if isinstance(f, dict) else derepFastq(f, device=device)
        drps.append(d)
        ab = np.asarray(d["abundances"], dtype=np.float64)
        NBASES += float(np.sum(ab * np.fromiter((len(s) for s in d["uniques"]), np.float64, len(d["uniques"]))))
        if NBASES > nbases:
            break
    if verbose:
        print("%d total bases in %d reads from %d samples will be used for learning the error rates." % (
            NBASES, sum(int(np.sum(d["abundances"])) for d in drps), len(drps)))
    dds = dada(drps, err=None, errorEstimationFunction=errorEstimationFunction, selfConsist=True, verbose=verbose, device=device,
               MAX_CONSIST=MAX_CONSIST, OMEGA_C=OMEGA_C, **opts)
    out = getErrors_detailed(dds)
    out["nsamples"] = len(drps)
    return out
