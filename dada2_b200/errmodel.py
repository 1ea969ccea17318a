"""Error-model refit of the selfConsist loop (SURVEY.md 8(f2)): host-side mirror of the reference's R code.

    accumulateTrans   /root/reference/R/errorModels.R:462-471
    loessErrfun       /root/reference/R/errorModels.R:28-67
    PacBioErrfun      R/errorModels.R:183-196 (reference)
    dada(selfConsist=TRUE) / learnErrors loop   /root/reference/R/dada.R:256-391, R/errorModels.R:270-330 (consist_loop;
                                                dada_selfconsist / learnErrors below run it on one resident sample)

The reference does these steps in R between the <= 11 dada_uniques() passes; they see a 16 x Q matrix, so they stay on the
host here as well (R is not in this image: Python mirrors the R functions name for name, like dada2_b200/api.py does for
dada_uniques).  What matters for the accelerated path is that the uniques stay RESIDENT in HBM across the passes
(dada2b_upload once, dada2b_run_resident per pass): `dada_selfconsist` below drives exactly that.

PARITY UNPINNED for `loess`: R's stats::loess (netlib dloess: k-d tree + blending interpolation, surface = "interpolate")
is not in /root/reference and R is not available, and the reference holds no fitted error matrices to compare with.  The
restatement below evaluates the same local regression -- degree 2, span 0.75, tricube neighbourhood weights times the
prior weights `tot`, gaussian family -- DIRECTLY at every quality score (R's surface = "direct"); R's default interpolates
that surface between k-d tree vertices, which changes low-order digits of the fit, not its shape.  Everything around it
(pseudo-counts, log10 rates, NA handling, clamping to [1e-7, 0.25], left-over self transitions) follows the R code line by line.
tests/test_errmodel.py pins what can be pinned without R: exact reproduction of quadratics, the row / column structure of
the result, invariance properties, and the fixed point of the loop on synthetic data.
"""
from __future__ import annotations

import numpy as np

ROWNAMES = [a + "2" + b for a in "ACGT" for b in "ACGT"]
MAX_ERROR_RATE = 0.25            # R/errorModels.R:54
MIN_ERROR_RATE = 1e-7            # R/errorModels.R:55


def accumulateTrans(trans):
    """Sum 16 x Q_i transition-count matrices, Q = max Q_i (R/errorModels.R:462-471)."""
    trans = [np.asarray(t) for t in trans]
    maxcol = max(t.shape[1] for t in trans)
    rval = np.zeros((16, maxcol), dtype=np.float64)
    for t in trans:
        if t.shape[0] != 16:
            raise ValueError("transition matrices must have 16 rows")
        rval[:, :t.shape[1]] += t
    return rval


def loess_direct(x, y, w, xout, span=0.75, degree=2):
    """Weighted local polynomial regression evaluated directly (R: loess(y ~ x, weights = w, span, degree, family = "gaussian",
    surface = "direct")).  Neighbourhood of an evaluation point: the q = floor(n * span + 1e-5) nearest observations
    (lowesd.f / ehg127: fc = floor(n * f + 1e-5)), bandwidth h = distance to the q-th nearest one, tricube weights
    (1 - (d / h)^3)^3 for d < h, multiplied by the prior weights; least squares on 1, (x - x0), (x - x0)^2.
    Returns NaN outside [min(x), max(x)] like R's interpolating surface (predict.loess does not extrapolate)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    xout = np.asarray(xout, dtype=np.float64)
    n = len(x)
    out = np.full(len(xout), np.nan)
    if n < degree + 1:
        raise ValueError("loess: too few observations")
    q = int(np.floor(n * span + 1e-5))
    q = max(min(q, n), degree + 1)
    for k, x0 in enumerate(xout):
        if not (x.min() <= x0 <= x.max()):
            continue
        d = np.abs(x - x0)
        h = np.sort(d)[q - 1]
        if h <= 0:
            h = 1.0
        u = np.minimum(d / h, 1.0)                     # d >= h: weight 0
        tw = (1.0 - u ** 3) ** 3
        ww = tw * w
        nz = ww > 0
        if nz.sum() < degree + 1:           # degenerate neighbourhood: fall back to the widest fit that is determined
            ww = w.copy()
            nz = ww > 0
        X = np.vander(x[nz] - x0, degree + 1, increasing=True)
        sw = np.sqrt(ww[nz])
        beta, *_ = np.linalg.lstsq(X * sw[:, None], y[nz] * sw, rcond=None)
        out[k] = beta[0]
    return out


def loessErrfun(trans, span=0.75, degree=2):
    """16 x Q transition counts -> 16 x Q error rates (R/errorModels.R:28-67).  Column j is quality score j."""
    trans = np.asarray(trans, dtype=np.float64)
    if trans.shape[0] != 16:
        raise ValueError("trans must have 16 rows (A2A, A2C, ..., T2T)")
    Q = trans.shape[1]
    qq = np.arange(Q, dtype=np.float64)                       # as.numeric(colnames(trans))
    est = []
    for i in range(4):
        tot = trans[4 * i:4 * i + 4].sum(axis=0)              # colSums over the four transitions out of nti
        for j in range(4):
            if i == j:
                continue
            errs = trans[4 * i + j]
            with np.errstate(divide="ignore", invalid="ignore"):
                rlogp = np.log10((errs + 1.0) / tot)          # 1 pseudocount per error; tot = 0 -> NA
            rlogp[~np.isfinite(rlogp)] = np.nan
            ok = ~np.isnan(rlogp)                             # loess drops rows with NA (na.action = na.omit)
            if ok.sum() < degree + 2:
                raise ValueError("Error rates could not be estimated (this is usually because of very few reads).")
            pred = loess_direct(qq[ok], rlogp[ok], tot[ok], qq, span=span, degree=degree)
            valid = np.where(~np.isnan(pred))[0]
            maxrli, minrli = valid.max(), valid.min()
            pred[maxrli + 1:] = pred[maxrli]
            pred[:minrli] = pred[minrli]
            est.append(10.0 ** pred)
    est = np.array(est)                                       # 12 x Q, order A2C A2G A2T C2A C2G C2T G2A G2C G2T T2A T2C T2G
    est[est > MAX_ERROR_RATE] = MAX_ERROR_RATE
    est[est < MIN_ERROR_RATE] = MIN_ERROR_RATE
    err = np.vstack([1 - est[0:3].sum(axis=0), est[0:3],
                     est[3], 1 - est[3:6].sum(axis=0), est[4:6],
                     est[6:8], 1 - est[6:9].sum(axis=0), est[8],
                     est[9:12], 1 - est[9:12].sum(axis=0)])
    return err


def PacBioErrfun(trans):
    """16 x Q transition counts -> 16 x Q error rates for reads whose qualities reach 93 (R/errorModels.R:183-196).
    Column j is quality score j, so R's `"93" %in% colnames(trans)` is Q >= 94.  Columns 0..92 are loessErrfun's fit;
    column 93 is the observed rate with pseudo-counts, (count + 1) / (total of the source base + 4)."""
    trans = np.asarray(trans, dtype=np.float64)
    Q = trans.shape[1]
    if Q < 94:
        print("The max qual score of 93 was not detected. Using standard error fitting.")
        return loessErrfun(trans)
    if Q > 94:
        raise ValueError("Max qual score of 93 not the last column as expected.")
    err = loessErrfun(trans[:, :93])
    tot93 = np.repeat(trans[:, 93].reshape(4, 4).sum(axis=1), 4)
    return np.hstack([err, ((trans[:, 93] + 1.0) / (tot93 + 4.0))[:, None]])


def getErrors_enforce(err):
    """The validation dada() applies in selfConsist mode (getErrors(err, enforce = TRUE), R/errorModels.R:380-420)."""
    if err is None:
        raise ValueError("Error matrix is NULL.")
    err = np.asarray(err)
    if err.ndim != 2 or err.shape[0] != 16 or not np.issubdtype(err.dtype, np.number):
        raise ValueError("Error matrix must be numeric with 16 rows.")
    if np.any(np.isnan(err)) or np.any(err < 0) or np.any(err > 1):
        raise ValueError("Error matrix must contain values between 0 and 1.")
    return err


def consist_loop(runners, err=None, errorEstimationFunction=loessErrfun, MAX_CONSIST=10, selfConsist=True, verbose=False,
                 pseudo=None, on_pass=None):
    """The main loop of dada() (R/dada.R:256-391) over samples.

    runners[i](err, max_clust) -> the dada_uniques() result of sample i.  err = None: the loop starts from initializeErr
    (R/dada.R:297-299, :342): every runner is called with err None and max_clust 1 and builds its own all-ones matrix.
    pseudo(results) is called where R computes the pseudo priors of pool = "pseudo" (:380-384); the loop then always runs
    a second pass.  Returns (results of the last pass, final err, list of the err matrices tried, number of passes)."""
    initializeErr = err is None
    nconsist = 0 if initializeErr else 1
    errs = []
    npass = 0
    while True:
        if nconsist > 0:
            errs.append(err)
        results = [run(None if initializeErr else err, 1 if initializeErr else 0) for run in runners]
        npass += 1
        if on_pass:
            on_pass(npass, nconsist, results)
        cur = accumulateTrans([r["subqual"] for r in results])
        try:
            err = errorEstimationFunction(cur) if errorEstimationFunction is not None else None
        except ValueError:
            if selfConsist or verbose:
                print("Error rates could not be estimated (this is usually because of very few reads).")
            err = None
        if selfConsist:
            getErrors_enforce(err)
        if initializeErr:
            initializeErr = False
            err = np.array(err, dtype=np.float64)
            err[[0, 5, 10, 15], :] = 1.0                      # self-transitions of the initial estimate forced to 1 (R/dada.R:385-388)
        if (not selfConsist) or any(e is not None and err is not None and np.array_equal(e, err) for e in errs) or nconsist >= MAX_CONSIST:
            if pseudo is None or nconsist >= 2:
                break
        if pseudo is not None and nconsist >= 1:
            pseudo(results)
        nconsist += 1
    return results, err, errs, npass


def dada_selfconsist(runner, ncol=41, err=None, errorEstimationFunction=loessErrfun, MAX_CONSIST=10, selfConsist=True, verbose=False,
                     on_pass=None):
    """consist_loop for one (pooled) sample whose uniques are resident on the device.

    runner(err, max_clust) -> result dict of one dada_uniques() pass (e.g. `lambda e, mc: resident.run(e, max_clust=mc)`).
    err = None: learnErrors' start (initializeErr: all-ones 16 x ncol matrix, MAX_CLUST = 1).
    Returns (last result, final err, list of the err matrices tried, number of passes)."""
    def one(e, mc):
        return runner(np.ones((16, ncol)) if e is None else np.asarray(e, dtype=np.float64), mc)
    hook = (lambda n, c, rs: on_pass(n, c, rs[0])) if on_pass else None
    results, err, errs, npass = consist_loop([one], err=err, errorEstimationFunction=errorEstimationFunction, MAX_CONSIST=MAX_CONSIST,
                                             selfConsist=selfConsist, verbose=verbose, on_pass=hook)
    return results[0], err, errs, npass


def learnErrors(runner, ncol=41, errorEstimationFunction=loessErrfun, MAX_CONSIST=10, verbose=False, on_pass=None):
    """learnErrors (R/errorModels.R:270-330) on already dereplicated, pooled input: dada(err = NULL, selfConsist = TRUE)."""
    res, err, errs, npass = dada_selfconsist(runner, ncol=ncol, err=None, errorEstimationFunction=errorEstimationFunction,
                                             MAX_CONSIST=MAX_CONSIST, selfConsist=True, verbose=verbose, on_pass=on_pass)
    return {"err_out": err, "err_in": errs, "trans": np.asarray(res["subqual"]), "passes": npass, "dada": res}
