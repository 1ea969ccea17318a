"""Randomised differential campaign of the dada() hot path: the CUDA sources on the host SIMT emulator (tests/emu) against the
reference's own C++ (oracle/_ref), full output compared (ints exact, fp64 <= 1e-10).  Test tooling, not part of the suite.
  python tools/fuzz_dada_emu.py <seed> <seconds>
Every iteration draws a sample (size, read length, variants, indel fraction, ragged ends, low-complexity stretches, priors) and
options (band, omegaA, greedy, detect_singletons, min_abund / min_fold / min_hamming, kdist_cutoff, max_clust), and the size class
switches (DADA2B_LANE_MAX) so that the thread-per-pair, the lane-group and the general kernels all take turns, DADA2B_PACK_BLK the
upload pipeline's block size, some quality matrices sit on exact halves and their neighbouring doubles; two iterations in
five shard the sample over 2-3 ranks (owner mode; ranks as threads, the emulator's in-process NCCL stand-in), half of those through
dada2b_reupload."""
import sys, os, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import numpy as np
import build_emu
lib = build_emu.build()
import dada2_b200.api as api
api._LIBPATH = lib
import dada2_b200
from oracle import ref
from tests import cases
from tools import synth

seed = int(sys.argv[1]) if len(sys.argv) > 1 else 0
rng = np.random.default_rng(seed)
t_end = time.time() + (float(sys.argv[2]) if len(sys.argv) > 2 else 600)
err = cases.tperr1()
it = 0; nraw_tot = 0; nclust_tot = 0
while time.time() < t_end:
    it += 1
    n = int(rng.choice([60, 150, 400, 900, 2000]))
    L = int(rng.choice([40, 90, 150, 250]))
    nvar = int(rng.integers(2, 25))
    seqs, ab, q, _ = synth.illumina(n, L=L, nvar=nvar, max_subs=int(rng.integers(2, max(3, L // 4))), indel_frac=float(rng.choice([0.0, 0.1, 0.5])),
                                    seed=int(rng.integers(1, 1 << 30)), lowq_frac=float(rng.choice([0.0, 0.02, 0.2])))
    seqs = list(seqs)
    if rng.random() < 0.3:                      # ragged 3' ends
        cut = rng.integers(0, 7, size=len(seqs)); cut[0] = 0
        seqs = [s[:len(s) - c] for s, c in zip(seqs, cut)]
        q = q.copy()
        for i, s in enumerate(seqs):
            q[i, len(s):] = np.nan
    if rng.random() < 0.2:                      # a low-complexity stretch in some reads: repeated 5-mers, shifted alignments tie
        k = int(rng.integers(0, max(1, L - 30)))
        rep = "".join(rng.choice(list("ACGT"), 2)) * 12
        for i in rng.choice(len(seqs), size=max(1, len(seqs) // 10), replace=False):
            s = seqs[i]
            if len(s) > k + 24: seqs[i] = s[:k] + rep[:24] + s[k + 24:]
    if rng.random() < 0.15:                     # mean qualities on exact halves and the doubles next to them ((uint8_t) round(q), containers.cpp:34)
        near = rng.random(q.shape)
        h = np.minimum(np.floor(q), 39.0) + 0.5          # 40.5 would round to 41, beyond the 41 columns of tperr1 (the reference reads past its table there)
        q = np.where(np.isnan(q), q, np.where(near < 0.25, np.nextafter(h, 0.0), np.where(near < 0.5, np.nextafter(h, 100.0), np.where(near < 0.75, h, q))))
        q[:, 0] = np.where(np.isnan(q[:, 0]), q[:, 0], 0.49999999999999994)
    priors = (rng.random(len(seqs)) < 0.05).astype(np.uint8) if rng.random() < 0.3 else None
    opts = dict(band_size=int(rng.choice([16, 16, 8, 32])), omegaA=float(rng.choice([1e-40, 1e-40, 1e-10, 1e-3])),
                greedy=int(rng.integers(0, 2)), detect_singletons=int(rng.random() < 0.2), min_abund=int(rng.choice([1, 1, 2, 8])),
                min_fold=float(rng.choice([1.0, 1.0, 2.0])), min_hamming=int(rng.choice([1, 1, 2])),
                kdist_cutoff=float(rng.choice([0.42, 0.42, 0.3, 0.6])), max_clust=int(rng.choice([0, 0, 0, 5])))
    if rng.random() < 0.15: opts["use_quals"] = 0
    if os.environ.get("FUZZ_RARE_OPTS"):        # the options the e2e goldens cover once each, a few at a time
        if rng.random() < 0.15: opts["gapless"] = 0
        if rng.random() < 0.15: opts["use_kmers"] = 0
        if rng.random() < 0.2: opts["SSE"] = int(rng.integers(0, 3))
        if rng.random() < 0.2:
            opts["vectorized_alignment"] = 0
            if rng.random() < 0.6: opts["homo_gap"] = int(rng.choice([-1, -4, -8]))
        if rng.random() < 0.2:
            m, mm, g = [(4, -5, -7), (5, -4, -4), (1, -1, -2), (5, -4, -16)][int(rng.integers(0, 4))]
            opts.update(match=m, mismatch=mm, gap=g)
            if "homo_gap" not in opts and not opts.get("vectorized_alignment", 1): opts["homo_gap"] = g
        if rng.random() < 0.15: opts["omegaC"] = float(rng.choice([1e-5, 0.0, 1.0]))
        if rng.random() < 0.15: opts["omegaP"] = float(rng.choice([1e-2, 0.5, 1e-10]))
        if rng.random() < 0.1: opts["band_size"] = int(rng.choice([0, 64] + ([-1] if L <= 90 else [])))
    if (opts["detect_singletons"] or opts["omegaA"] >= 1e-10) and opts["max_clust"] == 0 and len(seqs) > 400:
        opts["max_clust"] = 25                  # permissive thresholds bud hundreds of clusters: bound the emulated rounds
    os.environ["DADA2B_LANE_MAX"] = str(int(rng.choice([0, 32, 256, 16384])))
    eag = int(rng.choice([-1, -1, 0, 5, 64]))   # moves carried by the round's report copy (-1: the default, 8192 / 1024 sharded)
    if eag >= 0: os.environ["DADA2B_MOVES_EAGER"] = str(eag)
    else: os.environ.pop("DADA2B_MOVES_EAGER", None)
    blk = int(rng.choice([0, 0, 1, 13, 64]))    # upload pipeline: raws per packing block (0: the default, one block here)
    if blk: os.environ["DADA2B_PACK_BLK"] = str(blk)
    else: os.environ.pop("DADA2B_PACK_BLK", None)
    tsm = int(rng.choice([-1, -1, 0, 4, 16]))   # round tail: clusters staged in shared memory (-1: the default, every round here)
    if tsm >= 0: os.environ["DADA2B_TAIL_SMEM_CLUSTERS"] = str(tsm)
    else: os.environ.pop("DADA2B_TAIL_SMEM_CLUSTERS", None)
    if it < int(os.environ.get("FUZZ_SKIP_UNTIL", "0")): continue          # replay a campaign up to a given iteration (the draws above are all that matters)
    if os.environ.get("FUZZ_VERBOSE"): print("it", it, "n", len(seqs), "L", L, "nvar", nvar, opts, "lane_max", os.environ["DADA2B_LANE_MAX"], "priors", priors is not None, flush=True)
    want = ref.dada_uniques(seqs, ab, priors, err, q, **dict(dict(homo_gap=opts.get("gap", -8)), **opts))
    if os.environ.get("FUZZ_VERBOSE"): print("   reference done", flush=True)
    world = int(rng.choice([1, 1, 1, 2, 3])) if os.environ.get("FUZZ_SHARDED", "1") != "0" else 1
    if world == 1:
        got = dada2_b200.dada_uniques(seqs, ab, priors, err, q, **opts)
    else:                                       # owner-mode sharding: the ranks are threads, NCCL is the emulator's in-process stand-in
        import threading
        uid = api.nccl_unique_id()
        results = [None] * world
        reup = bool(rng.integers(0, 2))
        def rank_main(r):
            try:
                res = api.Resident(seqs, ab, priors, q)
                res.comm_init(r, world, uid)
                if reup:
                    from dada2_b200 import _abi
                    res.reupload(_abi.PackedIn(seqs, ab, priors, None, q))
                results[r] = res.run(err, **opts)
                res.close()
            except Exception as e:
                results[r] = e
        th = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
        for t in th: t.start()
        for t in th: t.join()
        for r in range(world):
            if isinstance(results[r], Exception): raise results[r]
        got = results[0]
        for r in range(1, world):
            cases.assert_same(results[r], got, rtol=0, prior_born=None, label="fuzz seed %d it %d: rank %d vs rank 0" % (seed, it, r))
        n_sharded = globals().get("n_sharded", 0) + 1
    pb = None
    if priors is not None:                      # prior-born clusters: the reference leaves birth_from uninitialised (cluster.cpp:334-339)
        pb = np.zeros(len(want["clustering"]["sequence"]), dtype=bool)
        pb[1:] = np.asarray(want["clustering"]["birth_pval"])[1:] >= opts["omegaA"] / len(seqs)    # birth_pval = pP there, and pP >= omegaA / nraw
    try:
        cases.assert_same(got, want, rtol=1e-10, prior_born=pb, label="fuzz seed %d it %d %r" % (seed, it, opts))
    except AssertionError:
        import pickle
        pickle.dump(dict(seqs=seqs, ab=ab, q=q, priors=priors, opts=opts, lane_max=os.environ["DADA2B_LANE_MAX"]), open("/tmp/fuzz_fail_%d_%d.pkl" % (seed, it), "wb"))
        raise
    nraw_tot += len(seqs); nclust_tot += len(got["clustering"]["sequence"])
    if it % 10 == 0:
        print("it %d: %d uniques, %d clusters so far, all identical" % (it, nraw_tot, nclust_tot), flush=True)
print("DONE seed %d: %d iterations (%d sharded over 2-3 ranks), %d uniques, %d clusters: all identical" % (seed, it, globals().get("n_sharded", 0), nraw_tot, nclust_tot))
