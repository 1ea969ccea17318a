"""Samples for the final pass's diagonal-list tally (dd_final.cu) and round 0's diagonal test, shared by
tests/test_emu_final_tally.py (host SIMT emulator) and tests/test_gpu_zz_final_tally.py (H100).  Every case is compared in full
against the reference's C++ (oracle.port) on the same input.

  big_cluster    one cluster of more than three tally chunks (dd_final.cu:FT_CHUNK members each)
  omegaC         omegaC = 0.01: many raws are not correct and stay out of the transition / quality tallies
  indels_ragged  unequal lengths (gapless pairs count positions below the shorter length only) and max_clust = 3 over variants
                 with indels, so that the final pass has gapped alignments beside the diagonal ones
  many_clusters  more clusters than dd_final.cu counts through shared memory (omegaA = 0.5, singletons, max_clust = 90)
"""
import numpy as np

from tests import cases

FT_CHUNK = 512          # dd_final.cu
FT_SMEM_CL = 64         # dd_final.cu: clusters counted through shared memory first
NAMES = ["big_cluster", "omegaC", "indels_ragged", "many_clusters"]


def sample(name):
    """-> (seqs, abundances, quals, opts)"""
    from tools import synth
    if name == "big_cluster":
        seqs, ab, q, _ = synth.illumina(1800, nvar=1, seed=41)
        return seqs, ab, q, {}
    if name == "omegaC":
        seqs, ab, q, _ = synth.illumina(900, nvar=6, seed=42)
        return seqs, ab, q, dict(omegaC=1e-2, omegaA=1e-20)
    if name == "indels_ragged":
        seqs, ab, q, _ = synth.illumina(900, nvar=8, indel_frac=1.0, seed=43)
        rng = np.random.default_rng(1043)
        cut = rng.integers(0, 7, size=len(seqs))
        cut[0] = 0
        seqs = [s[:len(s) - c] for s, c in zip(seqs, cut)]
        q = q.copy()
        for i, s in enumerate(seqs):
            q[i, len(s):] = np.nan
        return seqs, ab, q, dict(max_clust=3)
    if name == "many_clusters":
        seqs, ab, q, _ = synth.illumina(1000, nvar=100, seed=44)
        return seqs, ab, q, dict(omegaA=0.5, detect_singletons=True, max_clust=90)
    raise KeyError(name)


def expected(seqs, ab, q, opts):
    from oracle import port
    return port.dada_uniques(seqs, ab, None, cases.tperr1(), q, **dict(opts, homo_gap=opts.get("homo_gap", -8)))


def check_shape(name, want):
    """The sample reaches what its name says (on the reference's own result)."""
    nunq, mapped = want["clustering"]["nunq"], np.asarray(want["map"]) >= 1        # $map is NA (INT_MIN) for raws that are not correct
    if name == "big_cluster":
        assert int(np.max(nunq)) > 3 * FT_CHUNK
    if name == "omegaC":
        assert 0 < int(np.sum(~mapped)) < len(mapped) // 2
    if name == "many_clusters":
        assert len(nunq) > FT_SMEM_CL


def run_case(name, dada_uniques):
    seqs, ab, q, opts = sample(name)
    want = expected(seqs, ab, q, opts)
    check_shape(name, want)
    got = dada_uniques(seqs, ab, None, cases.tperr1(), q, **opts)
    cases.assert_same(got, want, rtol=1e-10, label=name)
    return want
