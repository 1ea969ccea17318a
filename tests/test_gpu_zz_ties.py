"""Large exact-tie sets in the b_bud scan (more candidates than the device reports inline): the host has to fetch the
whole set and apply the reference's (cluster, slot) scan order.  Checked against the CPU oracle."""
import pytest

from tests import cases

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("opts,tail_smem", [pytest.param(o, None, id=i) for o, i in zip([dict(), dict(greedy=False), dict(max_clust=30)],
                                                                                         ["default", "nogreedy", "maxclust30"])] +
                         [pytest.param(dict(), n, id=f"default-tail_smem{n}") for n in ("0", "40")])
def test_large_tie_sets_follow_scan_order(opts, tail_smem):
    """tail_smem: DADA2B_TAIL_SMEM_CLUSTERS (test hook), the round tail's per-cluster state in global memory from the first round (0)
    or from mid-run (40)."""
    import dada2_b200
    from oracle import port
    seqs, ab, q = cases.tie_case()
    err = cases.tperr1()
    with pytest.MonkeyPatch.context() as mp:
        if tail_smem is not None:
            mp.setenv("DADA2B_TAIL_SMEM_CLUSTERS", tail_smem)
        got = dada2_b200.dada_uniques(seqs, ab, None, err, q, **opts)
    want = port.dada_uniques(seqs, ab, None, err, q, **dict(opts, homo_gap=-8))
    cases.assert_same(got, want, rtol=1e-10, label="ties " + str(opts))
    cases.assert_same_screen_counts(got, want, label="ties " + str(opts))
    assert len(got["clustering"]["abundance"]) == (30 if "max_clust" in opts else 151)
