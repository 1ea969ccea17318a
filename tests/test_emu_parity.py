"""The CUDA sources run on the host SIMT emulator (tests/emu) against the reference goldens -- CPU suite.

tests/emu compiles dada2_b200/csrc/*.cu (kernels, round driver, C-ABI) for the host: every CUDA thread is a fiber, warp
shuffles / ballots / barriers are real rendezvous points, shared memory and atomics behave as on the device.  These
tests therefore check the *kernel logic itself* without a GPU: the same assertions as tests/test_gpu_parity.py, on the
emulated library.  They do not replace the `-m gpu` parity tests (hardware scheduling, memory model and the device
libm are not emulated) and nothing under dada2_b200/ ever loads the emulated library.

DADA2B_EMU_FULL=1 runs all e2e cases (about five minutes) instead of the quick subset.
"""
import ctypes
import os
import platform
import sys

import pytest

from tests import cases

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")

QUICK = ["syn800_default", "syn800_nogreedy", "syn600_band0", "syn800_maxclust5", "syn800_kdist", "syn800_ones_err", "syn700_ragged",
         "syn500_usequals0"]
E2E = list(cases.E2E_CASES) if os.environ.get("DADA2B_EMU_FULL") else QUICK


@pytest.fixture(scope="module")
def emu_lib():
    import build_emu
    return build_emu.build()


@pytest.fixture()
def emu(emu_lib, monkeypatch):
    """Points dada2_b200.api at the emulated library for one test; yields the launch-counter handle."""
    import dada2_b200.api as api
    monkeypatch.setattr(api, "_LIBPATH", emu_lib)
    monkeypatch.setattr(api, "_LIB", None)
    h = ctypes.CDLL(emu_lib)
    h.cuemu_launches.restype = ctypes.c_long
    h.cuemu_launches.argtypes = [ctypes.c_char_p]
    h.cuemu_reset_launches()
    yield h


def _gpu_tests():
    import tests.test_gpu_parity as T
    return T


def test_emu_calc_pA(emu):
    _gpu_tests().test_device_calc_pA_matches_oracle()


def test_emu_pair_corpus(emu):
    _gpu_tests().test_pair_corpus_kernels_match_reference()
    assert emu.cuemu_launches(b"k_classify") > 0 and emu.cuemu_launches(b"k_align") > 0


def test_emu_pair_corpus_loop_aligners(emu):
    _gpu_tests().test_pair_corpus_loop_aligners_match_traceback_kernel()
    assert emu.cuemu_launches(b"k_nwrow<") > 0 and emu.cuemu_launches(b"k_nwlane<") > 0 and emu.cuemu_launches(b"k_nwfwd<") > 0


def test_emu_config1(emu):
    _gpu_tests().test_config1_bit_identical()
    assert emu.cuemu_launches(b"k_nwrow<") > 0 and emu.cuemu_launches(b"k_prescreen") > 0


def test_emu_error_paths(emu):
    _gpu_tests().test_error_paths()


@pytest.mark.parametrize("name", E2E)
def test_emu_e2e(emu, name):
    _gpu_tests().test_e2e_matches_reference_golden(name, None)


@pytest.mark.parametrize("name", ["syn2000_default", "syn700_ragged", "syn800_nogreedy"])
def test_emu_e2e_one_sm(emu, monkeypatch, name):
    """CUEMU_SMS=1: one emulated SM, so every CTA of the grid-stride kernels takes several tiles / jobs (the streaming screen's ring
    stages are reused, pending raws are handed across tiles); goldens and screen counts stay the reference's."""
    monkeypatch.setenv("CUEMU_SMS", "1")
    monkeypatch.setenv("DADA2B_SMS", "1")
    _gpu_tests().test_e2e_golden_at_capped_sm_count(monkeypatch, name, "1")


@pytest.mark.parametrize("sms", ["1", "2"])
def test_emu_screen_stage(emu, monkeypatch, sms):
    """tests/screen_cases.py through the stage hook dada2b_test_screen on both paths, against tests/screen_ref.py (the GPU suite runs the
    same cases in test_gpu_zz_screen.py, plus a 250 k-raw full-grid case that is too slow here)."""
    import dada2_b200.api as api
    from tests import screen_cases as SC
    monkeypatch.setenv("CUEMU_SMS", sms)
    for case in SC.small_cases():
        SC.run_case(api.Resident, case, int(sms))
    assert emu.cuemu_launches(b"k_prescreen") > 0 and emu.cuemu_launches(b"k_kord") > 0 and emu.cuemu_launches(b"k_classify") > 0


@pytest.mark.parametrize("name", ["syn800_default", "syn800_band8", "syn800_kdist"] if not os.environ.get("DADA2B_EMU_FULL") else list(cases.E2E_CASES))
def test_emu_e2e_fallback_kernels(emu, monkeypatch, name):
    """DADA2B_FALLBACK=1: no thread-per-pair / lane kernels, no streaming screen -- the general kernels alone (the path of
    ragged lengths, other bands, homopolymer gap costs) reproduce the goldens on every case."""
    monkeypatch.setenv("DADA2B_FALLBACK", "1")
    _gpu_tests().test_e2e_matches_reference_golden(name, None)
    assert emu.cuemu_launches(b"k_nwrow<") == 0 and emu.cuemu_launches(b"k_nwlane<") == 0 and emu.cuemu_launches(b"k_prescreen") == 0


@pytest.mark.parametrize("lane_max", ["0", "32", "96"])
@pytest.mark.parametrize("name", ["syn800_default", "syn700_ragged"] if not os.environ.get("DADA2B_EMU_FULL") else ["syn800_default", "syn700_ragged", "syn2000_default", "syn800_band8", "syn800_priors"])
def test_emu_e2e_every_round_size_class(emu, monkeypatch, name, lane_max):
    """DADA2B_LANE_MAX (test hook) moves the job-count threshold between the lane-group kernel and the thread-per-pair kernels so that
    small inputs exercise what 1e6-unique runs do: rounds above the threshold (bound pass thread-per-pair, survivors through the
    lane kernel or, above the threshold again, the thread-per-pair exact kernel) and rounds below it (one lane-group launch)."""
    monkeypatch.setenv("DADA2B_LANE_MAX", lane_max)
    _gpu_tests().test_e2e_matches_reference_golden(name, None)
    assert emu.cuemu_launches(b"k_nwrow<") > 0
    assert (emu.cuemu_launches(b"k_nwlane<") > 0) == (lane_max != "0")


def test_emu_long_reads_band32_homopolymer(emu, monkeypatch):
    """BASELINE config 5 flavour at toy size: ~1.5 kb uniques, band 32, 94 quality columns; the homopolymer-gap scalar
    path (nwalign_endsfree.cpp:220-396) and the vectorized path with ragged lengths."""
    from oracle import port
    from tools import synth
    import dada2_b200
    seqs, ab, q = synth.pacbio(36, L=1500, nvar=3, seed=5)
    err = synth.extend_err(cases.tperr1(), 94)
    for opts in (dict(band_size=32, vectorized_alignment=False, homo_gap=-1), dict(band_size=32)):
        o = dict(opts)
        o.setdefault("homo_gap", -8)
        got = dada2_b200.dada_uniques(seqs, ab, None, err, q, **opts)
        want = port.dada_uniques(seqs, ab, None, err, q, **o)
        cases.assert_same(got, want, rtol=1e-10, label=str(opts))
    assert emu.cuemu_launches(b"k_nwfwd<") > 0              # ragged lengths / homopolymer costs: the general lane-group kernel


def _run_sharded(world, name, case=None, reupload=False):
    import threading

    import numpy as np

    import dada2_b200.api as api
    from tests.test_oracle import load_golden
    if case is None:
        seqs, ab, pri, err, q, opts = cases.build_case(name)
        want = load_golden(name)
    else:                                   # (seqs, abund, priors, quals, opts): expected result from the CPU oracle
        from oracle import port
        seqs, ab, pri, q, opts = case
        err = cases.tperr1()
        want = port.dada_uniques(seqs, ab, pri, err, q, **dict(opts, homo_gap=opts.get("homo_gap", -8)))
    uid = api.nccl_unique_id()
    results = [None] * world

    def rank_main(r):
        try:
            res = api.Resident(seqs, ab, pri, q)
            res.comm_init(r, world, uid)
            if reupload:                    # dada2b_reupload on a sharded context: only this rank's quality rows travel (bench.py's e2e at N > 1)
                from dada2_b200 import _abi
                res.reupload(_abi.PackedIn(seqs, ab, pri, None, q))
            results[r] = res.run(err, **opts)
            res.close()
        except Exception as e:      # surfaced below, on the main thread
            results[r] = e

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    pb = None
    if pri is not None:
        pb = np.zeros(len(want["clustering"]["sequence"]), dtype=bool)
        pb[1:] = want["clustering"]["birth_pval"][1:] >= opts.get("omegaA", 1e-40)
    for r in range(world):
        if isinstance(results[r], Exception):
            raise results[r]
        cases.assert_same(results[r], want, rtol=1e-10, prior_born=pb, label=f"{name} rank {r}/{world}")


@pytest.mark.parametrize("world,name", [(2, "syn800_default"), (3, "syn700_ragged"), (8, "syn800_maxclust5")])
def test_emu_sharded_ranks(emu, world, name):
    """The sharded multi-GPU path (raw r aligned by rank r % world; owner mode) with the ranks as threads and the emulator's
    in-process NCCL stand-in: every rank returns the reference's result."""
    _run_sharded(world, name)


@pytest.mark.parametrize("world,name", [(2, "syn800_default"), (3, "syn700_ragged"), (4, "syn800_priors")])
def test_emu_sharded_reupload_keeps_only_owned_quality_rows(emu, world, name):
    """dada2b_reupload after dada2b_comm_init packs and uploads the quality rows of the rank's own raws only; the rows of the
    cluster centres are exchanged before the birth subs; results stay the reference's on every rank."""
    _run_sharded(world, name, reupload=True)
    assert emu.cuemu_launches(b"k_qrows_scatter") > 0 and emu.cuemu_launches(b"k_qrows_gather") > 0


@pytest.mark.parametrize("blk", [1, 100])
def test_emu_upload_pipeline_many_blocks(emu, monkeypatch, blk):
    """do_upload packs blocks of raws on worker threads and sends every group of 16 finished blocks to the device while the
    later ones are still being packed: DADA2B_PACK_BLK (test hook) makes 800 raws span many blocks and groups, on one
    context and on sharded re-uploads (rows of the rank's own raws only, groups that start at any raw index)."""
    import dada2_b200
    from tests.test_oracle import load_golden
    monkeypatch.setenv("DADA2B_PACK_BLK", str(blk))
    name = "syn700_ragged"
    seqs, ab, pri, err, q, opts = cases.build_case(name)
    cases.assert_same(dada2_b200.dada_uniques(seqs, ab, pri, err, q, **opts), load_golden(name), rtol=1e-10, label=name)
    _run_sharded(3, name, reupload=True)


FUSED_E2E = ["syn800_default", "syn800_nogreedy", "syn800_maxclust5", "syn700_ragged"] if not os.environ.get("DADA2B_EMU_FULL") else list(cases.E2E_CASES)


TAIL_CASES = ([pytest.param(name, np_passes, None, id=f"{name}-{np_passes}") for name in FUSED_E2E for np_passes in (1, 3)] +
              [pytest.param(name, 3, n, id=f"{name}-3-tail_smem{n}") for name in ("syn800_default", "syn700_ragged") for n in ("0", "12")])


@pytest.mark.parametrize("name,np_passes,tail_smem", TAIL_CASES)
def test_emu_e2e_fused_tail(emu, monkeypatch, name, np_passes, tail_smem):
    """The round tail (dd_round2.cu): 1 + NP + 1 launches per round.  NP=1 makes every round that needs a second shuffle pass
    continue with one more pass at a time.  DADA2B_TAIL_SMEM_CLUSTERS (test hook) moves the cluster count above which the tail
    reads its per-cluster state from global memory instead of staging it in shared memory: 0 = every round, 12 = from mid-run on,
    as runs past ~32 k clusters do."""
    if np_passes == 1 and name not in ("syn800_default", "syn800_maxclust5") and not os.environ.get("DADA2B_EMU_FULL"):
        pytest.skip("quick subset")
    monkeypatch.setenv("DADA2B_NP", str(np_passes))
    _gpu_tests().test_e2e_matches_reference_golden(name, tail_smem)
    assert emu.cuemu_launches(b"k_tail_final") > 0
    assert (emu.cuemu_launches(b"k_tail_final<true>") > 0) == (tail_smem != "0")
    assert (emu.cuemu_launches(b"k_tail_pass<false>") > 0 and emu.cuemu_launches(b"k_tail_final<false>") > 0) == (tail_smem is not None)
    if np_passes == 1:      # rounds that moved raws in pass 0 continue with one more pass (and final) at a time
        extra = emu.cuemu_launches(b"k_tail_final") - emu.cuemu_launches(b"k_tail_link")
        assert extra >= 0 and (extra > 0 or name not in ("syn800_default", "syn800_maxclust5"))      # e.g. max_clust=1: nothing ever moves


@pytest.mark.parametrize("tail_smem", [None, "0"], ids=["default", "global_tail"])
def test_emu_large_tie_sets(emu, tail_smem):
    """b_bud tie sets larger than TIE_MAX: the host fetches the whole set (k_bud_collect_owned) and applies the scan order, with the
    round tail's per-cluster state in shared memory (default) and in global memory (DADA2B_TAIL_SMEM_CLUSTERS=0)."""
    import tests.test_gpu_zz_ties as TT
    for opts in (dict(), dict(greedy=False), dict(max_clust=30)):
        TT.test_large_tie_sets_follow_scan_order(opts, tail_smem)
    assert emu.cuemu_launches(b"k_bud_collect_owned") > 0
    assert (emu.cuemu_launches(b"k_tail_final<false>") > 0) == (tail_smem is not None)
    assert (emu.cuemu_launches(b"k_tail_final<true>") > 0) == (tail_smem is None)


@pytest.mark.parametrize("fallback", [False, True], ids=lambda e: "fallback" if e else "default")
def test_emu_edge_cases(emu, monkeypatch, fallback):
    """tests/cases.py:edge_cases() on the emulated library (the GPU suite runs the same table in test_gpu_zzz_edge.py),
    with the default kernels and with the general (fallback) kernels only."""
    import dada2_b200
    if fallback:
        monkeypatch.setenv("DADA2B_FALLBACK", "1")
    for case in cases.edge_cases():
        cases.check_edge_case(case, dada2_b200.dada_uniques)


@pytest.mark.parametrize("world,name,tail_smem", [(2, "syn800_default", None), (3, "syn700_ragged", None), (8, "syn800_nogreedy", None),
                                                  (2, "syn800_default", "0"), (3, "syn700_ragged", "12")],
                         ids=["2-syn800_default", "3-syn700_ragged", "8-syn800_nogreedy", "2-syn800_default-tail_smem0", "3-syn700_ragged-tail_smem12"])
def test_emu_sharded_owner_mode(emu, monkeypatch, world, name, tail_smem):
    """Owner mode (how sharded runs work): every rank keeps the stored comparisons and runs shuffle /
    p-update / bud scan for its own raws only; per pass one all-reduce of the cluster read deltas, per round one
    all-gather of the ranks' reports and (when raws moved) of the move lists.  No exchange of comparisons at all.
    DADA2B_TAIL_SMEM_CLUSTERS: the round tail's per-cluster state in global memory from the first round (0) or from mid-run (12)."""
    if tail_smem is not None:
        monkeypatch.setenv("DADA2B_TAIL_SMEM_CLUSTERS", tail_smem)
    _run_sharded(world, name)
    assert emu.cuemu_launches(b"k_cs_append") == 0 and emu.cuemu_launches(b"k_posthoc_owned") > 0
    assert (emu.cuemu_launches(b"k_tail_final<false>") > 0) == (tail_smem is not None)


@pytest.mark.parametrize("eager", [0, 3])
def test_emu_sharded_report_gather_carries_the_head_of_the_move_lists(emu, monkeypatch, eager):
    """The round's all-gather carries every rank's report AND the first DADA2B_MOVES_EAGER (test hook; default 1024 sharded, 8192 on
    one GPU) moves of its list; only rounds in which some rank moved more exchange the whole lists in a second all-gather.  0: always
    the second exchange; 3: rounds of both kinds (the default never needs it at this size: every other test).  World 1 is the same
    path with a device-to-host copy in place of each all-gather."""
    monkeypatch.setenv("DADA2B_MOVES_EAGER", str(eager))
    _run_sharded(3, "syn800_nogreedy")
    _run_sharded(2, "syn700_ragged", reupload=True)
    _run_sharded(1, "syn800_default")


def test_emu_sharded_owner_mode_ties_and_extra_passes(emu, monkeypatch):
    """Owner mode corner paths: tie sets larger than TIE_MAX (per-rank candidate lists exchanged), and NP=1 so that rounds
    needing more shuffle passes continue with one fused pass at a time."""
    monkeypatch.setenv("DADA2B_NP", "1")
    seqs, ab, q = cases.tie_case()
    _run_sharded(2, "ties", case=(seqs, ab, None, q, dict(max_clust=40)))
    assert emu.cuemu_launches(b"k_bud_collect_owned") > 0
    _run_sharded(3, "syn800_maxclust5")


