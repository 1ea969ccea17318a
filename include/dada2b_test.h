/* dada2b_test.h -- kernel-level entry points exported by libdada2b.so for the parity tests.
 * They run the SAME device kernels the dada2b_run() path uses (k_classify, k_align, calc_pA) on
 * caller-chosen pairs so that tests can diff individual stages against the oracle:
 *   raw_align / sub_new / compute_lambda_ts  (/root/reference/src/nwalign_endsfree.cpp:10-73,642-672; pval.cpp:144-197)
 *   calc_pA                                   (/root/reference/src/pval.cpp:44-64)
 */
#ifndef DADA2B_TEST_H
#define DADA2B_TEST_H
#include "dada2b.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Align npairs (centre[k], raw[k]) index pairs of an uploaded context.
 * kind: 0 shrouded (NULL sub), 1 gapless, 2 NW.  ops: opcap bytes per pair, alignment columns in
 * order, 1 = both bases, 2 = gap in the centre row, 3 = gap in the raw row.  Substitutions: subcap
 * entries per pair (pos0, nt0, nt1 as 0..3, q1). */
int dada2b_test_pairs(dada2b_ctx *ctx, int32_t npairs, const uint32_t *centre, const uint32_t *raw, const double *err,
                      int32_t Q, const dada2b_opts *opts, int32_t use_kmers, double kdist_cutoff, int32_t *kind,
                      double *lambda, int32_t *nsubs, uint8_t *ops, int32_t *nops, int32_t opcap, uint16_t *pos,
                      uint8_t *nt0, uint8_t *nt1, uint8_t *q1, int32_t subcap, char errbuf[DADA2B_ERRLEN]);

/* out[k] = calc_pA(reads[k], E[k], prior[k]) evaluated on the device. */
int dada2b_test_calc_pA(int32_t n, const int32_t *reads, const double *E, const int32_t *prior, double *out,
                        char errbuf[DADA2B_ERRLEN]);

/* Kernel-level hook for the LOOP aligners: every (centre[k], raw[k]) pair goes, alone, through one of the kernels that
 * produce b_compare's (lambda, hamming) without an alignment string (cluster.cpp:136-143):
 *   which = 0  k_nwrow<EXACT>   thread per pair, recorded moves + traceback        (dd_nwrow.cu)
 *   which = 1  k_nwlane         lane group per pair, software-pipelined rows        (dd_nwlane.cu)
 *   which = 2  k_nwfwd          lane-group anti-diagonal wavefront, carried lambda  (dd_nwfwd.cu)
 *   which = 3  k_nwrow<BOUND>   thread per pair, substitution count only (lambda[k] is left 0)
 * njobs_hint is the round size k_nwfwd picks its instantiation from, as in a run (above num_sms * 512: the "big" G = 4 / ND = 10
 * kernel for the narrowest slot class); the other kernels ignore it.
 * handled[k] = 0 when the kernel does not take the pair (lengths differ, band not instantiated, shared memory too small, ...) and
 * hands it on. */
int dada2b_test_loop_nw(dada2b_ctx *ctx, int32_t which, int32_t npairs, const uint32_t *centre, const uint32_t *raw, const double *err,
                        int32_t Q, const dada2b_opts *opts, uint64_t njobs_hint, double *lambda, int32_t *nsubs, int32_t *handled,
                        char errbuf[DADA2B_ERRLEN]);

/* Stage hook for the k-mer screen of one round (raw_align's shroud / gapless / NW decision, nwalign_endsfree.cpp:44-56, with the
 * greedy skip of cluster.cpp:127-131): centre `centre` against every raw r with r % world == rank, through the round's own launch
 * sequence.  opts->greedy, centre_reads and lock[nraw] (NULL: no raw locked) drive the skip; kdist_cutoff is passed separately, as
 * in the round.  max_sms caps the SM count the launches size their grids from (0: the context's).  path 0 is the product's selection
 * (k_prescreen -> k_kord, k_classify for raws whose repeat list overflowed; k_classify alone when kdist_cutoff >= 1), path 1
 * k_classify alone.  Per raw, nraw entries each:
 *   kind[r]   -1 raw of another rank, 0 neither gapless nor NW (shrouded or skipped), 1 gapless, 2 NW
 *   minsum[r] the min-sum k_prescreen handed on (0xFFFF: repeat list overflowed), -1 when the raw was no candidate
 * counters: CTR_ALIGN, CTR_SHROUD, CTR_GL, CTR_NW of the round.  Fails when a raw appears twice or a raw of another rank appears. */
int dada2b_test_screen(dada2b_ctx *ctx, uint32_t centre, const dada2b_opts *opts, double kdist_cutoff, uint32_t centre_reads,
                       const uint8_t *lock, int32_t rank, int32_t world, int32_t max_sms, int32_t path, int32_t *kind, int32_t *minsum,
                       int64_t *counters, char errbuf[DADA2B_ERRLEN]);

/* Per-raw factors of the two-phase loop NW's bound (DESIGN.md 9.3): k_raw_bounds for the raws r with r % world == rank, as a run
 * launches it.  S[r] = product over the raw's positions of its self-transition factor, rho[r] = largest substitution / self ratio at
 * the raw's (base, quality) positions; nraw entries each, NaN for the raws of other ranks. */
int dada2b_test_raw_bounds(dada2b_ctx *ctx, const double *err, int32_t Q, int32_t use_quals, int32_t rank, int32_t world, double *S, double *rho,
                           char errbuf[DADA2B_ERRLEN]);

/* Stage hook for the bound pass of a round: ONE launch of one bound-testing loop kernel over the job list jobs[njobs] (distinct raws)
 * against `centre`, as cluster `cluster_i` >= 1 compares them, with E_minmax[r] = e_minmax[r] (nraw entries) going in:
 *   which = 0  k_nwrow<BOUND>   (no lane-size early return)       which = 2  k_nwfwd, bound pass (njobs_hint picks the instantiation)
 *   which = 1  k_nwlane (njobs <= its lane_max)                     which = 3  k_gapless_loop with the bound
 * Per job: outcome 0 dropped by the bound, 1 in the survivor list, 2 in the gapless list (diagonal survivor of k_nwrow<BOUND>),
 * 3 handed back (length differs / band does not fit), 4 stored, 5 passed the bound but the store rule did not store it;
 * nsubs (-1 if not aligned); lambda (the stored lambda, NaN if not stored).  e_after: E_minmax after the launch (nraw entries).
 * counters: survivors listed, gapless-listed, handed back, stored.  Fails when a raw appears twice over the lists, a list holds a raw
 * that is no job, or a count is out of range. */
int dada2b_test_bound(dada2b_ctx *ctx, int32_t which, uint32_t centre, uint32_t cluster_i, int64_t njobs, const uint32_t *jobs, const double *e_minmax,
                      const double *err, int32_t Q, const dada2b_opts *opts, uint64_t njobs_hint, int32_t *outcome, int32_t *nsubs, double *lambda,
                      double *e_after, int64_t *counters, char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
