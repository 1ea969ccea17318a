// Kernel argument blocks + launch wrappers (product code).
#pragma once
#include "dd_common.h"
#include <algorithm>
#include <cstdlib>

namespace dd2 {

enum AlignMode : int { MODE_LOOP = 0, MODE_FINAL = 1, MODE_BIRTH = 2 };

struct ClassifyArgs {
  DevIn in;
  AlnParams P;
  int mode;                 // 0: centre_idx vs all raws; 1: block b = pair b
  uint32_t centre_idx, centre_reads;
  int greedy;
  const uint8_t *lock;
  const uint32_t *pair_centre, *pair_raw;
  uint32_t *nw_list, *gl_list;
  unsigned long long *ctr;
  uint8_t *kind_out;
  int kord_words;           // words reserved for the centre's ordered 5-mers
  int shard_rank, shard_world;
  const uint32_t *cand_list;             // mode 0: raws left undecided by k_prescreen (NULL: every raw of this rank)
  const unsigned long long *cand_count;
};
// dd_prescreen.cu: streaming first tier of the k-mer screen (TMA-staged 5-mer presence bitmaps)
void launch_kmer_bits(const DevIn &in, int rank, int world, int nown, uint32_t *kbits, uint32_t *kmeta, uint16_t *krep, unsigned *n_overflow, int num_sms, cudaStream_t s);
void launch_prescreen(const DevIn &in, const uint32_t *kbits, const uint32_t *kmeta, const uint16_t *krep, int nown, int rank, int world,
                      uint32_t centre_idx, uint32_t centre_reads, int greedy, const uint8_t *lock, double kdist_cutoff, uint32_t *cand_list,
                      uint16_t *cand_ms, unsigned long long *cand_count, unsigned long long *ctr, int num_sms, cudaStream_t s);
void launch_kord(const DevIn &in, const AlnParams &P, uint32_t centre_idx, const uint32_t *cand_list, const uint16_t *cand_ms,
                 const unsigned long long *cand_count, uint32_t *nw_list, uint32_t *gl_list, uint32_t *old_list, unsigned long long *old_count,
                 unsigned long long *ctr, unsigned long long upper, int num_sms, cudaStream_t s);

struct AlignArgs {
  DevIn in;
  AlnParams P;
  DevState st;
  const uint32_t *jobs;                 // job list (NULL => job = 0..njobs-1)
  const unsigned long long *njobs_ptr;  // device-side count (NULL => njobs_fixed)
  int njobs_fixed;
  int job_mul, job_add;                 // jobs == NULL: raw index = job * job_mul + job_add (owned raws of a sharded run)
  int kind;                             // KIND_NW or KIND_GAPLESS for every job of this launch
  uint32_t centre_idx, centre_reads, cluster_i, total_reads;   // LOOP
  const uint32_t *pair_centre, *pair_raw;                      // BIRTH
  uint32_t *b_nsubs, *b_nops;
  uint16_t *b_pos;
  uint8_t *b_nt0, *b_nt1, *b_q1, *b_ops;
  double *b_lambda;
  int b_cap, b_opcap;
  // per-warp shared-memory layout (32-bit words) and pointer-matrix placement
  int warp_words, seq_bytes, H_words, ops_words;
  int ptr_in_smem;
  uint32_t *ptr_scratch;
  unsigned long long ptr_words;         // words per warp in ptr_scratch
};

long long launches_count();
struct FwdArgs {
  DevIn in;
  AlnParams P;
  DevState st;
  const uint32_t *jobs;                 // raw indices to align against centre_idx
  const unsigned long long *njobs_ptr;  // device-side count
  uint32_t centre_idx, centre_reads, cluster_i, total_reads;
  uint32_t *fb_list;                    // pairs that do not fit the register band -> k_align
  unsigned long long *fb_count;
  int seq_bytes;
  int fast_ok;                          // interior fast path allowed (scores cannot approach the sentinel)
  int job_mul, job_add;                 // jobs == NULL: raw index = job * job_mul + job_add
  int mode;                             // 0 = LOOP (one centre, store rule), 1 = FINAL (own centre per raw, nsubs + path class)
  uint32_t *gl_out, *nw_out;            // FINAL: raws whose final alignment is gapless / needs a traceback
  unsigned long long *gl_count, *nw_count;
  // two-phase loop NW (bound pass): per-raw bound factors and the survivor list
  const double *raw_S, *raw_rho;
  uint32_t *surv_list;
  unsigned long long *surv_count;
  int no_cells;                         // pass 2 of the two-phase scheme: the bound pass already counted these pairs' DP cells
  uint32_t *ns_out;                     // test hook only (NULL in the product path): nsubs per raw of the bound-testing loop kernels,
                                        // bit 31 set when the pair passed the bound (k_nwlane, k_nwfwd's bound pass, k_gapless_loop)
};
bool launch_nwfwd(const FwdArgs &a, int slots_needed, unsigned long long njobs_upper, unsigned long long njobs_hint, int num_sms, cudaStream_t s,
                  bool bound_only = false);
// dd_nwrow.cu: thread-per-pair row kernel, bound pass over f.jobs (raws as long as the centre; the rest -> uneq_list)
bool launch_nwrow_bound(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, int len1, unsigned long long njobs_upper, int num_sms,
                        unsigned long long lane_max, cudaStream_t s, uint32_t *ns_out = nullptr);
// dd_nwlane.cu: G lanes per pair, bound + exact in one launch, for rounds with at most lane_max jobs
int nwlane_lanes(int band);
size_t nwlane_mv_words(int band, int maxlen, int groups);
size_t nwlane_sub_halfwords(int maxlen, int groups);
bool launch_nwlane(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, uint32_t *mv_scratch, uint16_t *sub_scratch, int len1,
                   unsigned long long lane_max, int groups_cap, cudaStream_t s);
// loop comparisons that need no DP (gapless alignments): one thread per pair, any lengths
void launch_gapless_loop(const FwdArgs &f, int use_bound, unsigned long long njobs_upper, int num_sms, cudaStream_t s);
bool launch_nwrow_final(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, unsigned long long njobs_upper, int num_sms,
                        cudaStream_t s);
// exact pass: per-thread scratch columns for the recorded moves / substitutions; the grid is capped by what was allocated
int nwrow_exact_grid(int num_sms, int nraw);
size_t nwrow_mv_words(int band, int maxlen, int grid);
size_t nwrow_sub_halfwords(int maxlen, int grid);
bool nwrow_usable(const AlnParams &P, int len1);
bool launch_nwrow_exact(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, uint32_t *mv_scratch, uint16_t *sub_scratch, int len1,
                        unsigned long long njobs_upper, int grid_cap, cudaStream_t s, unsigned long long lane_max = 0);
void launch_raw_bounds(const DevIn &in, const double *err_rowmajor, int ncol, int use_quals, double *S, double *rho, int rank, int world, cudaStream_t s);
void launch_qrows_gather(const uint8_t *qual, int QS, const uint32_t *rows, int nrows, int only_rank, int world, uint8_t *dense, cudaStream_t s);
void launch_qrows_scatter(uint8_t *qual, int QS, const uint32_t *rows, int nrows, int rank, int world, const uint8_t *dense, cudaStream_t s);
void count_launch(int n);
void launch_classify(const ClassifyArgs &a, int grid, int block, size_t smem, cudaStream_t s);
void launch_align(int mode, const AlignArgs &a, int grid, int block, size_t smem, cudaStream_t s);
cudaError_t align_set_smem(size_t bytes);

// round tail (dd_round2.cu): shuffle passes, p-update, bud scan and report of every round
struct BlkBest { unsigned long long pb, pbp; uint32_t rd, rdp, n, np; };
struct TailState {
  uint32_t *head;          // [nraw] newest stored comparison of the raw
  uint32_t *cs_prev;       // [cs_cap] the same raw's previous stored comparison (lower cluster index); chain ends at the cluster-0 entry
  int *rows;               // [MAX_PASS][row_stride] per shuffle pass: reads delta per cluster | touched flag per cluster | moves
  uint32_t cl_cap, row_stride;      // row_stride = 2 * cl_cap + 4
  uint32_t *nmove_pass;    // [MAX_PASS] moves THIS rank made in pass k of the current round
  int rank, world;         // this rank shuffles / scans raws r % world == rank only (1 rank: every raw)
  unsigned *done;          // block tickets of k_tail_final
  BlkBest *blk;            // [grid of k_tail_final] per-block bud minima
  uint32_t *blk_ties, *blk_ties_pr;   // [grid][TIE_MAX] their tie candidates
};
struct BudParams;
// largest cluster count whose per-cluster state the tail kernels can stage in shared memory (smem = true); above it, smem = false
int tail_smem_clusters_max();
int tail_grid(int nraw);
void launch_tail_link(const DevState &st, const TailState &ts, unsigned long long base, uint32_t cluster_i, int nraw, int nclust, cudaStream_t s);
void launch_tail_pass(const DevState &st, const DevIn &in, const TailState &ts, int pass, int nclust, bool smem, cudaStream_t s);
void launch_tail_final(const DevState &st, const DevIn &in, const TailState &ts, const BudParams &bp, int greedy, int detect_singletons,
                       int last_pass, int nclust, int mode, bool smem, cudaStream_t s);

void launch_bud_collect_owned(const DevState &st, const DevIn &in, const TailState &ts, const BudParams &bp, uint32_t *ties, uint32_t *ties_pr,
                              unsigned cap, cudaStream_t s);
void launch_mask_unowned(double *p, uint8_t *correct, int nraw, int rank, int world, cudaStream_t s);
void launch_posthoc_owned(const DevState &st, int nraw, unsigned long long n_entries, const int *center_cluster, uint32_t *trip_ij, double *trip_v,
                          unsigned cap, unsigned long long *count, int rank, int world, cudaStream_t s);

// per-round control kernels (dd_round.cu)
struct BudParams {
  double min_fold; int min_hamming, min_abund;
  // k_tail_final: log of the smallest p-value b_bud could still act on, plus a safety margin (raws without / with a prior);
  // +inf = always evaluate the exact tail
  double skip_log = 1e300, skip_log_prior = 1e300;
};
void launch_round_begin(const DevState &st, int apply, uint32_t r, uint32_t from, uint32_t newi, uint32_t reads_r, cudaStream_t s);
void launch_fill_f64(double *p, double v, size_t n, cudaStream_t s);
void launch_center_cluster(int *cc, const uint32_t *cl_center, int nclust, cudaStream_t s);
void launch_final_p(const DevState &st, const DevIn &in, double omegaC, cudaStream_t s);
// dd_final.cu: final pass, raws whose alignment against their own centre is the main diagonal (list / *count): nsubs_final, and
// trans / cq_sum / cq_cnt of the correct ones.  Scratch: off and chk [nclust + 1] (off zeroed by the caller), cur [nclust],
// ord [upper], scan_sums [final_tally_scan_words(nclust)].  upper bounds *count.
size_t final_tally_scan_words(int nclust);
void launch_final_tally(const DevIn &in, const DevState &st, const uint32_t *list, const unsigned long long *count, unsigned long long upper,
                        int nclust, int ncol, uint32_t *off, uint32_t *chk, uint32_t *cur, uint32_t *ord, uint32_t *scan_sums, int num_sms,
                        cudaStream_t s);
// dd_final.cu: per-cluster tallies of the final output and $map over this rank's raws.  tl [5 * nclust] (abundance, n0, n1, nunq,
// largest member reads) is zeroed by the caller; map [nraw] gets 0 for the raws of other ranks.
void launch_cluster_tally(const DevIn &in, const DevState &st, int nclust, int rank, int world, uint32_t *tl, int32_t *map, int num_sms, cudaStream_t s);
void launch_calc_pA_vec(const int *reads, const double *E, const int *prior, double *out, int n, cudaStream_t s);

}  // namespace dd2
