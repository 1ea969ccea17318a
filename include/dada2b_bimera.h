/* dada2b_bimera.h -- C-ABI of the H100-native bimera (chimera) detection kernels (libdada2b.so).
 *
 * SURVEY.md 8(f3): the next native hot spot after dada().  Drop-in boundary for the reference's Rcpp exports
 *     Rcpp::DataFrame C_table_bimera2(IntegerMatrix mat, vector<string> seqs, double min_fold, int min_abund,
 *                                     bool allow_one_off, int min_one_off_par_dist, int match, int mismatch,
 *                                     int gap_p, int max_shift)            /root/reference/src/chimera.cpp:194-207
 *     bool C_is_bimera(string sq, vector<string> pars, bool allow_one_off, int min_one_off_par_dist,
 *                      int match, int mismatch, int gap_p, int max_shift)  /root/reference/src/chimera.cpp:18-59
 * reached from R through isBimeraDenovoTable (R/chimeras.R:236-238) and isBimera / isBimeraDenovo
 * (R/chimeras.R:43-46, :124-132); .Call stubs at src/RcppExports.cpp:54-90.  The Rcpp shim is in INTEGRATION.md.
 *
 * Conventions are the reference's: `mat` is R's integer matrix, column-major, nrow = samples, ncol = sequences
 * (mat(i,j) = vals[i + j*nrow], chimera.cpp:196-197); sequences are A/C/G/T text.  (The reference compares raw
 * characters, so it accepts any alphabet; this library packs bases into 2 bits and rejects anything but A/C/G/T.)
 * Functions return 0 on success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_BIMERA_H
#define DADA2B_BIMERA_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

/* The scalar arguments shared by C_table_bimera2 and C_is_bimera (same names, same meaning). */
typedef struct {
  double min_fold;               /* minFoldParentOverAbundance (1.5 for the table, R/chimeras.R:220); table only */
  int32_t min_abund;             /* minParentAbundance (2); table only                                           */
  int32_t allow_one_off;         /* allowOneOff (FALSE)                                                          */
  int32_t min_one_off_par_dist;  /* minOneOffParentDistance (4)                                                  */
  int32_t match, mismatch, gap_p;/* getDadaOpt("MATCH"/"MISMATCH"/"GAP_PENALTY") = 5 / -4 / -8                   */
  int32_t max_shift;             /* maxShift (16): the band of the ends-free alignment and the end-gap credit    */
  int32_t shard_rank, shard_world; /* table only, multi-GPU: this call evaluates the sequences j with j % shard_world ==
                                    shard_rank and leaves nflag / nsam of the others 0, so the element-wise SUM over the
                                    shard_world calls (one per GPU / process) is the full result; 0 / 1 = everything   */
} dada2b_bimera_opts;

/* Work counters and timings of one call (all optional information; the reference returns none of this). */
typedef struct {
  int64_t n_pairs;               /* (query, parent) alignments performed                                         */
  int64_t n_cells;               /* NW cells updated                                                             */
  int64_t gpu_launches;
  int64_t h2d_bytes, d2h_bytes;
  double ms_device;              /* CUDA-event time of the whole device pipeline                                 */
  double ms_k_align;             /* CUDA-event time summed over the alignment kernel's launches                  */
  double ms_total;               /* host wall time of the call                                                   */
} dada2b_bimera_stats;

void dada2b_bimera_default_opts(dada2b_bimera_opts *opts);

/* C_table_bimera2: nflag[j] = number of samples in which sequence j has an exact (or one-off) two-parent model among
 * the sequences that are > min_fold times as abundant (and >= min_abund) in that sample; nsam[j] = number of samples
 * with mat(i,j) > 0.  nflag / nsam: caller-allocated int32[ncol].  stats may be NULL. */
int dada2b_table_bimera(int32_t nrow, int32_t ncol, const int32_t *mat, const char *seq_concat, const int64_t *seq_off,
                        const dada2b_bimera_opts *opts, int32_t device, int32_t *nflag, int32_t *nsam,
                        dada2b_bimera_stats *stats, char errbuf[DADA2B_ERRLEN]);

/* C_is_bimera for a batch of queries (the R loop of isBimeraDenovo, R/chimeras.R:124-147, in one call): query q is
 * sequence query_idx[q]; its candidate parents are the sequences par_idx[par_off[q] .. par_off[q+1]).
 * is_bimera: caller-allocated uint8[nquery] (1 = TRUE).  min_fold / min_abund of opts are not used here (the parent
 * lists are explicit, as in the reference).  stats may be NULL. */
int dada2b_is_bimera(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t nquery,
                     const int32_t *query_idx, const int64_t *par_off, const int32_t *par_idx,
                     const dada2b_bimera_opts *opts, int32_t device, uint8_t *is_bimera, dada2b_bimera_stats *stats,
                     char errbuf[DADA2B_ERRLEN]);

/* isBimeraDenovo (R/chimeras.R:124-133) applied to every row of a table: flags(i,j) = 1 iff
 *   (mat(i,j) > 0 || zero_queries) and |P(i,j)| >= 2 and C_is_bimera(seq j, P(i,j)),
 *   P(i,j) = { k : (double)mat(i,k) > min_fold * (double)mat(i,j)  &&  (double)mat(i,k) > min_parent_abund }.
 * mat / flags: column-major nrow x ncol as in dada2b_table_bimera; flags caller-allocated uint8[nrow*ncol].
 * A one-row call with zero_queries = 1 is isBimeraDenovo on a uniques vector (R evaluates zero abundances too); a
 * per-sample table passes zero_queries = 0, because a flagged zero cell stays zero.  Each (j, k) pair is aligned at most
 * once across all rows.  opts->min_abund is not used; opts->shard_world must be 1.  Negative counts are rejected.
 * stats may be NULL. */
int dada2b_denovo_bimera(int32_t nrow, int32_t ncol, const int32_t *mat, const char *seq_concat, const int64_t *seq_off,
                         const dada2b_bimera_opts *opts, double min_parent_abund, int32_t zero_queries, int32_t device,
                         uint8_t *flags, dada2b_bimera_stats *stats, char errbuf[DADA2B_ERRLEN]);

/* Kernel-level hook for the parity tests: align each (query, parent) pair and return what chimera.cpp's get_lr
 * (:239-269) and get_ham_endsfree (:210-236) compute on the alignment.  out5: int32[npairs][5] =
 * {left, right, left_oo, right_oo, ham}; left_oo / right_oo are only defined when allow_one_off is set. */
int dada2b_test_bimera_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs,
                             const int32_t *query, const int32_t *parent, const dada2b_bimera_opts *opts, int32_t device,
                             int32_t *out5, char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
