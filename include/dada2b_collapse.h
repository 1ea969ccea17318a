/* dada2b_collapse.h -- C-ABI of the H100-native core of collapseNoMismatch (libdada2b.so).
 *
 * collapseNoMismatch (R/multiSample.R:104-160) merges the columns of a sequence table whose sequences are identical up to
 * shifts and length.  Its inner loop (:125-144) tries each query, in order of decreasing column sum, against the output
 * sequences kept so far, in the order they were kept, and collapses it into the first one that passes
 *     grepl(substr(query, 1, minOverlap), ref, fixed=TRUE) || grepl(substr(ref, 1, minOverlap), query, fixed=TRUE)
 * and  nwhamming(query, ref, vec=vec, band=band) == 0      (R/misc.R:216-220: nwalign, then C_eval_pair's mismatch + indel)
 * This boundary replaces that loop with one call: the device decides, for every pair (i < j) of the query-ordered
 * sequences that passes the prefix screen, whether nwhamming(seq j, seq i) is 0, and the host resolves the greedy order
 * from those pairs.  Steps 1-2 (duplicate columns, query order) and 5 (output columns, ordering) stay with the caller.
 * The Rcpp shim is in INTEGRATION.md 2f.
 *
 * Sequences are A/C/G/T text (packed into 2 bits on the device); anything else is an error.  The reference compares raw
 * characters with vec=TRUE and would accept other letters.  Returns 0 on success, non-zero with a message in errbuf;
 * nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_COLLAPSE_H
#define DADA2B_COLLAPSE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

typedef struct {
  int32_t min_overlap;             /* minOverlap (20); <= 0 screens every pair in                                    */
  int32_t match, mismatch, gap_p;  /* getDadaOpt("MATCH"/"MISMATCH"/"GAP_PENALTY") = 5 / -4 / -8                     */
  int32_t band;                    /* nwhamming's band (-1 = unbanded, the default)                                  */
  int32_t vec;                     /* 1: nwalign_vectorized2 (C_nwvec, int16 scores), 0: nwalign_endsfree (C_nwalign) */
} dada2b_collapse_opts;

/* Work counters and timings of one call (information only). */
typedef struct {
  int64_t n_candidates;            /* pairs that passed the prefix screen                                             */
  int64_t n_filtered;              /* candidates the exact overlap filter proved to have nwhamming > 0                */
  int64_t n_aligned;               /* candidates aligned (n_candidates - n_filtered)                                  */
  int64_t n_zero;                  /* aligned pairs with nwhamming == 0                                               */
  int64_t n_cells;                 /* NW cells updated                                                                */
  int64_t n_blocks;                /* candidate blocks (each sized to the device-memory budget)                       */
  int64_t gpu_launches;
  double ms_device;                /* CUDA-event time of the device work                                              */
  double ms_k_align;               /* CUDA-event time summed over the alignment kernel's launches                     */
  double ms_total;                 /* host wall time of the call                                                      */
} dada2b_collapse_stats;

void dada2b_collapse_default_opts(dada2b_collapse_opts *opts);   /* 20, 5 / -4 / -8, band -1, vec 1 */

/* Sequences come in query order (decreasing column sum, ties in column order) and without duplicates.
 * rep: caller-allocated int32[nseq]; rep[j] = the position of the sequence that j collapses into, or j if j opens a new
 * output column.  stats may be NULL. */
int dada2b_collapse_nomismatch(int32_t nseq, const char *seq_concat, const int64_t *seq_off, const dada2b_collapse_opts *opts,
                               int32_t device, int32_t *rep, dada2b_collapse_stats *stats, char errbuf[DADA2B_ERRLEN]);

/* Stage hook for the tests: for each pair x, s1 = sequence query[x], s2 = sequence ref[x]:
 *   out3[x][0] = the prefix screen (1 = passes),
 *   out3[x][1] = the overlap filter's verdict (1 = needs alignment, 0 = proved nwhamming > 0),
 *   out3[x][2] = nwhamming(s1, s2), always aligned on the device whatever the two verdicts. */
int dada2b_test_collapse_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *query,
                               const int32_t *ref, const dada2b_collapse_opts *opts, int32_t device, int32_t *out3,
                               char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
