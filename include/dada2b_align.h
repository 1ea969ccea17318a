/* dada2b_align.h -- C-ABI of the H100-native pairwise aligner (nwalign) and of isShiftDenovo (libdada2b.so).
 *
 * nwalign (R/misc.R:179-191) aligns two sequences with C_nwalign (nwalign_endsfree, nwalign_endsfree_homo or, with
 * endsfree=FALSE, the global nwalign; evaluate.cpp:18-61) or C_nwvec (nwalign_vectorized2, nwalign_vectorized.cpp:321-343).
 * dada2b_nwalign runs a batch of such alignments, one warp per pair, and returns the two aligned rows and / or
 * C_eval_pair's (match, mismatch, indel) of each (evaluate.cpp:73-120).
 *
 * isShiftDenovo (R/chimeras.R:380-421) flags every unique that is an exact shift of a more abundant unique.
 * dada2b_shift_denovo replaces its double loop of nwalign + C_eval_pair with the prefix screen, overlap filter and
 * alignments of collapseNoMismatch's pipeline (include/dada2b_collapse.h).  The Rcpp shims are in INTEGRATION.md 2m.
 *
 * Sequences are A/C/G/T text of 1 to 9998 bases (packed into 2 bits on the device); anything else is an error, as are
 * empty sequences (the caller aligns "" itself: the other sequence against a row of gaps).  The reference compares raw
 * characters with vec=TRUE and would accept other letters.  Returns 0 on success, non-zero with a message in errbuf;
 * nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_ALIGN_H
#define DADA2B_ALIGN_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

typedef struct {
  int32_t match, mismatch, gap_p;  /* getDadaOpt("MATCH"/"MISMATCH"/"GAP_PENALTY") = 5 / -4 / -8                      */
  int32_t homo_gap_p;              /* homo_gap (-8 = gap_p: no homopolymer costs); only with endsfree=1, vec=0          */
  int32_t band;                    /* -1 = unbanded                                                                    */
  int32_t endsfree;                /* 1: free end gaps; 0: global alignment                                            */
  int32_t vec;                     /* 1: nwalign_vectorized2 (int16 scores, homo_gap_p must equal gap_p)               */
} dada2b_nwalign_opts;

/* Work counters and timings of one call (information only). */
typedef struct {
  int64_t n_pairs;                 /* pairs aligned                                                                    */
  int64_t n_cells;                 /* NW cells updated                                                                 */
  int64_t n_blocks;                /* pair blocks (each sized to the output budget)                                    */
  int64_t gpu_launches;
  double ms_device;                /* CUDA-event time of the device work                                               */
  double ms_k_align;               /* CUDA-event time summed over the alignment kernel's launches                      */
  double ms_total;                 /* host wall time of the call                                                       */
} dada2b_nwalign_stats;

void dada2b_nwalign_default_opts(dada2b_nwalign_opts *opts);     /* 5 / -4 / -8 / -8, band -1, endsfree 1, vec 0 */

/* Aligns s1 = sequence s1_idx[x] with s2 = sequence s2_idx[x] for every pair x.
 * al1 / al2 (both or neither may be NULL): caller-allocated rows.  Pair x owns the slot of len(s1) + len(s2) bytes that
 * follows the slots of pairs 0 .. x-1; its aligned rows (A/C/G/T/'-', no terminator) start there and al_len[x] holds
 * their length.  counts (may be NULL): int32[npairs][3] = C_eval_pair's match, mismatch, indel.  stats may be NULL.
 * With vec=1, scores must fit the reference's int16 arithmetic (DESIGN.md 24); larger inputs are refused. */
int dada2b_nwalign(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *s1_idx,
                   const int32_t *s2_idx, const dada2b_nwalign_opts *opts, int32_t device, char *al1, char *al2,
                   int32_t *al_len, int32_t *counts, dada2b_nwalign_stats *stats, char errbuf[DADA2B_ERRLEN]);

typedef struct {
  int32_t min_overlap;             /* minOverlap (20)                                                                  */
  int32_t match, mismatch, gap_p;  /* nwalign's scores (5 / -4 / -8)                                                   */
} dada2b_shift_opts;

typedef struct {
  int64_t n_screened;              /* unordered pairs that passed the prefix screen                                    */
  int64_t n_equal;                 /* of those, pairs of equal abundance (never compared by R)                         */
  int64_t n_candidates;            /* directed (less abundant, more abundant) pairs: n_screened - n_equal              */
  int64_t n_filtered;              /* candidates the overlap filter proved not to be shifts                            */
  int64_t n_aligned;               /* candidates aligned (n_candidates - n_filtered)                                   */
  int64_t n_flagged;               /* sequences flagged                                                                */
  int64_t n_cells;
  int64_t n_blocks;
  int64_t gpu_launches;
  double ms_device, ms_k_align, ms_total;
} dada2b_shift_stats;

void dada2b_shift_default_opts(dada2b_shift_opts *opts);         /* 20, 5 / -4 / -8 */

/* isShiftDenovo over distinct A/C/G/T sequences with int64 abundances: flag[i] = 1 iff some sequence p with
 * abund[p] > abund[i] gives, for the unbanded ends-free alignment of s1 = seq i with s2 = seq p, C_eval_pair counts with
 * match < len(i), match < len(p), match >= min_overlap, mismatch == 0 and indel == 0 (R/chimeras.R:380-411).
 * flag: caller-allocated uint8[nseq].  stats may be NULL. */
int dada2b_shift_denovo(int32_t nseq, const char *seq_concat, const int64_t *seq_off, const int64_t *abund,
                        const dada2b_shift_opts *opts, int32_t device, uint8_t *flag, dada2b_shift_stats *stats,
                        char errbuf[DADA2B_ERRLEN]);

/* Stage hook for the tests: for each pair x, s1 = sequence query[x], s2 = sequence parent[x]:
 *   out5[x][0] = the prefix screen (1 = passes),
 *   out5[x][1] = the overlap filter's verdict (1 = needs alignment, 0 = proved not a shift),
 *   out5[x][2..4] = C_eval_pair's match, mismatch, indel, always aligned on the device whatever the two verdicts. */
int dada2b_test_shift_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *query,
                            const int32_t *parent, const dada2b_shift_opts *opts, int32_t device, int32_t *out5,
                            char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
