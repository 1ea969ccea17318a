/* dada2b_merge.h -- C-ABI of the H100-native alignment / evaluation / consensus step of mergePairs (libdada2b.so).
 *
 * SURVEY.md 8(f4).  mergePairs (R/paired.R:150-168) runs, for every unique (forward ASV, reverse ASV) pairing of a sample,
 *     alvec <- nwalign(F, rc(R), band=-1)          -> C_nwalign(s1, s2, match, mismatch, gap_p, homo_gap_p, band, endsfree=TRUE)
 *                                                                                  /root/reference/src/evaluate.cpp:18-61
 *     C_eval_pair(alvec[1], alvec[2])              -> (match, mismatch, indel)     /root/reference/src/evaluate.cpp:73-120
 *     C_pair_consensus(alvec[1], alvec[2], prefer, trimOverhang)                   /root/reference/src/evaluate.cpp:131-174
 * one R-level call at a time (`mapply`); .Call stubs at src/RcppExports.cpp (C_nwalign, C_eval_pair, C_pair_consensus).
 * This boundary takes the whole batch of pairings in one call and fuses the three steps on the device; the aligned
 * strings themselves never leave it.  Everything else of mergePairs (pair tabulation, rc(), accept rule, sorting) stays in R.
 * Scores are the caller's (mergePairs sets MATCH 1, MISMATCH / GAP -64 for maxMismatch = 0, else -8: R/paired.R:153-157).
 * Sequences are A/C/G/T text (nwalign() rejects anything else, R/misc.R:186-188).  Returns 0 on success, non-zero with a
 * message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_MERGE_H
#define DADA2B_MERGE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

typedef struct {
  int32_t match, mismatch, gap_p;  /* C_nwalign's match / mismatch / gap_p                                        */
  int32_t homo_gap_p;              /* C_nwalign's homo_gap_p; == gap_p selects nwalign_endsfree, else ..._homo    */
  int32_t band;                    /* C_nwalign's band; -1 = unbanded (what mergePairs uses)                       */
  int32_t trim_overhang;           /* C_pair_consensus' trim_overhang (mergePairs' trimOverhang, default FALSE)    */
} dada2b_merge_opts;

typedef struct {
  int32_t npairs;
  int32_t *nmatch, *nmismatch, *nindel;   /* C_eval_pair per pairing                                              */
  char *cons_concat;                      /* C_pair_consensus per pairing, concatenated (no terminators) ...       */
  int64_t *cons_off;                      /* ... npairs + 1 offsets                                                */
  /* work counters and timings (information only) */
  int64_t n_cells, gpu_launches, h2d_bytes, d2h_bytes;
  double ms_device, ms_k_merge, ms_total;
} dada2b_merge_out;

void dada2b_merge_default_opts(dada2b_merge_opts *opts);   /* 1 / -64 / -64 / -64, band -1, trim_overhang 0 */

/* Pairing x aligns sequence s1_idx[x] (the forward ASV) with sequence s2_idx[x] (the reverse ASV, already
 * reverse-complemented by the caller as in R/paired.R:140) of one pool of nseq sequences; prefer[x] is 1 or 2
 * (R/paired.R:162); outputs are library-owned until dada2b_merge_free. */
int dada2b_merge_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *s1_idx,
                       const int32_t *s2_idx, const int32_t *prefer, const dada2b_merge_opts *opts, int32_t device,
                       dada2b_merge_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_merge_free(dada2b_merge_out *out);

/* ---- mergePairs over whole samples (R/paired.R:111-197 without the data.frame glue) ----
 * For S samples: every read's forward / reverse cluster (dadaF$map[mapF], dadaR$map[mapR]; NA propagates and NA reads are
 * dropped), the unique (forward, reverse) pairings tabulated on the device with their read counts and ordered per sample by
 * abundance descending, then first occurrence (order(abundance, decreasing = TRUE) over unique()'s rows), prefer =
 * 1 + (n0R[reverse] > n0F[forward]), one alignment per distinct (forward sequence, reverse sequence, prefer) across all
 * samples, the accept rule and blanking of rejected consensus sequences.  All maps are 1-based with NA = INT32_MIN.  Cluster
 * sequences are given as dada() reports them: the reverse ones NOT reverse-complemented (the device does rc()). */
typedef struct {
  int32_t nsamples;
  const int64_t *nreadsF, *nreadsR;       /* [S] reads per sample: lengths of derepF$map and derepR$map                    */
  const int32_t *mapF, *mapR;             /* derep maps, concatenated sample by sample                                     */
  const int32_t *nuniqF, *nuniqR;         /* [S] uniques per sample (length of dadaF$map / dadaR$map)                      */
  const int32_t *dmapF, *dmapR;           /* [sum nuniq] dada maps (unique -> cluster), concatenated                       */
  const int32_t *nclustF, *nclustR;       /* [S] clusters per sample                                                       */
  const int32_t *n0F, *n0R;               /* [sum nclust] clustering$n0, concatenated                                      */
  const char *seqF, *seqR;                /* cluster sequences, concatenated sample by sample ...                           */
  const int64_t *seqF_off, *seqR_off;     /* ... [sum nclust + 1] offsets each                                             */
} dada2b_pairs_in;

typedef struct {
  dada2b_merge_opts align;                /* scores, homo gap, trim_overhang; band must be -1                              */
  int32_t min_overlap, max_mismatch;      /* accept = nmatch >= min_overlap && nmismatch + nindel <= max_mismatch          */
  int32_t just_concatenate;               /* F + "NNNNNNNNNN" + rc(R); counts 0, prefer 0 (NA), accept 1, nothing aligned   */
} dada2b_pairs_opts;

typedef struct {
  int32_t nsamples;
  int64_t *pair_off;                      /* [S + 1] pairing offsets per sample                                            */
  int32_t *forward, *reverse, *abundance; /* per pairing, 1-based cluster indices within the sample and read count          */
  int32_t *nmatch, *nmismatch, *nindel, *prefer;
  uint8_t *accept;
  char *cons_concat;                      /* merged sequences, "" where rejected, concatenated ...                          */
  int64_t *cons_off;                      /* ... [npairings + 1]                                                            */
  /* work counters and timings (information only) */
  int64_t n_reads, n_pairings, n_aligned, n_batches, n_cells, gpu_launches, h2d_bytes, d2h_bytes;
  double ms_k_tab, ms_k_merge, ms_total;
} dada2b_pairs_out;

/* Samples are processed in batches of whole samples of at most DADA2B_PAIRS_BATCH reads (default 2^25; a larger sample runs
 * alone); the distinct alignments of all batches run in one launch at the end.  Returns 0 on success, non-zero with a
 * message in errbuf ("Non-corresponding derep-class and dada-class objects." as R/paired.R:116-119). */
int dada2b_merge_samples(const dada2b_pairs_in *in, const dada2b_pairs_opts *opts, int32_t device, dada2b_pairs_out **out,
                         char errbuf[DADA2B_ERRLEN]);
void dada2b_merge_samples_free(dada2b_pairs_out *out);

#ifdef __cplusplus
}
#endif
#endif
