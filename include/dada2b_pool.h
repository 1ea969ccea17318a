/* dada2b_pool.h -- C-ABI of the H100-native sample pooling (libdada2b.so).
 *
 * combineDereps2 (R/multiSample.R:165-203), the front door of dada(pool = TRUE): S samples' dereplicated reads become one
 * derep.  The pooled uniques are the union of the samples' uniques, ordered by decreasing pooled abundance with ties in
 * first-seen order over the samples taken in turn (R's stable order(decreasing = TRUE)); the pooled abundance is the sum
 * of the samples' abundances; the pooled mean quality at a position is sum_s(q_s * a_s) / sum_s(a_s), accumulated from
 * 0.0 in sample order, so it equals R's and dada2_b200.derep.combineDereps2's bit for bit (NA where any occurrence has
 * NA there, including positions beyond a sample's quality columns); the samples' maps are concatenated and translated.
 *
 * Input layout, sample after sample: sequence s's uniques are entries uoff[s] .. uoff[s+1]-1 of seq_off / abund / prior,
 * uoff = prefix sums of nuniq.  Quality rows are [nuniq_s, maxlen_s] row-major (derep$quals), concatenated; every
 * unique must fit its sample's maxlen_s.  Maps are 1-based into the sample's uniques, NA_integer_ allowed, concatenated.
 * Uniques must be A/C/G/T, non-empty, shorter than 9999 and distinct within a sample.
 * Returns 0 on success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_POOL_H
#define DADA2B_POOL_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

typedef struct {
  int32_t nsamples;
  const int32_t *nuniq;         /* [nsamples] uniques per sample                                                   */
  const int32_t *maxlen;        /* [nsamples] quality columns per sample (ncol(derep$quals))                      */
  const int64_t *nmap;          /* [nsamples] length of each sample's $map                                         */
  const char *seq_concat;       /* all samples' unique sequences, concatenated                                     */
  const int64_t *seq_off;       /* sum(nuniq) + 1 offsets into seq_concat                                          */
  const int32_t *abund;         /* [sum(nuniq)] derep$uniques                                                      */
  const double *quals;          /* sum(nuniq_s * maxlen_s) doubles: each sample's derep$quals, row-major           */
  const int32_t *map;           /* [sum(nmap)] each sample's derep$map                                             */
  const uint8_t *prior;         /* [sum(nuniq)] non-zero = prior sequence; NULL = none                            */
} dada2b_pool_in;

typedef struct {
  int32_t npool, maxlen;        /* pooled uniques; maxlen = max over samples of maxlen_s                          */
  int64_t nuniq_in, nmap;       /* sum(nuniq), sum(nmap)                                                           */
  char *seq_concat;             /* pooled unique sequences, concatenated ...                                      */
  int64_t *seq_off;             /* ... npool + 1 offsets                                                           */
  int32_t *abund;               /* [npool] pooled abundances                                                       */
  double *quals;                /* maxlen x npool column-major (== [npool, maxlen] row-major); NULL unless want_quals */
  int32_t *map;                 /* [nmap] pooled $map, 1-based, NA_integer_ where the input was NA                  */
  int32_t *index;               /* [nuniq_in] 1-based pooled position of every sample-unique                       */
  uint8_t *prior;               /* [npool] OR of the input flags over each sequence's occurrences (0 without input) */
  double qmax;                  /* largest non-NA pooled mean quality (dada()'s qmax is its ceiling)               */
  /* work counters and timings (information only) */
  int64_t gpu_launches, h2d_bytes, d2h_bytes;
  double ms_h2d, ms_kernels, ms_d2h, ms_total;
} dada2b_pool_out;

int dada2b_pool(const dada2b_pool_in *in, int32_t device, int32_t want_quals, dada2b_pool_out **out, char errbuf[DADA2B_ERRLEN]);

/* Pool and leave the pooled uniques packed and RESIDENT on the device as a dada2b_ctx (include/dada2b.h) for
 * dada2b_run_resident, with the pooled prior flags: the pooled means are rounded to dada()'s uint8 on the device and
 * never reach the host unless want_quals != 0.  A dada() run on the context equals dada2b_run on dada2b_pool's output.
 * Free the context with dada2b_ctx_free. */
struct dada2b_ctx;
int dada2b_pool_resident(const dada2b_pool_in *in, int32_t device, int32_t want_quals, dada2b_pool_out **out,
                         struct dada2b_ctx **ctx, char errbuf[DADA2B_ERRLEN]);
void dada2b_pool_free(dada2b_pool_out *out);

#ifdef __cplusplus
}
#endif
#endif
