/* dada2b_qprofile.h -- C-ABI of the H100-native read-quality profile (libdada2b.so).
 *
 * plotQualityProfile (R/plot-methods.R:163-243) draws ShortRead's qa(f, n)$perCycle$quality: for every cycle (base
 * position) and quality score, the number of bases of the sampled reads with that score at that cycle.
 * dada2b_quality_profile computes that table for one read set on the device; sampling, fastq parsing and the per-cycle
 * summaries stay on the host (dada2_b200/qc.py).  The Rcpp shim is in INTEGRATION.md 2n.
 *
 * Input is dada2b_derep_in's layout: only nreads, seq_off and qual_concat are read, and seq_concat may be NULL.
 * Qualities are numeric 0..93 (Phred+33 already removed); any other value is refused before anything is counted.  Zero
 * reads and zero-length reads are valid: a zero-length read counts in nreads and adds nothing to counts.  Returns 0 on
 * success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_QPROFILE_H
#define DADA2B_QPROFILE_H
#include <stdint.h>
#include "dada2b_derep.h"

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

#define DADA2B_QPROFILE_NSCORE 94      /* scores 0..93: one row of counts                                              */

typedef struct {
  int32_t ncycles;                     /* longest read tallied (0 if every read is empty)                              */
  int64_t *counts;                     /* [ncycles * 94]: number of bases with quality s at cycle c (c 0-based), at
                                          counts[c * 94 + s]                                                           */
  int64_t nreads, nbases;
  /* work counters and timings (information only), as in dada2b_filter_out */
  int64_t gpu_launches, h2d_bytes, d2h_bytes, kernel_bytes;
  double ms_h2d, ms_kernels, ms_d2h, ms_device, ms_total;
} dada2b_qprofile_out;

int dada2b_quality_profile(const dada2b_derep_in *reads, int32_t device, dada2b_qprofile_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_qprofile_free(dada2b_qprofile_out *out);

#ifdef __cplusplus
}
#endif
#endif
