/* dada2b_filter.h -- C-ABI of the H100-native read filter (libdada2b.so).
 *
 * filterAndTrim / fastqFilter / fastqPairedFilter (R/filter.R:402-497, :613-730, :878-1141) read a fastq in chunks of n
 * reads (FastqStreamer) and apply, per read, twelve stages in a fixed order: orient.fwd, maxLen, trimLeft, trimRight,
 * truncQ, truncLen, minLen, maxN, minQ, maxEE, rm.phix (isPhiX, :1180-1187, via C_matchRef of src/filter.cpp) and
 * rm.lowcomplex (seqComplexity, :1248-1275).  dada2b_filter replaces stages 1-12 for all chunks of a file with one call:
 * the device decides every read (pair), then writes the survivors, trimmed and oriented, in the reference's output order
 * and in the layout dada2b_derep_in takes (include/dada2b_derep.h).  Parsing and writing fastq stay on the host; the Rcpp
 * shim is in INTEGRATION.md 2g.
 *
 * Reads may hold any upper-case IUPAC letter (A C G T R Y S W K M B D H V N); anything else is an error.  Qualities are
 * numeric 0..93 (Phred+33 already removed).  Returns 0 on success, non-zero with a message in errbuf; nothing throws
 * across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_FILTER_H
#define DADA2B_FILTER_H
#include <stdint.h>
#include "dada2b_derep.h"

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

/* Reason codes: 0 = kept, otherwise the first stage that removed the read (pair). */
enum {
  DADA2B_FILTER_KEPT = 0, DADA2B_FILTER_ORIENT = 1, DADA2B_FILTER_MAXLEN = 2, DADA2B_FILTER_TRIMLEFT = 3,
  DADA2B_FILTER_TRIMRIGHT = 4, DADA2B_FILTER_TRUNCQ = 5, DADA2B_FILTER_TRUNCLEN = 6, DADA2B_FILTER_MINLEN = 7,
  DADA2B_FILTER_MAXN = 8, DADA2B_FILTER_MINQ = 9, DADA2B_FILTER_MAXEE = 10, DADA2B_FILTER_PHIX = 11,
  DADA2B_FILTER_LOWCOMPLEX = 12
};
/* Bits of dada2b_filter_out.flags. */
#define DADA2B_FILTER_MATE1 1          /* the first (forward) mate failed the reason's stage                            */
#define DADA2B_FILTER_MATE2 2          /* the second (reverse) mate failed it                                           */
#define DADA2B_FILTER_FLIPPED 4        /* orient.fwd: single-end read reverse-complemented, or mates of a pair swapped  */

/* One mate's options; fastqPairedFilter's length-1 values are recycled by the caller. */
typedef struct {
  int32_t trunc_q;                     /* truncQ (2), 0..93                                                            */
  int32_t trunc_len;                   /* truncLen (0), counted from the raw read's first base                         */
  int32_t trim_left, trim_right;       /* trimLeft / trimRight (0)                                                     */
  int32_t max_len;                     /* maxLen >= 0, or -1 = Inf (the default); other negatives are refused          */
  int32_t min_len;                     /* minLen (20)                                                                  */
  int32_t max_n;                       /* maxN (0): letters other than A/C/G/T allowed                                 */
  int32_t min_q;                       /* minQ (0), applied only when minQ > truncQ                                    */
  double max_ee;                       /* maxEE, INFINITY = off (the default)                                          */
  int32_t rm_phix;                     /* rm.phix (1)                                                                  */
  int32_t reserved;
  double rm_lowcomplex;                /* rm.lowcomplex (0 = off)                                                      */
} dada2b_filter_mate_opts;

typedef struct {
  dada2b_filter_mate_opts mate[2];     /* [0] forward / single-end, [1] reverse                                       */
  const char *orient_fwd;              /* orient.fwd primer (A/C/G/T), NULL = off                                      */
  const char *phix;                    /* the phiX genome (A/C/G/T), required when any tested mate has rm_phix        */
  int64_t chunk_n;                     /* FastqStreamer's n: reads per chunk; only orient.fwd's output order depends on
                                          it.  <= 0 means one chunk.  (dada2b_derep_in.chunk_n is not read here.)      */
} dada2b_filter_opts;

typedef struct {
  int32_t nreads, nout, paired;
  uint8_t *reason;                     /* [nreads]: 0 kept, else the first stage that removed the read (pair)         */
  uint8_t *flags;                      /* [nreads]: DADA2B_FILTER_MATE1/MATE2 for that stage, DADA2B_FILTER_FLIPPED   */
  int32_t *src;                        /* [nout]: input index of each output read (pair)                              */
  char *seq_concat[2];                 /* per mate: surviving reads, trimmed and oriented, concatenated ...           */
  int64_t *seq_off[2];                 /* ... nout + 1 offsets into seq_concat and qual_concat                        */
  uint8_t *qual_concat[2];             /* numeric qualities of the same bases (reversed where the read was flipped)   */
  /* work counters and timings (information only) */
  int64_t gpu_launches, h2d_bytes, d2h_bytes;
  int64_t kernel_bytes;                /* bytes read and written by the kernels (their compulsory traffic)            */
  double ms_h2d, ms_kernels, ms_d2h;   /* CUDA-event times of the three phases                                        */
  double ms_device, ms_total;          /* CUDA-event time of the whole device work; host wall time of the call        */
} dada2b_filter_out;

void dada2b_filter_default_opts(dada2b_filter_opts *opts);   /* filterAndTrim's defaults, chunk_n 1e5, no phiX genome */

/* fwd: the reads (forward mates); rev: the reverse mates, or NULL for single-end.  Both in dada2b_derep_in's layout. */
int dada2b_filter(const dada2b_derep_in *fwd, const dada2b_derep_in *rev, const dada2b_filter_opts *opts, int32_t device,
                  dada2b_filter_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_filter_free(dada2b_filter_out *out);

/* C_matchRef(seqs, ref, word_size, non_overlapping) (src/filter.cpp:7-32): hits[i] = the number of windows of seqs[i]
 * found among the word_size-mers of the circularised ref, scanned left to right; with non_overlapping the next window
 * tested after a hit at j starts at j + word_size + 1.  word_size 1..16; ref A/C/G/T and at least word_size long. */
int dada2b_match_ref(int32_t nseq, const char *seq_concat, const int64_t *seq_off, const char *ref, int32_t word_size,
                     int32_t non_overlapping, int32_t device, int32_t *hits, char errbuf[DADA2B_ERRLEN]);

/* seqComplexity(seqs, kmerSize) without window (R/filter.R:1248-1275): the Shannon effective number of the overlapping
 * k-mers over A/C/G/T (k-mers with other letters skipped); NaN where a sequence has no such k-mer (R's NA).  kmer_size
 * 1..4; window > 0 is refused. */
int dada2b_seq_complexity(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t kmer_size, int32_t window,
                          int32_t device, double *out, char errbuf[DADA2B_ERRLEN]);

/* Stage hook for the tests: the product's per-stage values for every read of one mate (single-end options mate[0]),
 * from the launch sequence dada2b_filter runs.  start/end: the 0-based window in the oriented read after stages 2-7
 * (trim_fail = the stage 1..7 that removed the read, else 0; the later fields are 0 then).  The others are computed on
 * that window whatever stages 8-12 decide: hits per phiX strand when opts->phix is set, complexity (kmerSize 2)
 * always. */
typedef struct {
  int32_t trim_fail, flipped, start, end;
  int32_t n_other, min_q, hits_fwd, hits_rc;
  double ee, complexity;
} dada2b_filter_stage;

int dada2b_test_filter_stages(const dada2b_derep_in *reads, const dada2b_filter_opts *opts, int32_t device,
                              dada2b_filter_stage *out, char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
