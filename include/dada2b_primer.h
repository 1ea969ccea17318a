/* dada2b_primer.h -- C-ABI of the H100-native primer removal (libdada2b.so).
 *
 * removePrimers (R/filter.R:81-233) finds the forward and, when given, the reverse primer in every read of a file and
 * in its reverse complement (Biostrings' vmatchPattern, max.mismatch mismatches, no indels), flips reads whose forward
 * primer is found only on the reverse complement, drops reads missing a primer and trims each kept read to the region
 * between the primers.  dada2b_remove_primers replaces the matching block (:118-213) for one file with one call: the
 * device scans every read four times (each primer against the read and against its reverse complement), decides every
 * read and writes the kept reads, oriented and trimmed, in input order and in dada2b_derep_in's layout.  Parsing and
 * writing fastq stay on the host; the Rcpp shim is in INTEGRATION.md 2h.
 *
 * The matching rule (Biostrings' naive inexact matcher): a primer of P letters is placed with its first letter at every
 * 0-based shift from min_shift = (P <= k ? 1 - P : -k) while its end stays at most L - min_shift; a primer letter placed
 * outside the read is a mismatch; a placement with at most k mismatches is a hit at 1-based [shift + 1, shift + P], so a
 * hit may hang off either end of the read.  Letters match when they are equal (a primer of A/C/G/T only: `fixed`) or,
 * when the primer has another IUPAC letter, when their IUPAC base sets intersect (both ways: N in the read matches).
 *
 * Reads may hold any upper-case IUPAC letter (A C G T R Y S W K M B D H V N); qualities are numeric 0..93.  Returns 0 on
 * success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_PRIMER_H
#define DADA2B_PRIMER_H
#include <stdint.h>
#include "dada2b_derep.h"

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

#define DADA2B_PRIMER_MAXLEN 64        /* primers are held in one 64-bit word per base plane */

/* Reason codes. */
enum {
  DADA2B_PRIMER_KEPT = 0, DADA2B_PRIMER_NO_FWD = 1, DADA2B_PRIMER_NO_REV = 2, DADA2B_PRIMER_EMPTY = 3,
  DADA2B_PRIMER_SKIPPED = 4            /* the whole file was skipped (see dada2b_primer_out.skipped)                    */
};
/* Bits of dada2b_primer_out.flags. */
#define DADA2B_PRIMER_FLIPPED 1        /* the read was reverse-complemented (orient)                                    */
#define DADA2B_PRIMER_MULTI_FWD 2      /* several forward hits on the read's final orientation: the first was used      */
#define DADA2B_PRIMER_MULTI_REV 4      /* several reverse hits on the read's final orientation: the last was used       */

typedef struct {
  const char *primer_fwd;              /* required, 1..64 upper-case IUPAC letters                                     */
  const char *primer_rev;              /* NULL = no reverse primer                                                    */
  int32_t max_mismatch;                /* max.mismatch (2), >= 0                                                       */
  int32_t allow_indels;                /* allow.indels (0); non-zero is refused                                        */
  int32_t trim_fwd, trim_rev, orient;  /* trim.fwd, trim.rev, orient (1, 1, 1)                                         */
  int32_t reserved;
} dada2b_primer_opts;

typedef struct {
  int32_t nreads, nout;
  int32_t skipped;                     /* no read has a forward hit as read (or, with a reverse primer, no read has a
                                          reverse hit as read): R skips the file, writes nothing and reports 0 reads out */
  int32_t multi;                       /* some read has several hits in a scan R's message looks at (as read, and on the
                                          reverse complement with orient); 0 when skipped                              */
  uint8_t *reason;                     /* [nreads]: DADA2B_PRIMER_KEPT ... DADA2B_PRIMER_SKIPPED                       */
  uint8_t *flags;                      /* [nreads]: DADA2B_PRIMER_FLIPPED / MULTI_FWD / MULTI_REV                      */
  int32_t *src;                        /* [nout]: input index of each output read (increasing)                         */
  char *seq_concat;                    /* kept reads, oriented and trimmed, concatenated ...                           */
  int64_t *seq_off;                    /* ... nout + 1 offsets into seq_concat and qual_concat                         */
  uint8_t *qual_concat;                /* numeric qualities of the same bases (reversed where the read was flipped)   */
  /* work counters and timings (information only) */
  int64_t gpu_launches, h2d_bytes, d2h_bytes;
  int64_t kernel_bytes;                /* bytes read and written by the kernels (their compulsory traffic)            */
  double ms_h2d, ms_kernels, ms_d2h;   /* CUDA-event times of the three phases                                        */
  double ms_device, ms_total;          /* CUDA-event time of the whole device work; host wall time of the call        */
} dada2b_primer_out;

void dada2b_primer_default_opts(dada2b_primer_opts *opts);   /* removePrimers' defaults, no primers */

int dada2b_remove_primers(const dada2b_derep_in *reads, const dada2b_primer_opts *opts, int32_t device, dada2b_primer_out **out,
                          char errbuf[DADA2B_ERRLEN]);
void dada2b_primer_free(dada2b_primer_out *out);

/* Stage hook for the tests: for every read i, out[4 i + s] holds scan s = 0 forward primer on the read, 1 reverse primer
 * on the read, 2 forward primer on the read's reverse complement, 3 reverse primer on the reverse complement: the hit
 * count and the first and last hit (by start) in 1-based coordinates of the scanned sequence, which may be <= 0 or > L
 * (all 0 without a hit; scans 1 and 3 are 0 without a reverse primer).  From dada2b_remove_primers' launch sequence. */
typedef struct {
  int32_t count, first_start, first_end, last_start, last_end;
} dada2b_primer_hit;

int dada2b_test_primer_hits(const dada2b_derep_in *reads, const dada2b_primer_opts *opts, int32_t device, dada2b_primer_hit *out,
                            char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
