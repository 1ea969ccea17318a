/* dada2b_seqtab.h -- C-ABI of the H100-native sequence-table merge (libdada2b.so).
 *
 * mergeSequenceTables (R/multiSample.R:290-364) joins per-run sequence tables into one.  dada2b_merge_seqtabs does
 * everything about columns on the device: the first-occurrence union of every table's column names, the reverse-
 * complement test of tryRC (a sequence whose reverse complement occurs earlier is re-oriented), the accumulation of
 * every table's cells into the dense [nrow_out, ncol_out] result, and its column order.  Validation, messages and sample
 * names stay on the host (dada2_b200/seqtab.py), which hands over each table row's output row.  The Rcpp shim is in
 * INTEGRATION.md 2o.
 *
 * Tables are concatenated: table t has nrow[t] rows and ncol[t] columns (both >= 1).  Its column names come next in
 * names / name_off (all tables' names, table after table; name c is names[name_off[c] .. name_off[c + 1])), its rows
 * next in row_out (the 0-based output row of each row, or -1 for a row that is skipped, e.g. a duplicate row name
 * superseded by a later row of the same table), and its cells next in entries (row-major int32, >= 0).
 * Column names must be non-empty upper-case IUPAC (ACGTMRWSYKVHDBN), with or without try_rc: they are packed 4 bits per
 * letter on the device.  Any other letter is refused, and the message names it.
 *
 * R's sub-assignment is reproduced: inside one table a duplicate column name is "last wins" (the last column of that
 * name is added, the others are not), except in a table that try_rc re-oriented, where R's collapseNoMismatch(
 * identicalOnly = TRUE) sums all columns of one name.  Across tables values add up.  A result cell or column sum above
 * INT32_MAX is refused (R would return NA).
 *
 * Returns 0 on success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_SEQTAB_H
#define DADA2B_SEQTAB_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

#define DADA2B_ORDER_NONE 0
#define DADA2B_ORDER_ABUNDANCE 1               /* order(colSums(rval), decreasing = TRUE), stable                        */
#define DADA2B_ORDER_NSAMPLES 2                /* order(colSums(rval > 0), decreasing = TRUE), stable                    */

typedef struct {
  int32_t ntab;
  const int32_t *nrow, *ncol;                  /* [ntab]                                                                 */
  const char *names;                           /* column names, table after table                                        */
  const int64_t *name_off;                     /* [sum(ncol) + 1]                                                        */
  const int32_t *row_out;                      /* [sum(nrow)]: output row, -1 = skip                                     */
  const int32_t *entries;                      /* [sum(nrow[t] * ncol[t])], row-major per table                          */
  int32_t nrow_out;                            /* >= 1                                                                   */
  int32_t try_rc;
  int32_t order_by;                            /* DADA2B_ORDER_*                                                         */
} dada2b_seqtab_merge_in;

typedef struct {
  int32_t ncol_out;
  int32_t *name_src;                           /* [ncol_out]: the input column whose name output column k carries (the
                                                  first occurrence of its oriented sequence), in output order            */
  int32_t *mat;                                /* [nrow_out * ncol_out], row-major                                       */
  int64_t n_rc;                                /* distinct sequences re-oriented (R's length(rc.seqs))                   */
  /* work counters and timings (information only) */
  int64_t gpu_launches, h2d_bytes, d2h_bytes;
  double ms_h2d, ms_kernels, ms_d2h, ms_device, ms_total;
} dada2b_seqtab_merge_out;

int dada2b_merge_seqtabs(const dada2b_seqtab_merge_in *in, int32_t device, dada2b_seqtab_merge_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_merge_seqtabs_free(dada2b_seqtab_merge_out *out);

#ifdef __cplusplus
}
#endif
#endif
