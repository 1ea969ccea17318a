/* dada2b_taxonomy.h -- C-ABI of the H100-native taxonomic classifier (libdada2b.so).
 *
 * assignTaxonomy (R/taxonomy.R:65-160) classifies sequences with the naive Bayesian classifier of Wang et al. (2007):
 * 8-mers, a per-genus table of log word probabilities, the best genus by summed log probability and 100 bootstrap
 * subsamples of one eighth of the query's 8-mers.  C_assign_taxonomy2 (src/taxonomy.cpp:206-338) does the work on host
 * threads; here the table is built on the device and stays resident (dada2b_tax_db), and every query is scored against
 * every genus on the device.  The Rcpp shim is in INTEGRATION.md 2j; the contract, including the points the reference
 * leaves open (the log, ties, random draws), is DESIGN.md 21.
 *
 * Pinned here (DESIGN.md 21):
 *   table  lgk[k][g] = (float)log((double)(((float)cnt_gk + prior_k) / genus_num_plus1[g])), the log in fp64 rounded once;
 *          prior_k = (float)(((double)count_k + 0.5) / (1.0 + nref))
 *   sums   sequential fp32 sums in the reference's order (sorted k-mers; bootstrap draws in draw order)
 *   ties   among genera of equal logp the smallest mix(mix(mix(seed) + j) + ((uint64)r << 32 | g)) wins, then the smaller
 *          g; mix is the splitmix64 finaliser, j the 0-based query, g the 0-based genus, r = 0..99 the bootstrap,
 *          100 the forward and 101 the reverse-complement main sum
 *   draws  unifs (the reference's layout: query j reads unifs[j * max_arraylen + b * (arraylen / 8) + i]), or, without
 *          unifs, uniform n = (mix(mix(seed ^ 0x9E3779B97F4A7C15) + n) >> 11) * 2^-53 read with the same layout
 *
 * Returns 0 on success, non-zero with a message in errbuf; nothing throws across the ABI.  There is no CPU path.
 */
#ifndef DADA2B_TAXONOMY_H
#define DADA2B_TAXONOMY_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef DADA2B_ERRLEN
#define DADA2B_ERRLEN 256
#endif

#define DADA2B_TAX_K 8                 /* k-mer size                                                                    */
#define DADA2B_TAX_NBOOT 100           /* bootstrap replicates                                                          */
#define DADA2B_TAX_MAXKMERS 9999       /* valid 8-mers of one query (the reference's stack arrays)                      */
#define DADA2B_TAX_MINLEN 50           /* shorter queries are not classified                                            */
#define DADA2B_TAX_NA INT32_MIN        /* R's NA_integer_                                                                */

typedef struct {
  int64_t max_table_bytes;             /* 0: one resident table of all genera.  Otherwise the genera are split into chunks
                                          whose table fits, and only one chunk's table is on the device at a time (each
                                          chunk is rebuilt when a call needs it)                                         */
  int32_t chunk_genera;                /* > 0: chunks of this many genera (overrides max_table_bytes).  The environment
                                          variable DADA2B_TAX_CHUNK_GENERA=<n> overrides both                            */
  int32_t reserved;
} dada2b_tax_opts;

typedef struct {                       /* n strings concatenated, n + 1 offsets                                         */
  int32_t n, reserved;
  const char *seq_concat;
  const int64_t *seq_off;
} dada2b_tax_seqs;

typedef struct dada2b_tax_db dada2b_tax_db;    /* opaque: the table (or the references of a chunked table) on a device */

typedef struct {
  int32_t nref, ngenus, nlevel, nchunk, chunk_genera, reserved;
  int64_t table_bytes;                 /* bytes of one resident table (one chunk's when chunked)                        */
  /* work counters and timings of the build (information only) */
  int64_t gpu_launches, h2d_bytes, d2h_bytes, kernel_bytes;
  double ms_h2d, ms_kernels, ms_d2h, ms_device, ms_total;
} dada2b_tax_db_info;

typedef struct {
  int32_t nseq, nlevel;
  int32_t *tax;                        /* [nseq]: 1-based genus, DADA2B_TAX_NA for a query shorter than 50 nt           */
  int32_t *boot;                       /* [nseq][nlevel]: bootstraps agreeing with the assignment down to each level   */
  int32_t *boot_tax;                   /* [nseq][100]: 1-based genus of each bootstrap, NA as tax                       */
  float *logp;                         /* [nseq]: log probability of the assignment (of the chosen orientation); NaN   */
  uint8_t *used_rc;                    /* [nseq]: 1 when the reverse complement was chosen (try_rc)                     */
  int64_t gpu_launches, h2d_bytes, d2h_bytes, kernel_bytes;
  double ms_h2d, ms_kernels, ms_d2h, ms_device, ms_total;
} dada2b_tax_out;

void dada2b_tax_default_opts(dada2b_tax_opts *opts);     /* one resident table, no chunks */

/* refs: the references (any bytes; only A/C/G/T form k-mers).  ref_to_genus: [nref] 1-based genus of each reference.
 * genusmat: [ngenus][nlevel] row-major integer code of each genus at each level (only compared for equality). */
int dada2b_tax_db_build(const dada2b_tax_seqs *refs, const int32_t *ref_to_genus, const int32_t *genusmat, int32_t ngenus,
                        int32_t nlevel, const dada2b_tax_opts *opts, int32_t device, dada2b_tax_db **db, char errbuf[DADA2B_ERRLEN]);
int dada2b_tax_db_info_get(const dada2b_tax_db *db, dada2b_tax_db_info *info);
void dada2b_tax_db_free(dada2b_tax_db *db);

/* unifs: NULL (draws from seed) or nseq * 100 * (max_arraylen / 8) uniforms, max_arraylen = max(len - 7) over the queries
 * of at least 7 nt. */
int dada2b_tax_classify(dada2b_tax_db *db, const dada2b_tax_seqs *seqs, int32_t try_rc, const double *unifs, int64_t nunifs,
                        uint64_t seed, dada2b_tax_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_tax_free(dada2b_tax_out *out);

/* One-shot mirror of C_assign_taxonomy2: build, classify, free. */
int dada2b_assign_taxonomy(const dada2b_tax_seqs *seqs, const dada2b_tax_seqs *refs, const int32_t *ref_to_genus, const int32_t *genusmat,
                           int32_t ngenus, int32_t nlevel, int32_t try_rc, const double *unifs, int64_t nunifs, uint64_t seed,
                           int32_t device, dada2b_tax_out **out, char errbuf[DADA2B_ERRLEN]);

/* Test hooks.  dada2b_test_tax_table: out[i][m] = lgk[kmers[i]][genera[m]] (0-based genera) from the device table.
 * dada2b_test_tax_logp: out[j][0][g] / out[j][1][g] = the forward / reverse-complement main logp of query j for every
 * genus g, from the classifier's own main-sum kernel (any query length; shorter than 8 nt: 0). */
int dada2b_test_tax_table(dada2b_tax_db *db, int32_t nk, const int32_t *kmers, int32_t ng, const int32_t *genera, float *out,
                          char errbuf[DADA2B_ERRLEN]);
int dada2b_test_tax_logp(dada2b_tax_db *db, const dada2b_tax_seqs *seqs, float *out, char errbuf[DADA2B_ERRLEN]);

#ifdef __cplusplus
}
#endif
#endif
