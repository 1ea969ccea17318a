/* dada2b.h -- C-ABI of the H100-native dada() core (libdada2b.so).
 *
 * Drop-in boundary: this is what a replacement for the reference's Rcpp export
 *     Rcpp::List dada_uniques(...)            /root/reference/src/Rmain.cpp:30-47
 * reached from R through
 *     .Call('_dada2_dada_uniques', ...)       /root/reference/R/RcppExports.R:8-10
 *     _dada2_dada_uniques(SEXP x28)           /root/reference/src/RcppExports.cpp:17-53
 * binds to.  Plain pointers and sizes only; no torch / CUDA types.  The Rcpp shim a
 * maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions are the reference's own (SURVEY.md 8b):
 *   - seqs are A/C/G/T text, sorted by decreasing abundance (R/sequenceIO.R:98);
 *   - quals is R's `unname(t(derep$quals))`: column-major, maxlen rows (position
 *     fastest) x nraw columns, NA/NaN beyond a read's length (R/dada.R:339);
 *   - err is column-major 16 x Q, rows A2A,A2C,..,T2T (R/dada.R:338);
 *   - every output array mirrors one column / matrix of the R list built at
 *     Rmain.cpp:294; NA_integer_ is INT32_MIN, NA_real_ is R's NaN payload 1954.
 *
 * Errors: functions return 0 on success, non-zero with a message in errbuf (the text
 * the reference passes to Rcpp::stop where one exists).  Nothing throws across the ABI.
 */
#ifndef DADA2B_H
#define DADA2B_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DADA2B_NA_INTEGER INT32_MIN
#define DADA2B_ERRLEN 256

/* Inputs of dada_uniques (Rmain.cpp:30-34). */
typedef struct {
  int32_t nraw;             /* seqs.size()                                            */
  int32_t maxlen;           /* quals.nrow(); 0 => no quality matrix (has_quals=false) */
  const char *seq_concat;   /* concatenated A/C/G/T bytes                             */
  const int64_t *seq_off;   /* nraw+1 offsets into seq_concat                         */
  const int32_t *abund;     /* abundances                                             */
  const uint8_t *prior;     /* priors (0/1); NULL => all FALSE                        */
  const double *quals;      /* maxlen x nraw column-major, NaN-padded; NULL iff maxlen==0 */
  const double *err;        /* 16 x Q column-major                                    */
  int32_t Q;                /* err.ncol()                                             */
} dada2b_in;

/* The 23 scalar arguments of dada_uniques, same order and meaning (Rmain.cpp:35-47). */
typedef struct {
  int32_t match, mismatch, gap;
  int32_t use_kmers;
  double kdist_cutoff;
  int32_t band_size;
  double omegaA, omegaP, omegaC;
  int32_t detect_singletons;
  int32_t max_clust;
  double min_fold;
  int32_t min_hamming, min_abund;
  int32_t use_quals;
  int32_t final_consensus;       /* ignored by the reference as well (R/dada.R:345) */
  int32_t vectorized_alignment;
  int32_t homo_gap;
  int32_t multithread;           /* accepted for signature parity; the GPU path is always parallel */
  int32_t verbose;
  int32_t SSE;                   /* accepted; results equal the reference's SSE=0/1/2 (identical by N1) */
  int32_t gapless, greedy;
} dada2b_opts;

/* The R list of Rmain.cpp:294, flattened. All arrays are owned by the library. */
typedef struct {
  int32_t nclust, nraw, maxlen, Q, n_birth_subs;
  /* $clustering (error.cpp:9-127), nclust rows */
  char *cl_seq_concat;      /* sequences, concatenated */
  int64_t *cl_seq_off;      /* nclust+1 */
  int32_t *cl_abundance, *cl_n0, *cl_n1, *cl_nunq;
  double *cl_pval;
  int32_t *cl_birth_from;   /* 1-based; NA for row 0 */
  double *cl_birth_pval, *cl_birth_fold;
  int32_t *cl_birth_ham;
  double *cl_birth_qave;
  /* $birth_subs (error.cpp:261-300), n_birth_subs rows */
  int32_t *bs_pos;          /* 1-based */
  char *bs_ref, *bs_sub;    /* one nucleotide letter per row */
  double *bs_qual;
  int32_t *bs_clust;        /* 1-based */
  /* $subqual 16 x Q (col-major; Q=1 without quals), $clusterquals maxlen x nclust (col-major) */
  int32_t *subqual;
  int32_t subqual_ncol;
  double *clusterquals;
  /* $map (1-based cluster or NA), $pval */
  int32_t *map;
  double *pval;
  /* diagnostics (not part of the R list): counters of Rmain.cpp:333 and timings */
  int64_t n_align, n_shroud;        /* loop: pairs screened / rejected by the k-mer screen      */
  int64_t n_nw, n_gapless;          /* loop: pairs aligned by NW / by the gapless shortcut      */
  int64_t nw_cells;                 /* DP cells filled (loop + final pass)                      */
  int64_t n_final_nw;               /* final pass: alignments (one per unique)                  */
  int32_t n_rounds, n_shuffles;
  int64_t gpu_launches;             /* kernels launched by this call                            */
  int64_t h2d_bytes, d2h_bytes;     /* bytes copied host->device / device->host by this call    */
  double ms_setup, ms_loop, ms_final, ms_total;   /* host wall clock                            */
  double ms_device;                 /* CUDA-event time, first to last device operation          */
  double ms_k_classify, ms_k_align_nw, ms_k_align_gl, ms_k_align_final;  /* CUDA-event sums per kernel family */
  int32_t n_k_classify, n_k_align_nw, n_k_align_gl, n_k_align_final;     /* launches in each sum              */
  /* finer split (ms_k_classify = prescreen + screen; ms_k_align_nw = bound + exact) and the round-control kernels */
  double ms_k_prescreen, ms_k_nw_bound, ms_k_nw_exact, ms_k_tail;
  int32_t n_k_prescreen, n_k_nw_bound, n_k_nw_exact, n_k_tail;
  int64_t prescreen_rows;           /* 5-mer bitmap rows (128 B + 13 B of per-raw metadata) streamed by k_prescreen */
  /* final pass split (ms_k_align_final = row + diag + gapped): the sweep that finds nsubs and the path class, the tally of the
   * raws whose final alignment is the main diagonal, and the traceback alignments of the rest */
  double ms_k_final_row, ms_k_final_diag, ms_k_final_gapped;
  int32_t n_k_final_row, n_k_final_diag, n_k_final_gapped;
} dada2b_out;

/* One-shot: host buffers in, host buffers out (what the Rcpp shim calls). */
int dada2b_run(const dada2b_in *in, const dada2b_opts *opts, dada2b_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_free(dada2b_out *out);

/* Resident variant: upload + pack the uniques once, then run any number of passes with
 * different err / options (the selfConsist loop of R/dada.R:256-391 calls dada_uniques
 * up to 11x on identical sequences).  in->err / in->Q are ignored by dada2b_upload. */
typedef struct dada2b_ctx dada2b_ctx;
int dada2b_upload(const dada2b_in *in, int32_t device, dada2b_ctx **ctx, char errbuf[DADA2B_ERRLEN]);
int dada2b_run_resident(dada2b_ctx *ctx, const double *err, int32_t Q, const dada2b_opts *opts,
                        dada2b_out **out, char errbuf[DADA2B_ERRLEN]);
void dada2b_ctx_free(dada2b_ctx *ctx);
/* Replace the uniques held by an existing context (keeps its buffers, stream and NCCL communicator). */
int dada2b_reupload(dada2b_ctx *ctx, const dada2b_in *in, char errbuf[DADA2B_ERRLEN]);

/* Sharded multi-GPU runs (one process per GPU).  Every rank uploads the same uniques and calls
 * dada2b_run_resident() with the same arguments; raw r is OWNED by rank r % world: that rank alone screens and aligns
 * it, keeps its stored comparisons and runs shuffle / p-update / bud scan for it.  Per shuffle pass one NCCL all-reduce
 * of the per-cluster read deltas, per split round one all-gather of the ranks' reports (bud candidates, move counts)
 * and, when raws moved, of the move lists; the final tallies are all-reduced.  Every rank returns the complete result.
 * The NCCL unique id is created on rank 0 and distributed by the caller (e.g. torch.distributed broadcast).
 * Threading: a dada2b_ctx is used by one thread at a time; dada2b_run() keeps one workspace per calling thread. */
#define DADA2B_NCCL_ID_BYTES 128
int dada2b_nccl_unique_id(char id[DADA2B_NCCL_ID_BYTES], char errbuf[DADA2B_ERRLEN]);
int dada2b_comm_init(dada2b_ctx *ctx, int32_t rank, int32_t world, const char id[DADA2B_NCCL_ID_BYTES],
                     char errbuf[DADA2B_ERRLEN]);

/* Defaults of R/dada.R:1-26 (dada_opts) as passed at R/dada.R:335-352. */
void dada2b_default_opts(dada2b_opts *opts);

#ifdef __cplusplus
}
#endif
#endif
