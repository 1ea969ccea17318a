// Shared host/device declarations for libdada2b.so (product code).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace dd2 {

constexpr int KMER = 5;              // KMER_SIZE, /root/reference/src/dada.h:27
constexpr int NKMER = 1 << (2 * KMER);
constexpr unsigned HAM_NULL = 0xFFFFFFFFu;  // hamming=-1 of a NULL sub (cluster.cpp:142)

enum PairKind : int { KIND_SHROUD = 0, KIND_GAPLESS = 1, KIND_NW = 2, KIND_SKIP = 3 };

// Resident, immutable inputs (packed once per dada2b_upload).
struct DevIn {
  int nraw, maxlen, minlen;
  int SW;             // uint32 words of 2-bit bases per raw (multiple of 4 -> 16 B rows)
  int QS;             // bytes of quality per raw (multiple of 16)
  uint32_t *seq2;     // [nraw][SW]  base b of raw r: (seq2[r*SW + b/16] >> 2*(b%16)) & 3, A,C,G,T = 0..3
  uint8_t *qual;      // [nraw][QS]  (uint8_t)round(mean quality), containers.cpp:34
  uint16_t *len;      // [nraw]
  uint32_t *reads;    // [nraw]
  uint8_t *prior;     // [nraw]
};

// Alignment / screen parameters (Rmain.cpp:35-47 subset used by raw_align).
struct AlnParams {
  int match, mismatch, gap, hgap;
  int band;           // BAND_SIZE; <0 unbanded
  int homo;           // 1 => homopolymer gap penalties (nwalign_endsfree_homo)
  int sentinel;       // out-of-band fill: -9999 (nwalign_endsfree.cpp:116) or int16 fill (nwalign_vectorized.cpp:106)
  int use_kmers, gapless, sse;
  double kdist_cutoff;
  int use_quals;
  int ncol;           // columns of err
};

enum Ctr : int {
  CTR_CS_COUNT = 0,   // entries in the comparison store
  CTR_NW, CTR_GL,     // job list lengths
  CTR_ALIGN, CTR_SHROUD, CTR_NWTOT, CTR_GLTOT, CTR_CELLS,
  CTR_NMOVE, CTR_ERR, CTR_FB, CTR_NE, CTR_PMIN, CTR_RMAX, CTR_NTIE, CTR_PMIN_PR, CTR_RMAX_PR, CTR_NTIE_PR,
  CTR_UNEQ_B, CTR_UNEQ_X,   // raws handed on by the thread-per-pair NW kernels (not as long as the centre): bound pass / exact pass
  CTR_N
};

constexpr int TIE_MAX = 64;      // tie candidates reported per round without a second copy
constexpr int MAX_PASS = 10;     // MAX_SHUFFLE, /root/reference/src/dada.h:30

// Written by the device (k_tail_final) once per round, at the head of the buffer that also holds the round's move list; the
// host copies it back together with the head of the move list after a single stream synchronisation.
struct RoundReport {
  unsigned long long ctr[CTR_N];
  uint32_t pinfo[MAX_PASS + 2];   // pinfo[p+1] = moves recorded up to and including shuffle pass p
  uint32_t converged;             // last launched pass moved nothing
  uint32_t pad;
  uint32_t tie_r[TIE_MAX], tie_ham[TIE_MAX], tiep_r[TIE_MAX], tiep_ham[TIE_MAX];
  double tie_lam[TIE_MAX], tiep_lam[TIE_MAX];
  // cluster of every tie candidate and that cluster's reads after the last pass, so that the host can open the next round
  // before it has replayed this round's moves on its member arrays (dd_driver.cu: replay worker)
  uint32_t tie_cl[TIE_MAX], tie_clreads[TIE_MAX], tiep_cl[TIE_MAX], tiep_clreads[TIE_MAX];
};


// Mutable per-run state.
struct DevState {
  // per raw
  uint8_t *lock, *is_center, *slot0, *correct;
  double *E_minmax, *p, *comp_lambda;
  uint32_t *comp_ham, *cluster_of;
  // comparison store (Bi::comp of every cluster, appended round by round)
  uint32_t *cs_index, *cs_i, *cs_ham;
  double *cs_lambda;
  unsigned long long cs_cap;
  // per cluster
  uint32_t *cl_reads, *cl_center;
  uint8_t *cl_update_e, *cl_check_locks;
  // job lists
  uint32_t *nw_list, *gl_list;
  // device counters / flags (see enum Ctr)
  unsigned long long *ctr;
  // error matrix, row-major 16 x ncol (cluster.cpp:162-170)
  double *err;
  // sharded runs (one process per GPU): raw r is owned by rank r % shard_world
  int shard_rank, shard_world;
  // per-round control block, report and move list (device memory; report and moves are views of one buffer)
  uint32_t *pinfo;                  // [MAX_PASS + 2]
  uint32_t *moves;                  // [move_cap] (raw, to) pairs
  unsigned move_cap;
  RoundReport *report;
  // final-pass accumulators
  int *trans;                       // [16][ncol] row-major
  unsigned long long *cq_sum, *cq_cnt;  // [nclust][maxlen]
  uint32_t *nsubs_final;            // per raw
};



// DP cells of a banded alignment (SURVEY.md 8d): sum_i [min(len2, i + rband) - max(1, i - lband) + 1], closed form.
// (dd_nwfwd.cu / dd_nwfwd2.cu keep their own copies: their SASS is pinned to the hardware-validated build.)
__host__ __device__ inline long long band_cells_cf(int n, int m, int l, int r) {
  const long long k = (m - r < 0 ? 0 : (m - r > n ? n : m - r));
  const long long A = k * (k + 1) / 2 + k * r + (long long)(n - k) * m;
  const long long k2 = (l + 1 < 0 ? 0 : (l + 1 > n ? n : l + 1));
  const long long B = k2 + ((long long)n * (n + 1) / 2 - k2 * (k2 + 1) / 2) - (long long)l * (n - k2);
  return A - B + n;
}

constexpr int CTR_SURV = CTR_NWTOT;   // survivor count of the two-phase bound pass (slot otherwise unused by kernels)
constexpr int CTR_CAND = CTR_GLTOT;   // k_prescreen: pairs of the round that are not shrouded ...
constexpr int CTR_OLD = CTR_NE;       // ... and raws forwarded to the warp-per-pair screen (list overflow)   (all four: zeroed by k_round_begin)

enum ErrCode : int { ERR_NONE = 0, ERR_LAMBDA = 1, ERR_QUAL = 2, ERR_TRACE = 3 };

}  // namespace dd2
