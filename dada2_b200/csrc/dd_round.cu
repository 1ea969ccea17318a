// Control kernels of the divisive loop (product code, sm_90a); the round tail (shuffle, p-update, bud scan, report) is
// dd_round2.cu.
//
//   k_round_begin     b_bud's container updates for the new cluster      cluster.cpp:315-330, containers.cpp:150-197
//   k_raw_bounds      per-raw factors of the two-phase loop NW's bound
//   k_qrows_*         quality / sequence rows of a list of raws <-> a dense buffer (sharded uploads, finish())
#include "dd_common.h"
#include "dd_kernels.h"

namespace dd2 {

void count_launch(int n);

// ---- new cluster + per-round counter reset (one thread) --------------------------------
__global__ void k_round_begin(DevState st, int apply, uint32_t r, uint32_t from, uint32_t newi, uint32_t reads_r) {
  if (threadIdx.x == 0) {
    if (apply) {   // bi_pop_raw(from) ; b_add_bi ; bi_add_raw ; bi_assign_center
      st.cluster_of[r] = newi; st.is_center[r] = 1; st.slot0[r] = 1; st.lock[r] = 0;
      st.cl_center[newi] = r;
      st.cl_reads[from] -= reads_r;
      st.cl_reads[newi] = reads_r;
      st.cl_update_e[from] = 1; st.cl_update_e[newi] = 1; st.cl_check_locks[newi] = 1;
    }
    st.ctr[CTR_NW] = 0; st.ctr[CTR_GL] = 0; st.ctr[CTR_FB] = 0; st.ctr[CTR_NMOVE] = 0;
    st.ctr[CTR_CAND] = 0; st.ctr[CTR_OLD] = 0; st.ctr[CTR_SURV] = 0; st.ctr[CTR_UNEQ_B] = 0; st.ctr[CTR_UNEQ_X] = 0;   // (no memsets in the round)
  }
  if (threadIdx.x < MAX_PASS + 2) st.pinfo[threadIdx.x] = 0;
}

// Two-phase loop NW: per-raw bound factors.  S_r = product over the raw's positions of its self-transition factor
// err[5*nt][q]; rho_r = max over positions and nt0 != nt of err[4*nt0+nt][q] / err[5*nt][q].
__global__ void k_raw_bounds(DevIn in, const double *err, int ncol, int use_quals, double *S, double *rho, int rank, int world) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) * world + rank;        // this rank's raws only (their quality rows may be the only ones uploaded)
  if (r >= in.nraw) return;
  const uint32_t *row = in.seq2 + (size_t)r * in.SW;
  const uint8_t *q = in.qual + (size_t)r * in.QS;
  double s = 1.0, rh = 0.0;
  const int L = in.len[r];
  for (int p = 0; p < L; p++) {
    const int b = (row[p >> 4] >> (2 * (p & 15))) & 3;
    const int qq = use_quals ? min((int)q[p], ncol - 1) : 0;
    const double self = err[(5 * b) * ncol + qq];
    s *= self;
    for (int a0 = 0; a0 < 4; a0++) if (a0 != b) rh = fmax(rh, err[(4 * a0 + b) * ncol + qq] / self);
  }
  S[r] = s; rho[r] = rh;
}

__global__ void k_fill_f64(double *p, double v, size_t n) {
  for (size_t x = blockIdx.x * (size_t)blockDim.x + threadIdx.x; x < n; x += (size_t)gridDim.x * blockDim.x) p[x] = v;
}
__global__ void k_center_cluster(int *cc, const uint32_t *cl_center, int nclust) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nclust) cc[cl_center[i]] = i;
}

// Quality rows of a list of raws <-> a dense buffer (16-byte units).  Sharded uploads keep a raw's quality row on its owner only
// (dd_driver.cu:do_upload); the rows of the cluster centres are exchanged before the birth subs need them.
__global__ void k_qrows_gather(const uint8_t *qual, int QS, const uint32_t *rows, int nrows, int only_rank, int world, uint8_t *dense) {
  const int u = QS / 16, x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= nrows * u) return;
  const uint32_t r = rows[x / u];
  uint4 v = make_uint4(0, 0, 0, 0);
  if (only_rank < 0 || (int)(r % (uint32_t)world) == only_rank) v = ((const uint4 *)(qual + (size_t)r * QS))[x % u];
  ((uint4 *)dense)[x] = v;
}
__global__ void k_qrows_scatter(uint8_t *qual, int QS, const uint32_t *rows, int nrows, int rank, int world, const uint8_t *dense) {
  const int u = QS / 16, x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= nrows * u) return;
  const uint32_t r = rows ? rows[x / u] : (uint32_t)(x / u) * (uint32_t)world + (uint32_t)rank;     // rows == NULL: the rank's own raws in order
  ((uint4 *)(qual + (size_t)r * QS))[x % u] = ((const uint4 *)dense)[x];
}

// ------------------------------- launch wrappers --------------------------------------
void launch_qrows_gather(const uint8_t *qual, int QS, const uint32_t *rows, int nrows, int only_rank, int world, uint8_t *dense, cudaStream_t s) {
  if (nrows <= 0) return;
  count_launch(1);
  k_qrows_gather<<<(nrows * (QS / 16) + 255) / 256, 256, 0, s>>>(qual, QS, rows, nrows, only_rank, world, dense);
}
void launch_qrows_scatter(uint8_t *qual, int QS, const uint32_t *rows, int nrows, int rank, int world, const uint8_t *dense, cudaStream_t s) {
  if (nrows <= 0) return;
  count_launch(1);
  k_qrows_scatter<<<(nrows * (QS / 16) + 255) / 256, 256, 0, s>>>(qual, QS, rows, nrows, rank, world, dense);
}
void launch_raw_bounds(const DevIn &in, const double *err_rowmajor, int ncol, int use_quals, double *S, double *rho, int rank, int world, cudaStream_t s) {
  count_launch(1);
  const int nown = (in.nraw - rank + world - 1) / world;
  k_raw_bounds<<<(nown + 127) / 128, 128, 0, s>>>(in, err_rowmajor, ncol, use_quals, S, rho, rank, world);
}
void launch_fill_f64(double *p, double v, size_t n, cudaStream_t s) {
  count_launch(1);
  k_fill_f64<<<(unsigned)std::min<size_t>((n + 255) / 256, 2048), 256, 0, s>>>(p, v, n);
}
void launch_center_cluster(int *cc, const uint32_t *cl_center, int nclust, cudaStream_t s) {
  count_launch(1);
  k_center_cluster<<<(nclust + 127) / 128, 128, 0, s>>>(cc, cl_center, nclust);
}
void launch_round_begin(const DevState &st, int apply, uint32_t r, uint32_t from, uint32_t newi, uint32_t reads_r, cudaStream_t s) {
  count_launch(1);
  k_round_begin<<<1, 32, 0, s>>>(st, apply, r, from, newi, reads_r);
}
}  // namespace dd2
