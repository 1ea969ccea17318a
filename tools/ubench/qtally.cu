// Design measurement for k_qp_tally (dd_qprofile.cu): the product kernel, one shared-memory atomic per base, against two
// alternatives on the same inputs:
//   runs   the same layout and loop, but each lane keeps a run (score, length) per owned cycle over its warp's
//          consecutive reads and adds a run when the score changes (fewer atomics when scores repeat, as binned ones do)
//   warp   per-warp sub-histograms of a 32-cycle tile (8 x 12 KB of shared memory), one atomic per base, no two warps
//          sharing a counter; the block sums the eight before it adds to the global table
// Inputs: 5e5 x 250-nt reads with uniform scores 2..41, the same with NovaSeq's four binned values, and 1e5 PacBio-like
// reads of 1000-2500 nt with scores 0..93.  Prints each kernel's CUDA-event time (median of 20) and checks that all three
// tables are equal.  Measurement tool, not product code:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/ubench/qtally tools/ubench/qtally.cu
#include "../../dada2_b200/csrc/dd_qprofile.cu"

#include <random>

namespace dd2 {

__global__ void __launch_bounds__(QP_WARPS * 32) k_runs(QpArgs a) {
  __shared__ unsigned h[QP_TILE * QP_STRIDE];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int x = threadIdx.x; x < QP_TILE * QP_STRIDE; x += blockDim.x) h[x] = 0u;
  __syncthreads();
  const long long items = (long long)a.nchunks * a.ntiles;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int t0 = (int)(it % a.ntiles) * QP_TILE, r0 = (int)(it / a.ntiles) * a.chunk;
    const int r1 = (int)min((long long)a.n, (long long)r0 + a.chunk);
    int cur[QP_K];
    unsigned run[QP_K];
#pragma unroll
    for (int k = 0; k < QP_K; k++) { cur[k] = 0; run[k] = 0u; }
    for (int b = r0 + w * 32; b < r1; b += QP_WARPS * 32) {
      const int r = b + lane;
      long long o = 0;
      int m = 0;
      if (r < r1) { o = a.off[r]; m = (int)(a.off[r + 1] - o) - t0; }
      if (!__any_sync(FULL, m > 0)) continue;
      for (int j0 = 0; j0 < 32; j0 += QP_U) {
        int s[QP_U][QP_K];
#pragma unroll
        for (int u = 0; u < QP_U; u++) {
          const long long oj = __shfl_sync(FULL, o, j0 + u) + t0;
          const int mj = __shfl_sync(FULL, m, j0 + u);
#pragma unroll
          for (int k = 0; k < QP_K; k++) { const int c = k * 32 + lane; s[u][k] = c < mj ? (int)__ldg(a.q + oj + c) : -1; }
        }
#pragma unroll
        for (int u = 0; u < QP_U; u++)
#pragma unroll
          for (int k = 0; k < QP_K; k++) {
            const int v = s[u][k];
            if (v < 0) continue;
            if (v == cur[k]) { run[k]++; continue; }
            if (run[k]) atomicAdd(&h[(k * 32 + lane) * QP_STRIDE + cur[k]], run[k]);
            cur[k] = v; run[k] = 1u;
          }
      }
    }
#pragma unroll
    for (int k = 0; k < QP_K; k++) if (run[k]) atomicAdd(&h[(k * 32 + lane) * QP_STRIDE + cur[k]], run[k]);
    __syncthreads();
    for (int x = threadIdx.x; x < QP_TILE * QP_NS; x += blockDim.x) {
      const int c = x / QP_NS, sc = x - c * QP_NS;
      unsigned &hv = h[c * QP_STRIDE + sc];
      if (hv) { atomicAdd(a.counts + (size_t)(t0 + c) * QP_NS + sc, (unsigned long long)hv); hv = 0u; }
    }
    __syncthreads();
  }
}

constexpr int WT = 32;                   // cycles per item of k_warp
__global__ void __launch_bounds__(QP_WARPS * 32) k_warp(QpArgs a) {   // a.ntiles counts 32-cycle tiles here
  extern __shared__ unsigned hw[];       // [QP_WARPS][WT * QP_STRIDE]
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned *h = hw + w * WT * QP_STRIDE;
  for (int x = threadIdx.x; x < QP_WARPS * WT * QP_STRIDE; x += blockDim.x) hw[x] = 0u;
  __syncthreads();
  const long long items = (long long)a.nchunks * a.ntiles;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int t0 = (int)(it % a.ntiles) * WT, r0 = (int)(it / a.ntiles) * a.chunk;
    const int r1 = (int)min((long long)a.n, (long long)r0 + a.chunk);
    for (int b = r0 + w * 32; b < r1; b += QP_WARPS * 32) {
      const int r = b + lane;
      long long o = 0;
      int m = 0;
      if (r < r1) { o = a.off[r]; m = (int)(a.off[r + 1] - o) - t0; }
      if (!__any_sync(FULL, m > 0)) continue;
      for (int j0 = 0; j0 < 32; j0 += 8) {
        int s[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
          const long long oj = __shfl_sync(FULL, o, j0 + u) + t0;
          const int mj = __shfl_sync(FULL, m, j0 + u);
          s[u] = lane < mj ? (int)__ldg(a.q + oj + lane) : -1;
        }
#pragma unroll
        for (int u = 0; u < 8; u++) if (s[u] >= 0) atomicAdd(&h[lane * QP_STRIDE + s[u]], 1u);
      }
    }
    __syncthreads();
    for (int x = threadIdx.x; x < WT * QP_NS; x += blockDim.x) {
      const int c = x / QP_NS, sc = x - c * QP_NS;
      unsigned v = 0;
      for (int k = 0; k < QP_WARPS; k++) { unsigned &e = hw[k * WT * QP_STRIDE + c * QP_STRIDE + sc]; v += e; e = 0u; }
      if (v) atomicAdd(a.counts + (size_t)(t0 + c) * QP_NS + sc, (unsigned long long)v);
    }
    __syncthreads();
  }
}

}  // namespace dd2

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s\n", cudaGetErrorString(e_), #x); exit(1); } } while (0)

struct Set { const char *name; std::vector<long long> off; std::vector<uint8_t> q; };

static Set make(const char *name, int n, int lmin, int lmax, int kind, unsigned seed) {
  std::mt19937_64 g(seed);
  Set s{name, {}, {}};
  s.off.push_back(0);
  const uint8_t bins[4] = {2, 12, 23, 37};
  for (int i = 0; i < n; i++) {
    const int L = lmin + (int)(g() % (unsigned long long)(lmax - lmin + 1));
    for (int p = 0; p < L; p++) {
      const unsigned r = (unsigned)(g() % 100);
      s.q.push_back(kind == 0 ? (uint8_t)(2 + r % 40) : kind == 1 ? bins[r < 2 ? 0 : r < 7 ? 1 : r < 20 ? 2 : 3] : (uint8_t)(g() % 94));
    }
    s.off.push_back((long long)s.q.size());
  }
  return s;
}

int main() {
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaDeviceProp pr;
  CK(cudaGetDeviceProperties(&pr, 0));
  printf("device %s, %d SMs\n", pr.name, sms);
  const size_t wsmem = (size_t)QP_WARPS * WT * QP_STRIDE * 4;
  CK(cudaFuncSetAttribute(k_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem));
  Set sets[3] = {make("illumina 5e5x250 Q2-41", 500000, 250, 250, 0, 1), make("binned 5e5x250 2/12/23/37", 500000, 250, 250, 1, 2),
                 make("pacbio 1e5x1000-2500 Q0-93", 100000, 1000, 2500, 2, 3)};
  for (auto &s : sets) {
    const int n = (int)s.off.size() - 1;
    int ncyc = 0;
    for (int i = 0; i < n; i++) ncyc = std::max(ncyc, (int)(s.off[i + 1] - s.off[i]));
    uint8_t *dq; long long *doff; unsigned long long *dc; unsigned *derr;
    const size_t ncell = (size_t)ncyc * QP_NS;
    CK(cudaMalloc(&dq, s.q.size())); CK(cudaMalloc(&doff, s.off.size() * 8)); CK(cudaMalloc(&dc, ncell * 8)); CK(cudaMalloc(&derr, 4));
    CK(cudaMemcpy(dq, s.q.data(), s.q.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(doff, s.off.data(), s.off.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemset(derr, 0, 4));
    std::vector<unsigned long long> ref;
    for (int variant = 0; variant < 3; variant++) {
      const int tile = variant == 2 ? WT : QP_TILE;
      const int ntiles = (ncyc + tile - 1) / tile;
      const long long blocks = (long long)sms * (variant == 2 ? 2 : QP_BLOCKS_PER_SM);
      long long nchunks = std::max(1LL, std::min(((long long)n + QP_CHUNK_ALIGN - 1) / QP_CHUNK_ALIGN, (2 * blocks + ntiles - 1) / ntiles));
      long long chunk = ((long long)n + nchunks - 1) / nchunks;
      chunk = (chunk + QP_CHUNK_ALIGN - 1) / QP_CHUNK_ALIGN * QP_CHUNK_ALIGN;
      nchunks = ((long long)n + chunk - 1) / chunk;
      QpArgs a{dq, doff, n, (int)chunk, (int)nchunks, ntiles, derr, dc};
      const unsigned grid = (unsigned)std::min(blocks, nchunks * ntiles);
      std::vector<float> ms;
      cudaEvent_t e0, e1;
      CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
      for (int rep = 0; rep < 23; rep++) {
        CK(cudaMemset(dc, 0, ncell * 8));
        CK(cudaEventRecord(e0));
        if (variant == 0) k_qp_tally<<<grid, QP_WARPS * 32>>>(a);
        else if (variant == 1) k_runs<<<grid, QP_WARPS * 32>>>(a);
        else k_warp<<<grid, QP_WARPS * 32, wsmem>>>(a);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float t; CK(cudaEventElapsedTime(&t, e0, e1));
        if (rep >= 3) ms.push_back(t);
      }
      std::sort(ms.begin(), ms.end());
      std::vector<unsigned long long> got(ncell);
      CK(cudaMemcpy(got.data(), dc, ncell * 8, cudaMemcpyDeviceToHost));
      if (variant == 0) ref = got;
      const char *vn[3] = {"base (product)", "runs", "warp"};
      printf("%-30s %-15s median %.3f ms  min %.3f ms  %.0f GB/s of qualities  %s\n", s.name, vn[variant], ms[ms.size() / 2], ms[0],
             s.q.size() / (ms[ms.size() / 2] * 1e6), got == ref ? "table equal" : "TABLE DIFFERS");
    }
    cudaFree(dq); cudaFree(doff); cudaFree(dc); cudaFree(derr);
  }
  return 0;
}
