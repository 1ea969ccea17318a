// Per-cycle quality tally on the H100 (include/dada2b_qprofile.h).  Product code.
//
// Replaces the table ShortRead's qa(f, n)$perCycle$quality hands to plotQualityProfile (R/plot-methods.R:163-243): the
// number of bases with score s at cycle c over a read set.  A histogram over (cycle, score) with 94 scores (DESIGN.md 25).
// Launch sequence of one call:
//   k_qp_check   16 bytes per thread: flags a quality above 93 (the tally indexes its table with the quality)
//   k_qp_tally   work items (read chunk x tile of QP_TILE cycles), grid-stride over the items.  Lane l of a warp owns the
//                cycles t0 + l + 32k of the tile, so one read's quality bytes load coalesced and no two lanes of a warp
//                share a counter; each base adds 1 to the block's u32 shared-memory counter of (cycle, score).  After
//                an item the block adds its non-zero counters to the u64 table in global memory and clears them.  The
//                kernel returns at once if k_qp_check flagged a quality, so nothing is counted.
//                One atomic per base was measured against run-length accumulation per lane and against per-warp
//                sub-histograms (tools/ubench/qtally.cu, DESIGN.md 25): it is the fastest of the three on uniform,
//                NovaSeq-binned and PacBio scores alike.
#include "../../include/dada2b_qprofile.h"
#include "dd_flt.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace dd2 {

constexpr int QP_NS = DADA2B_QPROFILE_NSCORE;
constexpr int QP_TILE = 128;            // cycles per work item; lane l owns cycles l + 32k, k < QP_K
constexpr int QP_K = QP_TILE / 32;
constexpr int QP_STRIDE = 95;           // shared row stride: 95 = -1 (mod 32), so 32 lanes on 32 cycles and one score use 32 banks
constexpr int QP_WARPS = 8;
constexpr int QP_U = 4;                 // reads whose bytes a warp loads before it tallies them
constexpr int QP_BLOCKS_PER_SM = 4;     // 4 x 48 640 B of shared counters fit in an SM's 228 KB
constexpr int QP_CHUNK_ALIGN = QP_WARPS * 32;

__global__ void __launch_bounds__(256) k_qp_check(const uint8_t *__restrict__ q, long long nbytes, unsigned *err) {
  const long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 16;
  if (i0 >= nbytes) return;
  bool bad = false;
  if (i0 + 16 <= nbytes) {                                  // the buffer comes from cudaMalloc: 16-byte aligned
    const uint4 v = *reinterpret_cast<const uint4 *>(q + i0);
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
    // bit 7 of a byte of (w + 0x22..) | w is set iff that byte is >= 94; a carry out of a byte >= 0xDE can only mark a
    // neighbour of a byte that is flagged anyway
    for (int k = 0; k < 4; k++) bad |= (((w[k] + 0x22222222u) | w[k]) & 0x80808080u) != 0u;
  } else {
    for (long long i = i0; i < nbytes; i++) bad |= q[i] > 93;
  }
  if (bad) atomicOr(err, 1u);
}

struct QpArgs {
  const uint8_t *q; const long long *off;
  int n, chunk, nchunks, ntiles;         // chunk: reads per item (a multiple of QP_CHUNK_ALIGN, < 2^31: u32 counters hold it)
  const unsigned *err;
  unsigned long long *counts;            // [ncycles][QP_NS]
};

__global__ void __launch_bounds__(QP_WARPS * 32) k_qp_tally(QpArgs a) {
  __shared__ unsigned h[QP_TILE * QP_STRIDE];
  if (*a.err) return;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int x = threadIdx.x; x < QP_TILE * QP_STRIDE; x += blockDim.x) h[x] = 0u;
  __syncthreads();
  const long long items = (long long)a.nchunks * a.ntiles;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int tile = (int)(it % a.ntiles), chunk = (int)(it / a.ntiles);
    const int t0 = tile * QP_TILE;
    const int r0 = chunk * a.chunk, r1 = (int)min((long long)a.n, (long long)r0 + a.chunk);
    for (int b = r0 + w * 32; b < r1; b += QP_WARPS * 32) {     // 32 consecutive reads per warp step
      const int r = b + lane;
      long long o = 0;
      int m = 0;                                                // bases of lane r's read inside this tile (<= 0: none)
      if (r < r1) { o = a.off[r]; m = (int)(a.off[r + 1] - o) - t0; }
      if (!__any_sync(FULL, m > 0)) continue;
      for (int j0 = 0; j0 < 32; j0 += QP_U) {
        int s[QP_U][QP_K];
#pragma unroll
        for (int u = 0; u < QP_U; u++) {
          const long long oj = __shfl_sync(FULL, o, j0 + u) + t0;
          const int mj = __shfl_sync(FULL, m, j0 + u);
#pragma unroll
          for (int k = 0; k < QP_K; k++) {
            const int c = k * 32 + lane;
            s[u][k] = c < mj ? (int)__ldg(a.q + oj + c) : -1;
          }
        }
#pragma unroll
        for (int u = 0; u < QP_U; u++)
#pragma unroll
          for (int k = 0; k < QP_K; k++)
            if (s[u][k] >= 0) atomicAdd(&h[(k * 32 + lane) * QP_STRIDE + s[u][k]], 1u);
      }
    }
    __syncthreads();
    for (int x = threadIdx.x; x < QP_TILE * QP_NS; x += blockDim.x) {
      const int c = x / QP_NS, sc = x - c * QP_NS;
      unsigned &hv = h[c * QP_STRIDE + sc];
      if (hv) {
        atomicAdd(a.counts + (size_t)(t0 + c) * QP_NS + sc, (unsigned long long)hv);
        hv = 0u;
      }
    }
    __syncthreads();
  }
}

// SMs the grid is sized from: the device's count, or fewer under DADA2B_SMS=<n> (test hook: with a cap of 1, one block
// walks many chunks and tiles).
static int qp_sms(int device) {
  int sms = 0;
  BCK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  if (const char *e = getenv("DADA2B_SMS")) {
    const int cap = atoi(e);
    if (cap < 1) throw BErr{"dada2b: DADA2B_SMS must be a positive integer"};
    sms = std::min(sms, cap);
  }
  return sms;
}

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_qprofile_free(dada2b_qprofile_out *o) {
  if (!o) return;
  free(o->counts);
  free(o);
}

int dada2b_quality_profile(const dada2b_derep_in *reads, int32_t device, dada2b_qprofile_out **out, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  dada2b_qprofile_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!reads || !out) throw BErr{"dada2b: NULL argument."};
    *out = nullptr;
    need_device(device);
    const int n = reads->nreads;
    if (n < 0) throw BErr{"dada2b: negative read count."};
    if (n > 0 && !reads->seq_off) throw BErr{"dada2b: NULL argument."};
    std::vector<long long> off;
    long long nbytes = 0;
    int ncycles = 0;
    if (n > 0) {
      nbytes = rebase(n, reads->seq_off, off);
      for (int r = 0; r < n; r++) ncycles = std::max(ncycles, (int)(off[r + 1] - off[r]));
    }
    if (nbytes > 0 && !reads->qual_concat) throw BErr{"dada2b: NULL argument."};
    res = (dada2b_qprofile_out *)calloc(1, sizeof(dada2b_qprofile_out));
    if (!res) throw BErr{"dada2b: out of host memory."};
    const size_t ncell = (size_t)ncycles * QP_NS;
    res->ncycles = ncycles; res->nreads = n; res->nbases = nbytes;
    res->counts = (int64_t *)calloc(std::max<size_t>(ncell, 1), 8);
    if (!res->counts) throw BErr{"dada2b: out of host memory."};
    if (nbytes > 0) {
      BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      for (auto &e : ev) BCK(cudaEventCreate(&e));
      BBuf<uint8_t> d_q; BBuf<long long> d_off; BBuf<unsigned long long> d_counts; BBuf<unsigned> d_err;
      d_q.alloc(nbytes); d_off.alloc((size_t)n + 1); d_counts.alloc(ncell); d_err.alloc(1);
      BCK(cudaEventRecord(ev[0], s));
      BCK(cudaMemcpyAsync(d_q.p, reads->qual_concat + reads->seq_off[0], nbytes, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_off.p, off.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, s));
      BCK(cudaMemsetAsync(d_counts.p, 0, ncell * 8, s));
      BCK(cudaMemsetAsync(d_err.p, 0, 4, s));
      BCK(cudaEventRecord(ev[1], s));
      const int sms = qp_sms(device);
      const int ntiles = (ncycles + QP_TILE - 1) / QP_TILE;
      const long long blocks = (long long)sms * QP_BLOCKS_PER_SM;
      // about two items per block; a chunk is a multiple of 256 reads so that every warp step but the last is full
      long long nchunks = std::max(1LL, std::min(((long long)n + QP_CHUNK_ALIGN - 1) / QP_CHUNK_ALIGN, (2 * blocks + ntiles - 1) / ntiles));
      long long chunk = ((long long)n + nchunks - 1) / nchunks;
      chunk = (chunk + QP_CHUNK_ALIGN - 1) / QP_CHUNK_ALIGN * QP_CHUNK_ALIGN;
      nchunks = ((long long)n + chunk - 1) / chunk;
      QpArgs a{d_q.p, d_off.p, n, (int)chunk, (int)nchunks, ntiles, d_err.p, d_counts.p};
      const uint8_t *qp = d_q.p; unsigned *ep = d_err.p;
      k_qp_check<<<(unsigned)((nbytes + 16 * 256 - 1) / (16 * 256)), 256, 0, s>>>(qp, nbytes, ep);
      k_qp_tally<<<(unsigned)std::min(blocks, nchunks * ntiles), QP_WARPS * 32, 0, s>>>(a);
      BCK(cudaEventRecord(ev[2], s));
      BCK(cudaMemcpyAsync(res->counts, d_counts.p, ncell * 8, cudaMemcpyDeviceToHost, s));
      unsigned err = 0;
      BCK(cudaMemcpyAsync(&err, d_err.p, 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaEventRecord(ev[3], s));
      BCK(cudaStreamSynchronize(s));
      BCK(cudaGetLastError());
      if (err) throw BErr{"dada2b: quality values must be 0..93."};
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ev[0], ev[1])); res->ms_h2d = ms;
      BCK(cudaEventElapsedTime(&ms, ev[1], ev[2])); res->ms_kernels = ms;
      BCK(cudaEventElapsedTime(&ms, ev[2], ev[3])); res->ms_d2h = ms;
      BCK(cudaEventElapsedTime(&ms, ev[0], ev[3])); res->ms_device = ms;
      res->gpu_launches = 2;
      res->h2d_bytes = nbytes + ((long long)n + 1) * 8;
      res->d2h_bytes = (long long)ncell * 8 + 4;
      // compulsory traffic: the check and the tally read every quality byte, the tally two offsets per read and tile,
      // and the table is written once
      res->kernel_bytes = 2 * nbytes + 16LL * n * ntiles + 8LL * (long long)ncell;
    }
    res->ms_total = bnow_ms() - t0;
    *out = res; res = nullptr;
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (auto &e : ev) if (e) cudaEventDestroy(e);
  if (s) cudaStreamDestroy(s);
  if (res) dada2b_qprofile_free(res);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

}  // extern "C"
