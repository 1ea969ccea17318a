// Final pass, diagonal list: nsubs and the transition / cluster-quality tallies of the raws whose final alignment against their
// own centre is the main diagonal (FinalSubsParallel, Rmain.cpp:179-236; error.cpp:131-172, :225-258).  Product code.
//
// For such a raw the alignment is position p against position p for p < min(len_c, len_r) (nwalign_gapless,
// nwalign_endsfree.cpp:539-555), so its contribution is a plain integer reduction over the raw's quality row:
//   k_ft_count    one thread per listed raw: Hamming distance of the packed rows -> nsubs_final; correct raws counted per cluster
//   (scans)       member offsets and chunk offsets per cluster (dd_sort.cuh's exclusive scan)
//   k_ft_scatter  the correct raws in cluster order
//   k_final_tally one block per chunk of at most FT_CHUNK members of one cluster: thread p owns position p of the centre and sums
//                 q * reads / reads in registers, the transitions in a shared [16][ncol] histogram; one global add per
//                 (cluster, position) and per non-zero transition entry at the end
// Every sum is an integer sum (cq_sum adds the 32-bit product q * reads, as the per-column form did), so the result does not
// depend on the order the raws are visited in.
#include "dd_common.h"
#include "dd_kernels.h"
#include "dd_sort.cuh"

namespace dd2 {

namespace {

constexpr int FT_CHUNK = 512;          // members per tally block: the largest cluster is spread over many blocks
constexpr int FT_THREADS = 256;
constexpr int FT_BATCH = 8;            // members whose quality bytes / base words are loaded together
// Clusters below FT_SMEM_CL are counted / placed through shared memory first: most raws belong to the few large, early-born
// clusters, and one global atomic per raw on their counters serialises in L2.  Later (smaller) clusters go to global memory
// directly.
constexpr int FT_SMEM_CL = 64;

struct FtArgs {
  DevIn in;
  DevState st;
  const uint32_t *list;                // raws whose final alignment is the main diagonal
  const unsigned long long *count;
  int nclust, ncol;
  uint32_t *off;                       // [nclust + 1] correct listed raws per cluster -> exclusive offsets
  uint32_t *chk;                       // [nclust + 1] chunks per cluster -> exclusive offsets
  uint32_t *cur;                       // [nclust] scatter cursors
  uint32_t *ord;                       // [listed] correct raws in cluster order
};

__device__ __forceinline__ uint32_t ft_centre(const FtArgs &a, uint32_t r, uint32_t *cl) {
  *cl = a.st.cluster_of[r];
  return a.st.cl_center[*cl];
}

__global__ void __launch_bounds__(FT_THREADS) k_ft_count(FtArgs a) {
  __shared__ uint32_t s_cnt[FT_SMEM_CL];
  const unsigned long long n = *a.count;
  const int SW = a.in.SW, H = min(a.nclust, FT_SMEM_CL);
  for (int x = threadIdx.x; x < H; x += blockDim.x) s_cnt[x] = 0;
  __syncthreads();
  for (unsigned long long jb = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; jb < n; jb += (unsigned long long)gridDim.x * blockDim.x) {
    const uint32_t r = a.list[jb];
    uint32_t cl;
    const uint32_t c = ft_centre(a, r, &cl);
    const int lc = min((int)a.in.len[c], (int)a.in.len[r]);
    const uint32_t *rrow = a.in.seq2 + (size_t)r * SW, *crow = a.in.seq2 + (size_t)c * SW;
    int ns = 0;
    for (int w = 0; w * 16 < lc; w++) {             // the word loop of k_gapless_loop
      const uint32_t x = rrow[w] ^ crow[w];
      uint32_t mis = (x | (x >> 1)) & 0x55555555u;
      const int left = lc - w * 16;
      if (left < 16) mis &= (1u << (2 * left)) - 1u;
      ns += __popc(mis);
    }
    a.st.nsubs_final[r] = (uint32_t)ns;
    if (!a.st.correct[r]) continue;
    if (cl < (uint32_t)H) atomicAdd(&s_cnt[cl], 1u);
    else atomicAdd(&a.off[cl], 1u);
  }
  __syncthreads();
  for (int x = threadIdx.x; x < H; x += blockDim.x)
    if (s_cnt[x]) atomicAdd(&a.off[x], s_cnt[x]);
}

// chk[i] = chunks of cluster i (its member count is still in off[i]); the scatter cursors start at zero
__global__ void __launch_bounds__(FT_THREADS) k_ft_chunks(FtArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > a.nclust) return;
  a.chk[i] = i < a.nclust ? (a.off[i] + FT_CHUNK - 1) / FT_CHUNK : 0u;
  if (i < a.nclust) a.cur[i] = 0;
}

// one tile of blockDim raws at a time: ranks inside the tile from shared counters, one global reservation per cluster and tile
__global__ void __launch_bounds__(FT_THREADS) k_ft_scatter(FtArgs a) {
  __shared__ uint32_t s_cnt[FT_SMEM_CL], s_base[FT_SMEM_CL];
  const unsigned long long n = *a.count;
  const uint32_t H = (uint32_t)min(a.nclust, FT_SMEM_CL);
  for (uint32_t x = threadIdx.x; x < H; x += blockDim.x) s_cnt[x] = 0;
  for (unsigned long long t0 = (unsigned long long)blockIdx.x * blockDim.x; t0 < n; t0 += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long jb = t0 + threadIdx.x;
    const uint32_t r = jb < n ? a.list[jb] : 0u;
    const bool on = jb < n && a.st.correct[r];
    const uint32_t cl = on ? a.st.cluster_of[r] : 0u;
    const bool sm = on && cl < H;
    __syncthreads();                               // s_cnt is clear (start, or the previous tile's reset)
    uint32_t lr = 0;
    if (sm) lr = atomicAdd(&s_cnt[cl], 1u);
    else if (on) a.ord[a.off[cl] + atomicAdd(&a.cur[cl], 1u)] = r;
    __syncthreads();
    if (sm && lr == 0) s_base[cl] = atomicAdd(&a.cur[cl], s_cnt[cl]);
    __syncthreads();
    if (sm) a.ord[a.off[cl] + s_base[cl] + lr] = r;
    __syncthreads();
    if (sm && lr == 0) s_cnt[cl] = 0;
  }
}

__global__ void __launch_bounds__(FT_THREADS) k_final_tally(FtArgs a) {
  extern __shared__ int s_trans[];                 // [16][ncol]
  __shared__ uint32_t s_r[FT_CHUNK], s_rd[FT_CHUNK];
  __shared__ uint16_t s_lc[FT_CHUNK];
  const int ncol = a.ncol, SW = a.in.SW, QS = a.in.QS, maxlen = a.in.maxlen;
  const uint32_t nchunks = a.chk[a.nclust];
  if (blockIdx.x >= nchunks) return;
  for (int x = threadIdx.x; x < 16 * ncol; x += blockDim.x) s_trans[x] = 0;
  for (uint32_t g = blockIdx.x; g < nchunks; g += gridDim.x) {
    // the chunk's cluster: the last one whose first chunk is at or below g (clusters without chunks share their offset)
    int lo = 0, hi = a.nclust;                     // chk[lo] <= g < chk[hi]
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (a.chk[mid] <= g) lo = mid; else hi = mid; }
    const uint32_t cl = (uint32_t)lo, c = a.st.cl_center[cl];
    const uint32_t m0 = a.off[cl] + (g - a.chk[cl]) * FT_CHUNK, m1 = min(m0 + FT_CHUNK, a.off[cl + 1]);
    const int nm = (int)(m1 - m0), lenc = (int)a.in.len[c];
    __syncthreads();                               // the previous chunk's members are no longer read
    for (int k = threadIdx.x; k < nm; k += blockDim.x) {
      const uint32_t r = a.ord[m0 + k];
      s_r[k] = r; s_rd[k] = a.in.reads[r]; s_lc[k] = (uint16_t)min(lenc, (int)a.in.len[r]);
    }
    __syncthreads();
    const uint32_t *crow = a.in.seq2 + (size_t)c * SW;
    for (int p = threadIdx.x; p < lenc; p += blockDim.x) {
      const uint32_t nt0 = (crow[p >> 4] >> (2 * (p & 15))) & 3u;
      unsigned long long qsum = 0, rsum = 0;
      for (int k0 = 0; k0 < nm; k0 += FT_BATCH) {
        // the batch's loads are all issued before the first shared atomic: one memory latency per FT_BATCH members
        uint32_t qv[FT_BATCH], bw[FT_BATCH];
#pragma unroll
        for (int u = 0; u < FT_BATCH; u++) {
          const int k = k0 + u;
          const bool on = k < nm && p < s_lc[k];
          const uint32_t r = on ? s_r[k] : 0u;
          qv[u] = on ? (uint32_t)a.in.qual[(size_t)r * QS + p] : 0xFFFFFFFFu;
          bw[u] = on ? a.in.seq2[(size_t)r * SW + (p >> 4)] : 0u;
        }
#pragma unroll
        for (int u = 0; u < FT_BATCH; u++) {
          if (qv[u] == 0xFFFFFFFFu) continue;
          const uint32_t qa = qv[u], rd = s_rd[k0 + u], nt1 = (bw[u] >> (2 * (p & 15))) & 3u;
          if (qa < (uint32_t)ncol) atomicAdd(&s_trans[(nt0 * 4 + nt1) * ncol + qa], (int)rd);
          qsum += (unsigned long long)(qa * rd);
          rsum += rd;
        }
      }
      if (rsum) {
        atomicAdd(&a.st.cq_sum[(size_t)cl * maxlen + p], qsum);
        atomicAdd(&a.st.cq_cnt[(size_t)cl * maxlen + p], rsum);
      }
    }
  }
  __syncthreads();
  for (int x = threadIdx.x; x < 16 * ncol; x += blockDim.x)
    if (s_trans[x]) atomicAdd(&a.st.trans[x], s_trans[x]);
}

__device__ __forceinline__ void ct_add(uint32_t *t, size_t stride, uint32_t rd, bool ok, uint32_t ns) {
  atomicMax(&t[4 * stride], rd);
  if (!ok) return;
  atomicAdd(&t[0], rd);
  atomicAdd(&t[3 * stride], 1u);
  if (ns == 0) atomicAdd(&t[stride], rd);
  else if (ns == 1) atomicAdd(&t[2 * stride], rd);
}

// One thread per raw of this rank (raw r with r % world == rank): the per-cluster tallies of $clustering (error.cpp:9-52) and
// $map (Rmain.cpp:239-279).  tl = [abundance | n0 | n1 | nunq | largest reads of any member] x nclust, zeroed by the caller.
// map[r] = cluster + 1 where correct, INT_MIN where not, 0 for the other ranks' raws (a sum all-reduce completes it).
// Sums wrap modulo 2^32 like the int32 sums they restate; every result is an integer sum or maximum, so order-independent.
__global__ void __launch_bounds__(FT_THREADS) k_cluster_tally(DevIn in, DevState st, int nclust, int rank, int world, uint32_t *tl, int32_t *map) {
  __shared__ uint32_t s_tl[5 * FT_SMEM_CL];
  const uint32_t H = (uint32_t)min(nclust, FT_SMEM_CL);
  for (int x = threadIdx.x; x < 5 * FT_SMEM_CL; x += blockDim.x) s_tl[x] = 0;
  __syncthreads();
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < in.nraw; r += gridDim.x * blockDim.x) {
    if (r % world != rank) { map[r] = 0; continue; }
    const uint32_t cl = st.cluster_of[r], rd = in.reads[r], ns = st.nsubs_final[r];
    const bool ok = st.correct[r] != 0;
    map[r] = ok ? (int32_t)cl + 1 : INT_MIN;
    if (cl < H) ct_add(&s_tl[cl], FT_SMEM_CL, rd, ok, ns);
    else ct_add(&tl[cl], (size_t)nclust, rd, ok, ns);
  }
  __syncthreads();
  for (uint32_t x = threadIdx.x; x < 5 * H; x += blockDim.x) {
    const uint32_t k = x / H, cl = x % H, v = s_tl[k * FT_SMEM_CL + cl];
    if (!v) continue;
    if (k == 4) atomicMax(&tl[4 * (size_t)nclust + cl], v);
    else atomicAdd(&tl[k * (size_t)nclust + cl], v);
  }
}

}  // namespace

void launch_cluster_tally(const DevIn &in, const DevState &st, int nclust, int rank, int world, uint32_t *tl, int32_t *map, int num_sms, cudaStream_t s) {
  const int grid = std::max(1, std::min((in.nraw + FT_THREADS - 1) / FT_THREADS, num_sms * 8));
  k_cluster_tally<<<grid, FT_THREADS, 0, s>>>(in, st, nclust, rank, world, tl, map);
  count_launch(1);
}

size_t final_tally_scan_words(int nclust) { return ((size_t)nclust + 1 + 1023) / 1024; }

void launch_final_tally(const DevIn &in, const DevState &st, const uint32_t *list, const unsigned long long *count, unsigned long long upper,
                        int nclust, int ncol, uint32_t *off, uint32_t *chk, uint32_t *cur, uint32_t *ord, uint32_t *scan_sums, int num_sms,
                        cudaStream_t s) {
  if (upper == 0) return;
  FtArgs a{in, st, list, count, nclust, ncol, off, chk, cur, ord};
  const int grid = (int)std::min<unsigned long long>((upper + FT_THREADS - 1) / FT_THREADS, (unsigned long long)num_sms * 8);
  const size_t n1 = (size_t)nclust + 1, nb = final_tally_scan_words(nclust);
  k_ft_count<<<grid, FT_THREADS, 0, s>>>(a);
  k_ft_chunks<<<(unsigned)((n1 + FT_THREADS - 1) / FT_THREADS), FT_THREADS, 0, s>>>(a);
  for (uint32_t *v : {off, chk}) {                 // exclusive scans, in place (Sorter::scan's three steps)
    k_scan1<<<(unsigned)nb, 256, 0, s>>>(v, v, scan_sums, n1);
    k_scan2<<<1, 1024, 0, s>>>(scan_sums, nb);
    k_scan3<<<(unsigned)nb, 256, 0, s>>>(v, scan_sums, n1);
  }
  k_ft_scatter<<<grid, FT_THREADS, 0, s>>>(a);
  const unsigned long long chunks_max = (upper + FT_CHUNK - 1) / FT_CHUNK + (unsigned long long)nclust;
  const int tgrid = (int)std::min<unsigned long long>(chunks_max, (unsigned long long)num_sms * 8);
  k_final_tally<<<tgrid, FT_THREADS, (size_t)16 * ncol * 4, s>>>(a);
  count_launch(10);
}

}  // namespace dd2
