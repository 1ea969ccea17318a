// Bimera (chimera) detection on the H100: kernels + host driver behind include/dada2b_bimera.h.  Product code.
//
// Replaces (under /root/reference/src)
//   C_table_bimera2 / BimeraTableParallel   chimera.cpp:61-207     -> dada2b_table_bimera
//   C_is_bimera                             chimera.cpp:18-59      -> dada2b_is_bimera (batched)
//   isBimeraDenovo's loop, every table row  R/chimeras.R:124-133   -> dada2b_denovo_bimera
//   get_lr, get_ham_endsfree                chimera.cpp:210-269    -> bim_scan (on the traceback's 2-bit move string)
// The alignment is the reference's nwalign_vectorized2(query, parent, match, mismatch, gap_p, end_gap 0, band max_shift)
// (chimera.cpp:27, :122): the warp-per-pair banded ends-free NW of dd_nw_warp.cuh (bit-exact alignments, same kernel
// family as the final pass of dada()).
//
// Pipeline of the table call, per batch of JB query sequences (all stream-ordered, no host synchronisation inside):
//   k_bim_need    thread per (query j, candidate k): is k a parent of j in ANY sample?  (chimera.cpp:121-123: the
//                 reference aligns a pair the first time a sample needs it)  -> compact job list, warp-aggregated append
//   k_bim_align   warp per job: NW + traceback, then get_lr / get_ham_endsfree on bit masks of the alignment columns
//                 -> one packed 64-bit record per (j, k)
//   k_bim_flag    CTA per query, warp per sample: max of left / right (+ one-off variants) over the parents eligible
//                 in that sample (coalesced reads of the sample-major count table and of the record row) -> nflag, nsam
// The de novo call runs the same pipeline with isBimeraDenovo's parent rule in k_bim_need and k_bim_denovo_flag in
// place of k_bim_flag: it counts the parents next to the maxima and writes one flag per (sample, query) cell.
// Integer work throughout; no tensor cores by construction.  There is NO CPU fallback.
#include "../../include/dada2b_bimera.h"
#include "dd_common.h"
#include "dd_kernels.h"
#include "dd_nw_warp.cuh"
#include "dd_bimera.cuh"
#include "dd_hostutil.h"

#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace dd2 {

__global__ void __launch_bounds__(128) k_bim_align(BimAlignArgs a) {
  extern __shared__ uint32_t smem[];
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = lane_id();
  const unsigned long long njobs = a.njobs_ptr ? *a.njobs_ptr : a.njobs_fixed;
  if ((unsigned long long)blockIdx.x * nwarps >= njobs) return;
  uint32_t *wbase = smem + (size_t)wid * a.warp_words;
  uint8_t *s1 = (uint8_t *)wbase;
  uint8_t *s2 = s1 + a.seq_bytes;
  int *H = (int *)(wbase + 2 * (a.seq_bytes >> 2));
  uint32_t *opw = (uint32_t *)(H + a.H_words);
  uint32_t *mQ = opw + a.ops_words, *mP = mQ + a.mask_words, *mE = mP + a.mask_words;
  uint32_t *ptr_s = mE + a.mask_words;
  const int gw = blockIdx.x * nwarps + wid, tw = gridDim.x * nwarps;
  uint32_t *ptr = a.ptr_in_smem ? ptr_s : a.ptr_scratch + (size_t)gw * a.ptr_words;
  int errflag = 0;
  unsigned long long cells_lane = 0;
  for (unsigned long long jx = gw; jx < njobs; jx += tw) {
    const unsigned long long jb = a.job_list ? (unsigned long long)a.job_list[jx] : jx;
    const uint32_t q = a.jq[jb], k = a.jk[jb];
    const int len1 = a.sq.len[q], len2 = a.sq.len[k];
    unpack_row(a.sq.seq2 + (size_t)q * a.sq.SW, len1, s1, false);       // s1 = query  (al[0]),  rows i
    unpack_row(a.sq.seq2 + (size_t)k * a.sq.SW, len2, s2, false);       // s2 = parent (al[1]),  columns j
    const int nops = nw_warp(s1, len1, s2, len2, a.P, H, ptr, opw, &cells_lane, &errflag);
    // column masks, forward order (the traceback wrote the moves in reverse): 1 diag, 2 gap in the query row, 3 gap in the parent row
    int i0b = 0, i1b = 0, neq = 0;
    const int nch = (nops + 31) >> 5;
    for (int ch = 0; ch < nch; ch++) {
      const int col = ch * 32 + lane;
      int op = 0;
      if (col < nops) { const int e = nops - 1 - col; op = (opw[e >> 4] >> (2 * (e & 15))) & 3; }
      const unsigned b0 = __ballot_sync(0xffffffffu, op == 1 || op == 3), b1 = __ballot_sync(0xffffffffu, op == 1 || op == 2);
      const int i0 = i0b + __popc(b0 & lanemask_lt()), i1 = i1b + __popc(b1 & lanemask_lt());
      const bool eq = op == 1 && ((s1[i0] ^ s2[i1]) & 3) == 0;
      const unsigned bq = __ballot_sync(0xffffffffu, op == 2), bp = __ballot_sync(0xffffffffu, op == 3), be = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) { mQ[ch] = bq; mP[ch] = bp; mE[ch] = be; }
      neq += __popc(be);
      i0b += __popc(b0); i1b += __popc(b1);
    }
    if (lane == 0) { mQ[nch] = 0; mP[nch] = 0; mE[nch] = 0; }
    __syncwarp();
    int v[5];
    bim_scan(mQ, mP, mE, nops, neq, a.allow_one_off != 0, a.max_shift, v);
    if (lane == 0) {
      if (a.raw5) { int32_t *o = a.raw5 + (size_t)jb * 5; o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3]; o[4] = v[4]; }
      if (a.rec) {
        const bool allowed = a.allow_one_off && v[4] >= a.min_one_off_par_dist;      // chimera.cpp:125-127
        const bool keep = v[0] + v[1] < len1;                                         // :129-142 id / pure-shift / internal-indel "parents" count as 0
        const size_t dst = a.dst_mode ? (size_t)((q - (uint32_t)a.q_add) / (uint32_t)a.q_mul - a.j0) * a.ncol + k : (size_t)jb;
        a.rec[dst] = keep ? bim_pack(v[0], v[1], a.allow_one_off ? v[2] : 0, a.allow_one_off ? v[3] : 0, allowed) : bim_pack(0, 0, 0, 0, allowed);
      }
    }
    __syncwarp();
  }
  if (errflag && lane == 0) atomicMax(&a.ctr[2], (unsigned long long)errflag);
  {
    unsigned cl = (unsigned)cells_lane;
#pragma unroll
    for (int o = 16; o; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
    if (lane == 0 && cl) atomicAdd(&a.ctr[1], (unsigned long long)cl);
  }
}

// 32 x 32 tiled transpose: mat [ncol][nrow] (R's column-major nrow x ncol) -> matT [nrow][ncol] (sample-major)
__global__ void k_bim_transpose(const int32_t *mat, int32_t *matT, int nrow, int ncol) {
  __shared__ int32_t tile[32][33];
  const int i0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  for (int y = threadIdx.y; y < 32; y += blockDim.y) {
    const int k = k0 + y, i = i0 + threadIdx.x;
    if (k < ncol && i < nrow) tile[y][threadIdx.x] = mat[(size_t)k * nrow + i];
  }
  __syncthreads();
  for (int y = threadIdx.y; y < 32; y += blockDim.y) {
    const int i = i0 + y, k = k0 + threadIdx.x;
    if (i < nrow && k < ncol) matT[(size_t)i * ncol + k] = tile[threadIdx.x][y];
  }
}

struct BimTableArgs {
  const int32_t *mat, *matT;                // [ncol][nrow], [nrow][ncol]
  int nrow, ncol;
  uint32_t j0; int jb;                      // queries [j0, j0 + jb) of this batch ...
  int q_mul, q_add;                         // ... query of batch slot s is (j0 + s) * q_mul + q_add (sharded calls own every world-th sequence)
  double min_fold; int min_abund, allow_one_off;
  double min_parent_abund; int zero_queries;   // de novo rule only
  uint32_t *jq, *jk; unsigned long long *ctr;
  unsigned long long *rec;                  // [jb][ncol]
  int32_t *nflag, *nsam;                    // table call
  uint8_t *flags;                           // de novo call: [ncol][nrow]
  const uint16_t *len;                      // [ncol] sequence lengths
};

// The two parent rules.  TABLE (C_table_bimera2, chimera.cpp:117-122): samples with mat(i,j) > 0, parents
// mat(i,k) > min_fold * mat(i,j) and mat(i,k) >= min_abund.  DENOVO (isBimeraDenovo, R/chimeras.R:127): every sample
// (zero-count queries too when zero_queries is set), parents strictly above a numeric minParentAbundance.
enum BimRule { BIM_TABLE, BIM_DENOVO };
template <BimRule RULE> __device__ __forceinline__ bool bim_query_in(const BimTableArgs &a, int vj) {
  return RULE == BIM_DENOVO ? (vj > 0 || a.zero_queries) : vj > 0;
}
template <BimRule RULE> __device__ __forceinline__ bool bim_parent(const BimTableArgs &a, double bound, int vk) {
  return RULE == BIM_DENOVO ? (double)vk > bound && (double)vk > a.min_parent_abund : (double)vk > bound && vk >= a.min_abund;
}

// k is compared with j iff k is a parent of j in some sample that takes j as a query (chimera.cpp:121-123: the reference
// aligns a pair the first time a sample needs it).  grid (ceil(ncol / 256), jb); thread per candidate k, the query's
// column is read uniformly.
template <BimRule RULE>
__global__ void __launch_bounds__(256) k_bim_need(BimTableArgs a) {
  const uint32_t slot = blockIdx.y;
  const uint32_t j = (a.j0 + slot) * (uint32_t)a.q_mul + (uint32_t)a.q_add;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  bool need = false;
  if (k < a.ncol) {
    const int32_t *cj = a.mat + (size_t)j * a.nrow;
    for (int i = 0; i < a.nrow; i++) {
      const int vj = cj[i];
      if (!bim_query_in<RULE>(a, vj)) continue;
      const int vk = a.matT[(size_t)i * a.ncol + k];
      if (bim_parent<RULE>(a, a.min_fold * (double)vj, vk)) { need = true; break; }
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, need);
  if (m) {
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(&a.ctr[0], (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (need) { const unsigned long long p = base + __popc(m & ((1u << lane) - 1u)); a.jq[p] = j; a.jk[p] = (uint32_t)k; }
  }
}

// chimera.cpp:116-171 for one query per CTA: warps take the samples the query occurs in; lanes stride over the candidate
// parents k with coalesced reads of matT[i][k] and rec[slot][k]; the six maxima are reduced over the warp.
__global__ void __launch_bounds__(256) k_bim_flag(BimTableArgs a) {
  const uint32_t slot = blockIdx.x;
  const uint32_t j = (a.j0 + slot) * (uint32_t)a.q_mul + (uint32_t)a.q_add;
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t *cj = a.mat + (size_t)j * a.nrow;
  const unsigned long long *rrow = a.rec + (size_t)slot * a.ncol;
  __shared__ int s_flag, s_sam;
  if (threadIdx.x == 0) { s_flag = 0; s_sam = 0; }
  __syncthreads();
  int nflag = 0, nsam = 0;
  for (int i = wid; i < a.nrow; i += nwarps) {
    const int vj = cj[i];
    if (vj <= 0) continue;                                              // :117
    nsam++;
    const double bound = a.min_fold * (double)vj;
    int ml = 0, mr = 0, ol = 0, orr = 0, olo = 0, oro = 0;
    const int32_t *ti = a.matT + (size_t)i * a.ncol;
    for (int k = lane; k < a.ncol; k += 32) {
      const int vk = ti[k];
      if ((double)vk > bound && vk >= a.min_abund) {                    // :122
        const unsigned long long r = rrow[k];
        const int l = (int)(r & 0x7FFF), rr = (int)((r >> 15) & 0x7FFF);
        ml = max(ml, l); mr = max(mr, rr);                              // :149-150
        if (a.allow_one_off && (r & BIM_ALLOWED)) {                     // :151-156
          ol = max(ol, l); orr = max(orr, rr);
          olo = max(olo, (int)((r >> 30) & 0x7FFF)); oro = max(oro, (int)((r >> 45) & 0x7FFF));
        }
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      ml = max(ml, __shfl_xor_sync(0xffffffffu, ml, o)); mr = max(mr, __shfl_xor_sync(0xffffffffu, mr, o));
      ol = max(ol, __shfl_xor_sync(0xffffffffu, ol, o)); orr = max(orr, __shfl_xor_sync(0xffffffffu, orr, o));
      olo = max(olo, __shfl_xor_sync(0xffffffffu, olo, o)); oro = max(oro, __shfl_xor_sync(0xffffffffu, oro, o));
    }
    const int L = a.len[j];                                             // :162-169
    if (mr + ml >= L) nflag++;
    else if (a.allow_one_off && (ol + oro >= L || olo + orr >= L)) nflag++;
  }
  if (lane == 0) { if (nflag) atomicAdd(&s_flag, nflag); if (nsam) atomicAdd(&s_sam, nsam); }
  __syncthreads();
  if (threadIdx.x == 0) { a.nflag[j] = s_flag; a.nsam[j] = s_sam; }    // :172-173
}

// isBimeraDenovo's loop body (R/chimeras.R:124-132 + C_is_bimera, chimera.cpp:18-59) for every sample of one query, in
// the shape of k_bim_flag: CTA per query, warp per sample.  The parents are counted with a ballot next to the six maxima;
// fewer than two parents is FALSE without a model (:128-129).  Every cell (i, j) of the batch is written, 0 when the
// sample does not take j as a query.
__global__ void __launch_bounds__(256) k_bim_denovo_flag(BimTableArgs a) {
  const uint32_t slot = blockIdx.x;
  const uint32_t j = (a.j0 + slot) * (uint32_t)a.q_mul + (uint32_t)a.q_add;
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int32_t *cj = a.mat + (size_t)j * a.nrow;
  const unsigned long long *rrow = a.rec + (size_t)slot * a.ncol;
  const int L = a.len[j];
  for (int i = wid; i < a.nrow; i += nwarps) {
    const int vj = cj[i];
    bool bim = false;
    if (bim_query_in<BIM_DENOVO>(a, vj)) {
      const double bound = a.min_fold * (double)vj;
      int npar = 0, ml = 0, mr = 0, ol = 0, orr = 0, olo = 0, oro = 0;
      const int32_t *ti = a.matT + (size_t)i * a.ncol;
      for (int k0 = 0; k0 < a.ncol; k0 += 32) {                         // warp-uniform trip count: the ballot sees every lane
        const int k = k0 + lane;
        const bool par = k < a.ncol && bim_parent<BIM_DENOVO>(a, bound, ti[k]);     // :127
        npar += __popc(__ballot_sync(0xffffffffu, par));
        if (par) {
          const unsigned long long r = rrow[k];
          const int l = (int)(r & 0x7FFF), rr = (int)((r >> 15) & 0x7FFF);
          ml = max(ml, l); mr = max(mr, rr);                            // chimera.cpp:33-34
          if (a.allow_one_off && (r & BIM_ALLOWED)) {                   // :37-42
            ol = max(ol, l); orr = max(orr, rr);
            olo = max(olo, (int)((r >> 30) & 0x7FFF)); oro = max(oro, (int)((r >> 45) & 0x7FFF));
          }
        }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        ml = max(ml, __shfl_xor_sync(0xffffffffu, ml, o)); mr = max(mr, __shfl_xor_sync(0xffffffffu, mr, o));
        ol = max(ol, __shfl_xor_sync(0xffffffffu, ol, o)); orr = max(orr, __shfl_xor_sync(0xffffffffu, orr, o));
        olo = max(olo, __shfl_xor_sync(0xffffffffu, olo, o)); oro = max(oro, __shfl_xor_sync(0xffffffffu, oro, o));
      }
      bim = npar >= 2 && (mr + ml >= L || (a.allow_one_off && (ol + oro >= L || olo + orr >= L)));   // :45-52
    }
    if (lane == 0) a.flags[(size_t)j * a.nrow + i] = bim ? 1 : 0;
  }
}

// C_is_bimera (chimera.cpp:18-59) for a batch: warp per query over its job range.
struct BimIsArgs {
  const int32_t *query_idx; const long long *par_off; int nquery;
  const unsigned long long *rec; const uint16_t *len; int allow_one_off; uint8_t *out;
};
__global__ void __launch_bounds__(128) k_bim_is(BimIsArgs a) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (q >= a.nquery) return;
  int ml = 0, mr = 0, ol = 0, orr = 0, olo = 0, oro = 0;
  for (long long x = a.par_off[q] + lane; x < a.par_off[q + 1]; x += 32) {
    const unsigned long long r = a.rec[x];
    const int l = (int)(r & 0x7FFF), rr = (int)((r >> 15) & 0x7FFF);
    ml = max(ml, l); mr = max(mr, rr);                                  // :33-34 (skipped pairs were stored as zeros, :30-32)
    if (a.allow_one_off && (r & BIM_ALLOWED)) {                         // :37-42
      ol = max(ol, l); orr = max(orr, rr);
      olo = max(olo, (int)((r >> 30) & 0x7FFF)); oro = max(oro, (int)((r >> 45) & 0x7FFF));
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    ml = max(ml, __shfl_xor_sync(0xffffffffu, ml, o)); mr = max(mr, __shfl_xor_sync(0xffffffffu, mr, o));
    ol = max(ol, __shfl_xor_sync(0xffffffffu, ol, o)); orr = max(orr, __shfl_xor_sync(0xffffffffu, orr, o));
    olo = max(olo, __shfl_xor_sync(0xffffffffu, olo, o)); oro = max(oro, __shfl_xor_sync(0xffffffffu, oro, o));
  }
  const int L = a.len[a.query_idx[q]];
  bool rval = mr + ml >= L;                                             // :45-47 (the maxima only grow: the early exit changes nothing)
  if (a.allow_one_off && (ol + oro >= L || olo + orr >= L)) rval = true;   // :48-52
  if (lane == 0) a.out[q] = rval ? 1 : 0;
}

}  // namespace dd2

// =====================================================================================================================
// Host driver
// =====================================================================================================================
using namespace dd2;

namespace {

struct BimRun {
  int device = 0, num_sms = 148;
  cudaStream_t s = nullptr;
  BimSeqs sq{};
  BBuf<uint32_t> d_seq2, d_jq, d_jk, d_ptr, d_fwd_moves, d_fb, d_uneq;
  bool use_fwd = false, use_fwd16 = false; int fwd_slots = 0;
  BBuf<uint16_t> d_len;
  BBuf<unsigned long long> d_ctr, d_rec;
  std::vector<uint16_t> len;
  long long launches = 0, h2d = 0, d2h = 0;
  BimAlignArgs aa{};
  size_t smem = 0; int grid = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> align_ev;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;

  ~BimRun() {
    for (auto &e : align_ev) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (s) cudaStreamDestroy(s);
  }

  void open(int dev) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    device = dev;
    BCK(cudaSetDevice(dev));
    BCK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    BCK(cudaEventCreate(&ev0)); BCK(cudaEventCreate(&ev1));
    BCK(cudaEventRecord(ev0, s));
  }

  void upload_seqs(int nseq, const char *seq_concat, const int64_t *seq_off) {
    upload_packed_seqs(nseq, seq_concat, seq_off, s, d_seq2, d_len, len, sq, h2d, "bimera detection");
  }

  // shared-memory layout of k_bim_align (mirrors Run::setup_params of dd_driver.cu) and alignment parameters
  void setup_align(const dada2b_bimera_opts &o) {
    AlnParams &P = aa.P;
    P = AlnParams{};
    P.match = o.match; P.mismatch = o.mismatch; P.gap = o.gap_p; P.hgap = o.gap_p; P.band = o.max_shift; P.homo = 0;
    const int m = std::min(std::min(o.mismatch, o.gap_p), std::min(o.match, 0));
    P.sentinel = (int)(int16_t)(INT16_MIN - m);                                    // nwalign_vectorized.cpp:106
    const int maxlen = sq.maxlen, minlen = sq.minlen;
    const int lbmax = P.band < 0 ? maxlen : std::min(P.band + (maxlen - minlen), maxlen), rbmax = lbmax;
    const int Wmax = lbmax + rbmax + 1;
    const int nchunk = (((Wmax + 1) >> 1) + 31) >> 5;
    aa.sq = sq;
    aa.seq_bytes = (maxlen + 15) & ~15;
    aa.H_words = (Wmax + 2 + 3) & ~3;
    aa.ops_words = ((2 * maxlen) / 16 + 2 + 3) & ~3;
    aa.mask_words = ((2 * maxlen + 31) / 32 + 2 + 3) & ~3;
    aa.ptr_words = (unsigned long long)(2 * maxlen + 2) * 2 * nchunk;
    const int base_words = 2 * (aa.seq_bytes / 4) + aa.H_words + aa.ops_words + 3 * aa.mask_words;
    aa.ptr_in_smem = (4 * ((size_t)base_words + aa.ptr_words) * 4 <= 96 * 1024) ? 1 : 0;
    aa.warp_words = base_words + (aa.ptr_in_smem ? (int)aa.ptr_words : 0);
    smem = (size_t)4 * aa.warp_words * 4;
    if (smem > 200 * 1024) throw BErr{"dada2b: band/sequence length too large for the alignment kernel's shared memory."};
    BCK(cudaFuncSetAttribute(k_bim_align, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
    grid = num_sms * 8;
    if (!aa.ptr_in_smem) { d_ptr.alloc((size_t)grid * 4 * aa.ptr_words); aa.ptr_scratch = d_ptr.p; }
    aa.allow_one_off = o.allow_one_off != 0; aa.min_one_off_par_dist = o.min_one_off_par_dist; aa.max_shift = o.max_shift;
    d_ctr.alloc(8);
    BCK(cudaMemsetAsync(d_ctr.p, 0, 8 * 8, s));
    aa.ctr = d_ctr.p;
    // alignment kernel: 2 (default) = two jobs per lane group on the 16-bit SIMD datapath (dd_bimfwd16.cu), falling back per job to 1 = register wavefront (dd_bimfwd.cu) and 0 = warp-per-pair
    // traceback (k_bim_align).  DADA2B_BIMFWD=0|1|2 is a test hook that pins the first choice.
    const char *bf = getenv("DADA2B_BIMFWD");
    const int bf_mode = bf ? atoi(bf) : 2;
    use_fwd = bf_mode >= 1 && P.band >= 0;
    use_fwd16 = use_fwd && bf_mode == 2;
    fwd_slots = ((lbmax + 1) & ~1) + rbmax + 1;
    if (use_fwd) {
      const size_t w = bimfwd_scratch_words(fwd_slots, maxlen, num_sms);
      if (!w) use_fwd = false;
      else { d_fwd_moves.alloc(w); }
      const long worst = (long)maxlen * std::max(std::abs(P.mismatch), std::abs(P.match)) + std::abs(P.gap) + 16;
      aa.fast_ok = (worst < std::abs((long)P.sentinel) / 2 && !getenv("DADA2B_NO_FAST")) ? 1 : 0;
    }
  }

  void launch_align(unsigned long long njobs_upper) {
    cudaEvent_t a, b;
    BCK(cudaEventCreate(&a)); BCK(cudaEventCreate(&b));
    align_ev.emplace_back(a, b);
    const int g = (int)std::min<unsigned long long>((unsigned long long)grid, std::max<unsigned long long>(1, (njobs_upper + 3) / 4));
    BCK(cudaEventRecord(a, s));
    bool done = false;
    if (use_fwd) {
      // pass 1: every job through the register kernel; jobs whose band does not fit are listed in d_fb (count in ctr[4]) ...
      if (d_fb.n < njobs_upper) d_fb.alloc((size_t)njobs_upper);
      BCK(cudaMemsetAsync(d_ctr.p + 4, 0, 8, s));
      BimAlignArgs f = aa;
      f.ptr_scratch = d_fwd_moves.p; f.fb_list = d_fb.p; f.fb_count = d_ctr.p + 4; f.job_list = nullptr;
      bool done16 = false;
      if (use_fwd16) {          // pass 0: matching neighbours two at a time; the rest comes back in d_uneq (count in ctr[5]) for pass 1
        if (d_uneq.n < njobs_upper + 2) d_uneq.alloc((size_t)njobs_upper + 2);
        BCK(cudaMemsetAsync(d_ctr.p + 5, 0, 8, s));
        done16 = launch_bimfwd16(f, d_uneq.p, d_ctr.p + 5, fwd_slots, njobs_upper, num_sms, s);
        if (done16) { launches++; f.job_list = d_uneq.p; f.njobs_ptr = d_ctr.p + 5; }
      }
      done = launch_bimfwd(f, fwd_slots, njobs_upper, num_sms, s, nullptr);
      if (done) {
        launches++;
        // ... pass 2: and go through the warp-per-pair traceback kernel
        BimAlignArgs r = aa;
        r.job_list = d_fb.p; r.njobs_ptr = d_ctr.p + 4;
        k_bim_align<<<g, 128, smem, s>>>(r);
        launches++;
      }
    }
    if (!done) { k_bim_align<<<g, 128, smem, s>>>(aa); launches++; }
    BCK(cudaEventRecord(b, s));
  }

  void finish(dada2b_bimera_stats *st, double t0) {
    BCK(cudaEventRecord(ev1, s));
    unsigned long long h[8];
    BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    d2h += sizeof h;
    if (h[2]) throw BErr{"N-W Align out of range."};                               // nwalign_vectorized.cpp:279
    if (st) {
      float ms = 0, tot = 0;
      for (auto &e : align_ev) { BCK(cudaEventElapsedTime(&ms, e.first, e.second)); tot += ms; }
      st->ms_k_align = tot;
      BCK(cudaEventElapsedTime(&ms, ev0, ev1));
      st->ms_device = ms;
      st->n_pairs = (int64_t)h[3]; st->n_cells = (int64_t)h[1]; st->gpu_launches = launches;
      st->h2d_bytes = h2d; st->d2h_bytes = d2h; st->ms_total = bnow_ms() - t0;
    }
  }
};

__global__ void k_bim_count(unsigned long long *ctr) { ctr[3] += ctr[0]; ctr[0] = 0; }

void check_opts(const dada2b_bimera_opts *o) {
  if (!o) throw BErr{"dada2b: NULL options."};
  if (o->match < -16000 || o->match > 16000 || o->mismatch < -16000 || o->mismatch > 16000 || o->gap_p < -16000 || o->gap_p > 16000)
    throw BErr{"dada2b: alignment scores must fit the reference's int16 arithmetic."};
}

int fail(char *errbuf, const std::string &m) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", m.c_str()); return 1; }

}  // namespace

extern "C" {

void dada2b_bimera_default_opts(dada2b_bimera_opts *o) {
  // R/chimeras.R:220 (isBimeraDenovoTable) and R/dada.R:1-26 (MATCH / MISMATCH / GAP_PENALTY)
  o->min_fold = 1.5; o->min_abund = 2; o->allow_one_off = 0; o->min_one_off_par_dist = 4;
  o->match = 5; o->mismatch = -4; o->gap_p = -8; o->max_shift = 16; o->shard_rank = 0; o->shard_world = 1;
}

int dada2b_table_bimera(int32_t nrow, int32_t ncol, const int32_t *mat, const char *seq_concat, const int64_t *seq_off,
                        const dada2b_bimera_opts *opts, int32_t device, int32_t *nflag, int32_t *nsam,
                        dada2b_bimera_stats *stats, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  try {
    check_opts(opts);
    if (nrow < 0 || ncol <= 0) throw BErr{"Zero input sequences."};
    const int world = std::max(1, opts->shard_world), rank = opts->shard_rank;
    if (rank < 0 || rank >= world) throw BErr{"dada2b: bad shard_rank / shard_world."};
    BimRun R;
    R.open(device);
    R.upload_seqs(ncol, seq_concat, seq_off);
    R.setup_align(*opts);
    BBuf<int32_t> d_mat, d_matT, d_nflag, d_nsam;
    const size_t cells = (size_t)nrow * ncol;
    d_mat.alloc(cells); d_matT.alloc(cells); d_nflag.alloc(ncol); d_nsam.alloc(ncol);
    BCK(cudaMemsetAsync(d_nflag.p, 0, (size_t)ncol * 4, R.s));
    BCK(cudaMemsetAsync(d_nsam.p, 0, (size_t)ncol * 4, R.s));
    if (cells) {
      BCK(cudaMemcpyAsync(d_mat.p, mat, cells * 4, cudaMemcpyHostToDevice, R.s));
      R.h2d += (long long)cells * 4;
      const int32_t *src = d_mat.p; int32_t *dst = d_matT.p;
      k_bim_transpose<<<dim3((nrow + 31) / 32, (ncol + 31) / 32), dim3(32, 8), 0, R.s>>>(src, dst, nrow, ncol);
      R.launches++;
    }
    const int nq = (ncol - rank + world - 1) / world;                 // queries owned by this shard: j = slot * world + rank
    // batch size: record (8 B) + job (8 B) per (query, candidate) within ~2 GiB; grid.y <= 65535
    long long JB = std::min<long long>(65535, std::max<long long>(1, (2LL << 30) / (16LL * ncol)));
    JB = std::min<long long>(JB, std::max(nq, 1));
    R.d_rec.alloc((size_t)JB * ncol); R.d_jq.alloc((size_t)JB * ncol); R.d_jk.alloc((size_t)JB * ncol);
    BimTableArgs ta{};
    ta.mat = d_mat.p; ta.matT = d_matT.p; ta.nrow = nrow; ta.ncol = ncol; ta.q_mul = world; ta.q_add = rank;
    ta.min_fold = opts->min_fold; ta.min_abund = opts->min_abund; ta.allow_one_off = opts->allow_one_off != 0;
    ta.jq = R.d_jq.p; ta.jk = R.d_jk.p; ta.ctr = R.d_ctr.p; ta.rec = R.d_rec.p; ta.nflag = d_nflag.p; ta.nsam = d_nsam.p; ta.len = R.d_len.p;
    R.aa.jq = R.d_jq.p; R.aa.jk = R.d_jk.p; R.aa.njobs_ptr = R.d_ctr.p; R.aa.dst_mode = 1; R.aa.ncol = ncol; R.aa.rec = R.d_rec.p; R.aa.raw5 = nullptr;
    R.aa.q_mul = world; R.aa.q_add = rank;
    for (long long s0 = 0; s0 < nq; s0 += JB) {
      const int jb = (int)std::min<long long>(JB, nq - s0);
      ta.j0 = (uint32_t)s0; ta.jb = jb; R.aa.j0 = (uint32_t)s0;
      BCK(cudaMemsetAsync(R.d_rec.p, 0, (size_t)jb * ncol * 8, R.s));
      k_bim_need<BIM_TABLE><<<dim3((ncol + 255) / 256, jb), 256, 0, R.s>>>(ta);
      R.launch_align((unsigned long long)jb * ncol);
      k_bim_flag<<<jb, 256, 0, R.s>>>(ta);
      k_bim_count<<<1, 1, 0, R.s>>>(ta.ctr);
      R.launches += 3;
    }
    BCK(cudaMemcpyAsync(nflag, d_nflag.p, (size_t)ncol * 4, cudaMemcpyDeviceToHost, R.s));
    BCK(cudaMemcpyAsync(nsam, d_nsam.p, (size_t)ncol * 4, cudaMemcpyDeviceToHost, R.s));
    R.d2h += (long long)ncol * 8;
    R.finish(stats, t0);
    return 0;
  } catch (BErr &e) { return fail(errbuf, e.msg); }
  catch (std::exception &e) { return fail(errbuf, e.what()); }
}

int dada2b_denovo_bimera(int32_t nrow, int32_t ncol, const int32_t *mat, const char *seq_concat, const int64_t *seq_off,
                         const dada2b_bimera_opts *opts, double min_parent_abund, int32_t zero_queries, int32_t device,
                         uint8_t *flags, dada2b_bimera_stats *stats, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  try {
    check_opts(opts);
    if (nrow < 0 || ncol <= 0) throw BErr{"Zero input sequences."};
    if (opts->shard_world > 1 || opts->shard_rank != 0) throw BErr{"dada2b: the de novo bimera call is not sharded (shard_world must be 1)."};
    if (min_parent_abund != min_parent_abund || opts->min_fold != opts->min_fold) throw BErr{"dada2b: NaN parent rule."};
    const size_t cells = (size_t)nrow * ncol;
    for (size_t c = 0; c < cells; c++)
      if (mat[c] < 0) throw BErr{"dada2b: negative counts in the de novo bimera input."};
    BimRun R;
    R.open(device);
    R.upload_seqs(ncol, seq_concat, seq_off);
    R.setup_align(*opts);
    BBuf<int32_t> d_mat, d_matT;
    BBuf<uint8_t> d_flags;
    d_mat.alloc(std::max<size_t>(cells, 1)); d_matT.alloc(std::max<size_t>(cells, 1)); d_flags.alloc(std::max<size_t>(cells, 1));
    if (cells) {
      BCK(cudaMemcpyAsync(d_mat.p, mat, cells * 4, cudaMemcpyHostToDevice, R.s));
      R.h2d += (long long)cells * 4;
      const int32_t *src = d_mat.p; int32_t *dst = d_matT.p;
      k_bim_transpose<<<dim3((nrow + 31) / 32, (ncol + 31) / 32), dim3(32, 8), 0, R.s>>>(src, dst, nrow, ncol);
      R.launches++;
    }
    // batch size as in the table call; DADA2B_BIM_JB=<n> caps it (test hook: small tables cross batch boundaries)
    long long JB = std::min<long long>(65535, std::max<long long>(1, (2LL << 30) / (16LL * ncol)));
    if (const char *e = getenv("DADA2B_BIM_JB")) { const long long cap = atoll(e); if (cap > 0) JB = std::min(JB, cap); }
    JB = std::min<long long>(JB, ncol);
    R.d_rec.alloc((size_t)JB * ncol); R.d_jq.alloc((size_t)JB * ncol); R.d_jk.alloc((size_t)JB * ncol);
    BimTableArgs ta{};
    ta.mat = d_mat.p; ta.matT = d_matT.p; ta.nrow = nrow; ta.ncol = ncol; ta.q_mul = 1; ta.q_add = 0;
    ta.min_fold = opts->min_fold; ta.allow_one_off = opts->allow_one_off != 0;
    ta.min_parent_abund = min_parent_abund; ta.zero_queries = zero_queries != 0;
    ta.jq = R.d_jq.p; ta.jk = R.d_jk.p; ta.ctr = R.d_ctr.p; ta.rec = R.d_rec.p; ta.flags = d_flags.p; ta.len = R.d_len.p;
    R.aa.jq = R.d_jq.p; R.aa.jk = R.d_jk.p; R.aa.njobs_ptr = R.d_ctr.p; R.aa.dst_mode = 1; R.aa.ncol = ncol; R.aa.rec = R.d_rec.p; R.aa.raw5 = nullptr;
    R.aa.q_mul = 1; R.aa.q_add = 0;
    for (long long s0 = 0; s0 < ncol && nrow > 0; s0 += JB) {
      const int jb = (int)std::min<long long>(JB, ncol - s0);
      ta.j0 = (uint32_t)s0; ta.jb = jb; R.aa.j0 = (uint32_t)s0;
      BCK(cudaMemsetAsync(R.d_rec.p, 0, (size_t)jb * ncol * 8, R.s));
      k_bim_need<BIM_DENOVO><<<dim3((ncol + 255) / 256, jb), 256, 0, R.s>>>(ta);
      R.launch_align((unsigned long long)jb * ncol);
      k_bim_denovo_flag<<<jb, 256, 0, R.s>>>(ta);
      k_bim_count<<<1, 1, 0, R.s>>>(ta.ctr);
      R.launches += 3;
    }
    if (cells) {
      BCK(cudaMemcpyAsync(flags, d_flags.p, cells, cudaMemcpyDeviceToHost, R.s));
      R.d2h += (long long)cells;
    }
    R.finish(stats, t0);
    return 0;
  } catch (BErr &e) { return fail(errbuf, e.msg); }
  catch (std::exception &e) { return fail(errbuf, e.what()); }
}

int dada2b_is_bimera(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t nquery, const int32_t *query_idx,
                     const int64_t *par_off, const int32_t *par_idx, const dada2b_bimera_opts *opts, int32_t device,
                     uint8_t *is_bimera, dada2b_bimera_stats *stats, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  try {
    check_opts(opts);
    if (nquery < 0) throw BErr{"dada2b: negative query count."};
    BimRun R;
    R.open(device);
    R.upload_seqs(nseq, seq_concat, seq_off);
    R.setup_align(*opts);
    const long long njobs = nquery ? (long long)(par_off[nquery] - par_off[0]) : 0;
    std::vector<uint32_t> jq((size_t)njobs), jk((size_t)njobs);
    std::vector<long long> off((size_t)nquery + 1);
    for (int q = 0; q <= nquery; q++) off[q] = (long long)(par_off[q] - par_off[0]);
    for (int q = 0; q < nquery; q++) {
      if (query_idx[q] < 0 || query_idx[q] >= nseq || off[q + 1] < off[q]) throw BErr{"dada2b: bad query index / parent offsets."};
      for (long long x = off[q]; x < off[q + 1]; x++) {
        const int32_t k = par_idx[par_off[0] + x];
        if (k < 0 || k >= nseq) throw BErr{"dada2b: bad parent index."};
        jq[x] = (uint32_t)query_idx[q]; jk[x] = (uint32_t)k;
      }
    }
    BBuf<int32_t> d_q; BBuf<long long> d_off; BBuf<uint8_t> d_out;
    d_q.alloc(std::max(nquery, 1)); d_off.alloc((size_t)nquery + 1); d_out.alloc(std::max(nquery, 1));
    R.d_jq.alloc(std::max<size_t>(njobs, 1)); R.d_jk.alloc(std::max<size_t>(njobs, 1)); R.d_rec.alloc(std::max<size_t>(njobs, 1));
    if (njobs) {
      BCK(cudaMemcpyAsync(R.d_jq.p, jq.data(), (size_t)njobs * 4, cudaMemcpyHostToDevice, R.s));
      BCK(cudaMemcpyAsync(R.d_jk.p, jk.data(), (size_t)njobs * 4, cudaMemcpyHostToDevice, R.s));
    }
    if (nquery) BCK(cudaMemcpyAsync(d_q.p, query_idx, (size_t)nquery * 4, cudaMemcpyHostToDevice, R.s));
    BCK(cudaMemcpyAsync(d_off.p, off.data(), ((size_t)nquery + 1) * 8, cudaMemcpyHostToDevice, R.s));
    R.h2d += njobs * 8 + (long long)nquery * 12 + 8;
    R.aa.jq = R.d_jq.p; R.aa.jk = R.d_jk.p; R.aa.njobs_ptr = nullptr; R.aa.njobs_fixed = (unsigned long long)njobs; R.aa.dst_mode = 0;
    R.aa.rec = R.d_rec.p; R.aa.raw5 = nullptr; R.aa.q_mul = 1; R.aa.q_add = 0;
    if (njobs) R.launch_align((unsigned long long)njobs);
    if (nquery) {
      BimIsArgs ia{d_q.p, d_off.p, nquery, R.d_rec.p, R.d_len.p, opts->allow_one_off != 0, d_out.p};
      k_bim_is<<<(nquery + 3) / 4, 128, 0, R.s>>>(ia);
      R.launches++;
      BCK(cudaMemcpyAsync(is_bimera, d_out.p, (size_t)nquery, cudaMemcpyDeviceToHost, R.s));
      R.d2h += nquery;
    }
    {  // pairs counter for the stats
      unsigned long long n = (unsigned long long)njobs;
      BCK(cudaMemcpyAsync(R.d_ctr.p + 3, &n, 8, cudaMemcpyHostToDevice, R.s));
      BCK(cudaStreamSynchronize(R.s));
    }
    R.finish(stats, t0);
    return 0;
  } catch (BErr &e) { return fail(errbuf, e.msg); }
  catch (std::exception &e) { return fail(errbuf, e.what()); }
}

int dada2b_test_bimera_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *query,
                             const int32_t *parent, const dada2b_bimera_opts *opts, int32_t device, int32_t *out5,
                             char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  try {
    check_opts(opts);
    if (npairs <= 0) return 0;
    BimRun R;
    R.open(device);
    R.upload_seqs(nseq, seq_concat, seq_off);
    R.setup_align(*opts);
    std::vector<uint32_t> jq(npairs), jk(npairs);
    for (int x = 0; x < npairs; x++) {
      if (query[x] < 0 || query[x] >= nseq || parent[x] < 0 || parent[x] >= nseq) throw BErr{"dada2b: bad pair index."};
      jq[x] = (uint32_t)query[x]; jk[x] = (uint32_t)parent[x];
    }
    BBuf<int32_t> d_raw;
    d_raw.alloc((size_t)npairs * 5);
    R.d_jq.alloc(npairs); R.d_jk.alloc(npairs);
    BCK(cudaMemcpyAsync(R.d_jq.p, jq.data(), (size_t)npairs * 4, cudaMemcpyHostToDevice, R.s));
    BCK(cudaMemcpyAsync(R.d_jk.p, jk.data(), (size_t)npairs * 4, cudaMemcpyHostToDevice, R.s));
    R.aa.jq = R.d_jq.p; R.aa.jk = R.d_jk.p; R.aa.njobs_ptr = nullptr; R.aa.njobs_fixed = (unsigned long long)npairs; R.aa.dst_mode = 0;
    R.aa.rec = nullptr; R.aa.raw5 = d_raw.p; R.aa.q_mul = 1; R.aa.q_add = 0;
    R.launch_align((unsigned long long)npairs);
    BCK(cudaMemcpyAsync(out5, d_raw.p, (size_t)npairs * 5 * 4, cudaMemcpyDeviceToHost, R.s));
    R.finish(nullptr, t0);
    return 0;
  } catch (BErr &e) { return fail(errbuf, e.msg); }
  catch (std::exception &e) { return fail(errbuf, e.what()); }
}

}  // extern "C"
