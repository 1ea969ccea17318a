// CUDA kernels of the H100-native dada() core (sm_90a).  Product code.
//
// Kernel                reference function(s) it replaces (under /root/reference/src)
// k_classify            raw_align's k-mer screen + gapless test   nwalign_endsfree.cpp:10-55, kmers.cpp:13-150
// k_align<LOOP>         sub_new + compute_lambda_ts + "selectively store"  nwalign_endsfree.cpp:76-216/220-396/539-672,
//                       nwalign_vectorized.cpp:71-318, pval.cpp:144-197, cluster.cpp:90-204
// k_align<FINAL>        FinalSubsParallel + transition / quality matrices   Rmain.cpp:179-236, error.cpp:131-172,225-258
// k_align<BIRTH>        birth subs                                          Rmain.cpp:206-209, error.cpp:261-300
// k_final_p             final p / correct flag                              Rmain.cpp:239-252
// (b_shuffle2 / b_p_update / b_bud: the round tail of dd_round2.cu)
//
// Integer DP + scalar fp64: no tensor cores by construction (SURVEY.md 8d).
#include "dd_common.h"
#include "dd_kernels.h"
#include "ppois.cuh"
#include "dd_nw_warp.cuh"
#include <math_constants.h>

namespace dd2 {

// 5-mer (10 bits, first base most significant like kmers.cpp:226) starting at base p of a packed row.
__device__ __forceinline__ unsigned kmer_at(const uint32_t *row, int p) {
  // 10-bit label of the 5-mer starting at base p.  The reference labels 5-mers with the first base most
  // significant (kmers.cpp:226); counts, min-sums and position-wise equality are invariant under any
  // bijective relabelling, so the raw bit order of the packed row is used as is.
  uint32_t w0 = row[p >> 4], w1 = row[(p + 4) >> 4];
  return __funnelshift_r(w0, w1, 2 * (p & 15)) & 0x3FFu;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// =====================================================================================
// k_classify : k-mer screen / gapless decision for (centre, raw) pairs; one warp per pair.
//   mode 0: every block uses centre a.centre_idx; warps stride over raws [0, nraw)
//   mode 1: block b handles the single pair (pair_centre[b], pair_raw[b])   (birth subs)
// shared: centre 5-mer counts (1024 x u16 packed in 512 words), centre ordered 5-mers,
//         per-warp 1024 x u16 scratch counts, per-warp packed raw row.
// =====================================================================================
__global__ void __launch_bounds__(256) k_classify(ClassifyArgs a) {
  extern __shared__ uint32_t smem[];
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = lane_id();
  const int SW = a.in.SW;
  uint32_t *cen_cnt = smem;                                  // 512 words
  uint16_t *cen_kord = (uint16_t *)(smem + 512);             // kord_words*2 entries
  uint32_t *wtab = smem + 512 + a.kord_words + wid * 512;    // per warp
  uint32_t *wseq = smem + 512 + a.kord_words + nwarps * 512 + wid * SW;
  const AlnParams &P = a.P;

  const uint32_t c = a.mode == 0 ? a.centre_idx : a.pair_centre[blockIdx.x];
  const int len1 = a.in.len[c];
  __shared__ uint32_t cen_bits_s[32];      // presence bitmap of the centre's 5-mers (1024 bits)
  uint32_t cen_bits = 0;                   // lane l keeps word l
  if (P.use_kmers) {
    if (threadIdx.x < 32) cen_bits_s[threadIdx.x] = 0;
    for (int x = threadIdx.x; x < 512; x += blockDim.x) cen_cnt[x] = 0;
    for (int x = threadIdx.x; x < nwarps * 512; x += blockDim.x) smem[512 + a.kord_words + x] = 0;
    __syncthreads();
    const uint32_t *crow = a.in.seq2 + (size_t)c * SW;
    for (int p = threadIdx.x; p + KMER <= len1; p += blockDim.x) {
      unsigned km = kmer_at(crow, p);
      cen_kord[p] = (uint16_t)km;
      atomicAdd(&cen_cnt[km >> 1], 1u << (16 * (km & 1)));
      atomicOr(&cen_bits_s[km >> 5], 1u << (km & 31));
    }
    __syncthreads();
    cen_bits = cen_bits_s[lane];
  }

  const int gw = blockIdx.x * nwarps + wid, tw = gridDim.x * nwarps;
  // mode 0 walks this rank's raws only: r = it * shard_world + shard_rank (every raw when not sharded)
  const int sw = a.mode == 0 ? max(a.shard_world, 1) : 1, sr = a.mode == 0 ? a.shard_rank : 0;
  const bool from_list = a.mode == 0 && a.cand_list != nullptr;     // raws the streaming tier (k_prescreen) could not settle
  int r0 = a.mode == 0 ? gw : 0, rstep = a.mode == 0 ? tw : 1, rend = a.mode == 0 ? (a.in.nraw - sr + sw - 1) / sw : (wid == 0 ? 1 : 0);
  if (from_list) rend = (int)*a.cand_count;
  // Job ids are staged per warp (one register slot per lane) and flushed 32 at a time with a single
  // atomic reservation; the diagnostic counters are accumulated per warp.  (One same-address global
  // atomic per pair costs more than the screen itself.)
  uint32_t st_nw = 0, st_gl = 0;      // lane l holds staged entry l
  int n_nw = 0, n_gl = 0, c_align = 0, c_shroud = 0;
  auto flush = [&](uint32_t *list, unsigned long long *counter, uint32_t &stage, int &n) {
    if (n == 0) return;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(counter, (unsigned long long)n);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (lane < n) list[base + lane] = stage;
    n = 0;
  };
  for (int it = r0; it < rend; it += rstep) {
    const uint32_t r = from_list ? a.cand_list[it] : (a.mode == 0 ? (uint32_t)(it * sw + sr) : a.pair_raw[blockIdx.x]);
    const uint32_t job = a.mode == 0 ? r : blockIdx.x;
    if (a.mode == 0 && a.greedy && (a.in.reads[r] > a.centre_reads || a.lock[r])) continue;   // cluster.cpp:127-131
    const int len2 = a.in.len[r];
    int kind;
    if (P.use_kmers) {
      const uint32_t *rrow = a.in.seq2 + (size_t)r * SW;
      for (int x = lane; x < SW; x += 32) wseq[x] = rrow[x];
      __syncwarp();
      const int minlen = min(len1, len2), nko = minlen - KMER + 1;
      const double denom = (double)(minlen - KMER) + 1.;
      // Tier 1 (no atomics): U = #raw 5-mers present in the centre >= sum_k min(c_raw, c_centre).  kdist is
      // monotone in that sum, so 1 - U/denom > cutoff proves the pair is shrouded exactly (raw_align :51).
      {
        int U = 0;
        for (int p0 = 0; p0 + KMER <= len2; p0 += 32) {
          const int p = p0 + lane;
          const bool ok = p + KMER <= len2;
          const unsigned km = ok ? kmer_at(wseq, p) : 0u;
          const uint32_t w = __shfl_sync(0xffffffffu, cen_bits, km >> 5);
          U += ok ? (int)((w >> (km & 31)) & 1u) : 0;
        }
        U = warp_sum(U);
        const double kd_lb = 1. - ((double)(U & 0xFFFF)) / denom;
        if (kd_lb > P.kdist_cutoff) {
          c_align++; c_shroud++;
          if (lane == 0 && a.kind_out) a.kind_out[job] = (uint8_t)KIND_SHROUD;
          continue;
        }
      }
      int ms = 0, om = 0;
      for (int p = lane; p + KMER <= len2; p += 32) {
        unsigned km = kmer_at(wseq, p);
        unsigned sh = 16 * (km & 1);
        unsigned old = atomicAdd(&wtab[km >> 1], 1u << sh);
        unsigned rank = (old >> sh) & 0xFFFFu;
        unsigned cc = (cen_cnt[km >> 1] >> sh) & 0xFFFFu;
        ms += rank < cc;                     // sum_k min(c_raw[k], c_centre[k])   kmers.cpp:13-26
        if (p < nko) om += (km == cen_kord[p]);  // ordered matches           kmers.cpp:102-116
      }
      ms = warp_sum(ms);
      om = warp_sum(om);
      __syncwarp();
      for (int p = lane; p + KMER <= len2; p += 32) wtab[kmer_at(wseq, p) >> 1] = 0;
      __syncwarp();
      // kmers.cpp:24 / :91: dot = dotsum/(min(len)-k+1.), dist = 1-dot ; raw_align :51,:54
      double kdist = 1. - ((double)(ms & 0xFFFF)) / denom;
      bool ko_valid = P.gapless && !(P.sse == 0 && len1 != len2);
      double kodist = ko_valid ? 1. - ((double)(om & 0xFFFF)) / denom : -1.0;
      if (kdist > P.kdist_cutoff) kind = KIND_SHROUD;
      else if (P.band == 0 || (P.gapless && kodist == kdist)) kind = KIND_GAPLESS;
      else kind = KIND_NW;
    } else {
      kind = (P.band == 0) ? KIND_GAPLESS : KIND_NW;
    }
    c_align++;
    if (kind == KIND_SHROUD) c_shroud++;
    else if (kind == KIND_GAPLESS) { if (lane == n_gl) st_gl = job; if (++n_gl == 32) flush(a.gl_list, &a.ctr[CTR_GL], st_gl, n_gl); }
    else { if (lane == n_nw) st_nw = job; if (++n_nw == 32) flush(a.nw_list, &a.ctr[CTR_NW], st_nw, n_nw); }
    if (lane == 0 && a.kind_out) a.kind_out[job] = (uint8_t)kind;
  }
  flush(a.gl_list, &a.ctr[CTR_GL], st_gl, n_gl);
  flush(a.nw_list, &a.ctr[CTR_NW], st_nw, n_nw);
  if (lane == 0 && c_align) { atomicAdd(&a.ctr[CTR_ALIGN], (unsigned long long)c_align); if (c_shroud) atomicAdd(&a.ctr[CTR_SHROUD], (unsigned long long)c_shroud); }
}

// =====================================================================================
// k_align: alignment (NW or gapless) -> substitutions -> lambda, then mode-specific sink.
// =====================================================================================
template <int MODE>
__global__ void __launch_bounds__(128) k_align(AlignArgs a) {
  extern __shared__ uint32_t smem[];
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = lane_id();
  const AlnParams &P = a.P;
  // ---- shared layout: [err 16*ncol doubles][trans ints (FINAL)] then per-warp regions ----
  {
    const unsigned long long nj = a.njobs_ptr ? *a.njobs_ptr : (unsigned long long)a.njobs_fixed;
    if ((unsigned long long)blockIdx.x * nwarps >= nj) return;            // idle block: skip the prologue
  }
  double *s_err = (double *)smem;
  int *s_trans = (int *)(s_err + 16 * P.ncol);
  uint32_t *wbase = (uint32_t *)(s_trans + (MODE == MODE_FINAL ? 16 * P.ncol : 0)) + (size_t)wid * a.warp_words;
  uint8_t *s1 = (uint8_t *)wbase;
  uint8_t *s2 = s1 + a.seq_bytes;
  int *H = (int *)(wbase + 2 * (a.seq_bytes >> 2));
  uint32_t *opw = (uint32_t *)(H + a.H_words);
  uint32_t *ptr_s = opw + a.ops_words;
  for (int x = threadIdx.x; x < 16 * P.ncol; x += blockDim.x) s_err[x] = a.st.err[x];
  if (MODE == MODE_FINAL) for (int x = threadIdx.x; x < 16 * P.ncol; x += blockDim.x) s_trans[x] = 0;
  __syncthreads();

  const int gw = blockIdx.x * nwarps + wid, tw = gridDim.x * nwarps;
  uint32_t *ptr = a.ptr_in_smem ? ptr_s : a.ptr_scratch + (size_t)gw * a.ptr_words;
  const unsigned long long njobs = a.njobs_ptr ? *a.njobs_ptr : (unsigned long long)a.njobs_fixed;
  int errflag = 0;
  unsigned long long cells_lane = 0;

  for (unsigned long long jb = gw; jb < njobs; jb += tw) {
    uint32_t r, c, job = a.jobs ? a.jobs[jb] : (uint32_t)jb * (uint32_t)a.job_mul + (uint32_t)a.job_add;
    uint32_t cluster = 0;
    int kind = a.kind;
    if (MODE == MODE_LOOP) { r = job; c = a.centre_idx; }
    else if (MODE == MODE_FINAL) { r = job; cluster = a.st.cluster_of[r]; c = a.st.cl_center[cluster]; }
    else { r = a.pair_raw[job]; c = a.pair_centre[job]; }
    const int len1 = a.in.len[c], len2 = a.in.len[r];
    unpack_row(a.in.seq2 + (size_t)c * a.in.SW, len1, s1, P.homo && kind == KIND_NW);
    unpack_row(a.in.seq2 + (size_t)r * a.in.SW, len2, s2, P.homo && kind == KIND_NW);
    int nops;
    if (kind == KIND_NW) {
      nops = nw_warp(s1, len1, s2, len2, P, H, ptr, opw, &cells_lane, &errflag);
    } else {
      nops = max(len1, len2);   // nwalign_gapless, nwalign_endsfree.cpp:539-555
    }
    // ---- forward pass over alignment columns: al2subs (:570-639) + compute_lambda_ts (pval.cpp:144-197)
    const uint8_t *q2 = a.in.qual + (size_t)r * a.in.QS;
    const int minlen = min(len1, len2);
    double lambda = 1.0;
    int nsubs = 0, i0b = 0, i1b = 0, qerr = 0;
    const uint32_t rreads = a.in.reads[r];
    const bool acc = (MODE == MODE_FINAL) && a.st.correct[r];
    for (int cb = 0; cb < nops; cb += 32) {
      const int col = cb + lane;
      int op = 0;
      if (col < nops) {
        if (kind == KIND_NW) { const int e = nops - 1 - col; op = (opw[e >> 4] >> (2 * (e & 15))) & 3; }
        else op = col < minlen ? 1 : (len1 > len2 ? 3 : 2);
      }
      const unsigned b0 = __ballot_sync(0xffffffffu, op == 1 || op == 3);   // consumes a centre base
      const unsigned b1 = __ballot_sync(0xffffffffu, op == 1 || op == 2);   // consumes a raw base
      const int i0 = i0b + __popc(b0 & lanemask_lt()), i1 = i1b + __popc(b1 & lanemask_lt());
      double f = 1.0;
      bool sub = false;
      if (op == 1 || op == 2) {
        const int nt1 = s2[i1] & 3;
        const int qq = P.use_quals ? q2[i1] : 0;
        if (qq > P.ncol - 1) qerr = 1;                                  // pval.cpp:169-171
        int t = nt1 * 5;                                                // self transition, pval.cpp:160
        if (op == 1) {
          const int nt0 = s1[i0] & 3;
          t = nt0 * 4 + nt1;                                            // pval.cpp:183-185
          sub = nt0 != nt1;
          if (MODE == MODE_FINAL && acc) {                              // error.cpp:150-165, :243-250
            const int qa = q2[i1];
            if (qa < P.ncol) atomicAdd(&s_trans[t * P.ncol + qa], (int)rreads);
            atomicAdd(&a.st.cq_sum[(size_t)cluster * a.in.maxlen + i0], (unsigned long long)((unsigned)qa * rreads));
            atomicAdd(&a.st.cq_cnt[(size_t)cluster * a.in.maxlen + i0], (unsigned long long)rreads);
          }
        }
        f = s_err[t * P.ncol + min(qq, P.ncol - 1)];
      }
      if (MODE == MODE_BIRTH) {
        const unsigned sb = __ballot_sync(0xffffffffu, sub);
        if (sub) {
          const int slot = nsubs + __popc(sb & lanemask_lt());
          if (slot < a.b_cap) {
            const size_t o = (size_t)job * a.b_cap + slot;
            a.b_pos[o] = (uint16_t)i0; a.b_nt0[o] = s1[i0] & 3; a.b_nt1[o] = s2[i1] & 3; a.b_q1[o] = q2[i1];
          }
        }
        if (a.b_ops && col < nops) a.b_ops[(size_t)job * a.b_opcap + col] = (uint8_t)op;
      }
      nsubs += __popc(__ballot_sync(0xffffffffu, sub));
      // lambda: strictly sequential fp64 product in raw-position order (pval.cpp:190-193)
      const int ncol_here = min(32, nops - cb);
      for (int s = 0; s < ncol_here; s++) lambda = lambda * __shfl_sync(0xffffffffu, f, s);
      i0b += __popc(b0); i1b += __popc(b1);
    }
    if (__any_sync(0xffffffffu, qerr)) errflag = ERR_QUAL;
    if (lambda < 0 || lambda > 1) errflag = ERR_LAMBDA;                 // pval.cpp:195 / cluster.cpp:184
    // ---- sinks ----
    if (lane == 0) {
      if (MODE == MODE_LOOP) {                                           // cluster.cpp:179-201
        double emm = a.st.E_minmax[r];
        if (lambda * (double)a.total_reads > emm) {
          const double ec = lambda * (double)a.centre_reads;
          if (ec > emm) a.st.E_minmax[r] = ec;
          {                                    // sharded runs: every rank stores the comparisons of its own raws (owner mode)
            unsigned long long slot = a.cluster_i == 0 ? (unsigned long long)r : atomicAdd(&a.st.ctr[CTR_CS_COUNT], 1ull);
            if (slot < a.st.cs_cap) {
              a.st.cs_index[slot] = r; a.st.cs_i[slot] = a.cluster_i; a.st.cs_lambda[slot] = lambda; a.st.cs_ham[slot] = (uint32_t)nsubs;
            }
            if (a.cluster_i == 0 || r == c) { a.st.comp_lambda[r] = lambda; a.st.comp_ham[r] = (uint32_t)nsubs; }
          }
        }
      } else if (MODE == MODE_FINAL) {
        a.st.nsubs_final[r] = (uint32_t)nsubs;
      } else {
        a.b_nsubs[job] = (uint32_t)nsubs; a.b_lambda[job] = lambda; if (a.b_nops) a.b_nops[job] = (uint32_t)nops;
      }
    }
    __syncwarp();
  }
  if (errflag && lane == 0) atomicMax(&a.st.ctr[CTR_ERR], (unsigned long long)errflag);
  {
    unsigned cl = (unsigned)cells_lane;
#pragma unroll
    for (int o = 16; o; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
    if (lane == 0 && cl) atomicAdd(&a.st.ctr[CTR_CELLS], (unsigned long long)cl);
  }
  if (MODE == MODE_FINAL) {
    __syncthreads();
    for (int x = threadIdx.x; x < 16 * P.ncol; x += blockDim.x)
      if (s_trans[x]) atomicAdd(&a.st.trans[x], s_trans[x]);
  }
}

template __global__ void k_align<MODE_LOOP>(AlignArgs);
template __global__ void k_align<MODE_FINAL>(AlignArgs);
template __global__ void k_align<MODE_BIRTH>(AlignArgs);

// Rmain.cpp:239-252: final within-cluster p and the correct flag.
__global__ void k_final_p(DevState st, DevIn in, double omegaC) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= in.nraw) return;
  const uint32_t ci = st.cluster_of[r];
  double p;
  uint8_t correct = 1;
  if (st.cl_center[ci] == (uint32_t)r) p = 1.0;
  else {
    p = calc_pA((int)in.reads[r], st.comp_lambda[r] * (double)st.cl_reads[ci], true);
    if (p < omegaC) correct = 0;
  }
  st.p[r] = p;
  st.correct[r] = correct;
}

// error.cpp:99-119 post-hoc cluster p-value; one thread per cluster evaluates calc_pA(centre.reads, tot_e, true)
__global__ void k_calc_pA_vec(const int *reads, const double *E, const int *prior, double *out, int n) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x < n) out[x] = calc_pA(reads[x], E[x], prior[x] != 0);
}

// ------------------------------- launch wrappers --------------------------------------
// kernel launches of the CALLING thread (a context is driven by one thread at a time, include/dada2b.h: per-run deltas stay
// exact when several contexts run on several threads, e.g. the ranks of a sharded run inside one process)
static thread_local long long g_launches = 0;
long long launches_count() { return g_launches; }
void count_launch(int n) { g_launches += n; }
#define COUNT_LAUNCH(n) (g_launches += (n))
void launch_classify(const ClassifyArgs &a, int grid, int block, size_t smem, cudaStream_t s) {
  COUNT_LAUNCH(1);
  k_classify<<<grid, block, smem, s>>>(a);
}
cudaError_t align_set_smem(size_t bytes) {
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(k_align<MODE_LOOP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes))) return e;
  if ((e = cudaFuncSetAttribute(k_align<MODE_FINAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes))) return e;
  if ((e = cudaFuncSetAttribute(k_align<MODE_BIRTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes))) return e;
  return cudaFuncSetAttribute(k_classify, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
}
void launch_align(int mode, const AlignArgs &a, int grid, int block, size_t smem, cudaStream_t s) {
  COUNT_LAUNCH(1);
  if (mode == MODE_LOOP) k_align<MODE_LOOP><<<grid, block, smem, s>>>(a);
  else if (mode == MODE_FINAL) k_align<MODE_FINAL><<<grid, block, smem, s>>>(a);
  else k_align<MODE_BIRTH><<<grid, block, smem, s>>>(a);
}
void launch_final_p(const DevState &st, const DevIn &in, double omegaC, cudaStream_t s) {
  COUNT_LAUNCH(1);
  k_final_p<<<(in.nraw + 127) / 128, 128, 0, s>>>(st, in, omegaC);
}
void launch_calc_pA_vec(const int *reads, const double *E, const int *prior, double *out, int n, cudaStream_t s) {
  COUNT_LAUNCH(1);
  k_calc_pA_vec<<<(n + 127) / 128, 128, 0, s>>>(reads, E, prior, out, n);
}

}  // namespace dd2
