// Round tail (product code, sm_90a): b_shuffle2 / b_p_update / b_bud of every round, in 1 + NP + 1 launches.
//
//   k_tail_link    threads the round's new stored comparisons onto per-raw chains (newest first) and clears the scratch
//   k_tail_pass    one b_shuffle2 pass (cluster.cpp:210-266) in ONE kernel: every raw walks its own chain for the
//                  arg-max of lambda * reads(cluster); the pass-wide frozen reads (Appendix A.4 of SURVEY.md) are
//                  reads_at_round_start + sum of the earlier passes' deltas, and a pass only ever adds to its own delta
//                  row, so no commit kernel is needed
//   k_tail_final   b_p_update (pval.cpp:14-40) + the b_bud scan (cluster.cpp:274-308) + the report: per-block
//                  lexicographic (p asc, reads desc) minima with their tie candidates, reduced by the last block to
//                  finish (ticket counter), which also commits the cluster reads and clears the per-cluster flags
//
// k_tail_pass / k_tail_final come in two forms.  SMEM = true stages the per-cluster state (frozen reads, update flags) per
// block in shared memory, which holds it up to ~32 k clusters; SMEM = false reads it from global memory at every use, for
// any cluster count.  The host picks the form per launch from the round's cluster count.
//
// The arg-max prefers the lowest cluster index among equal e (chain walked from the newest entry with '>='), moves are
// recorded per pass (the host replays them in the reference's order) and the host resolves exact (p, reads) ties by
// (cluster, slot).
#include "dd_common.h"
#include "dd_kernels.h"
#include "ppois.cuh"

namespace dd2 {

constexpr uint32_t CHAIN_END = 0xFFFFFFFFu;

// Per-pass scratch rows (TailState::rows): [delta(cl_cap) | touched(cl_cap) | moves of the pass (1) | pad].  One row is one
// NCCL all-reduce in sharded runs (every rank shuffles its own raws only).
__device__ __forceinline__ int &row_delta(const TailState &ts, int pass, uint32_t c) { return ts.rows[(size_t)pass * ts.row_stride + c]; }
__device__ __forceinline__ int &row_touched(const TailState &ts, int pass, uint32_t c) { return ts.rows[(size_t)pass * ts.row_stride + ts.cl_cap + c]; }
__device__ __forceinline__ int &row_nmove(const TailState &ts, int pass) { return ts.rows[(size_t)pass * ts.row_stride + 2 * (size_t)ts.cl_cap]; }
// the raw handled by global thread `it`: this rank's raws only (one rank: every raw)
__device__ __forceinline__ long long tail_raw(const TailState &ts, long long it) { return it * ts.world + ts.rank; }

__global__ void k_tail_link(DevState st, TailState ts, unsigned long long base, uint32_t cluster_i, int nraw, int nclust) {
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const unsigned long long t0 = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (cluster_i == 0) {                       // cluster 0 owns slots [0, nraw): one entry per raw, the chain's tail
    for (unsigned long long x = t0; x < (unsigned long long)nraw; x += stride) { ts.head[x] = (uint32_t)x; ts.cs_prev[x] = CHAIN_END; }
  } else {
    const unsigned long long n = st.ctr[CTR_CS_COUNT];
    for (unsigned long long x = base + t0; x < n; x += stride) {       // at most one new entry per raw and round
      const uint32_t r = st.cs_index[x];
      ts.cs_prev[x] = ts.head[r];
      ts.head[r] = (uint32_t)x;
    }
  }
  for (unsigned long long x = t0; x < (unsigned long long)MAX_PASS * ts.row_stride; x += stride) {
    const unsigned c = (unsigned)(x % ts.row_stride);
    if (c >= 2 * ts.cl_cap || (int)(c % ts.cl_cap) < nclust) ts.rows[x] = 0;
  }
  if (t0 < MAX_PASS) ts.nmove_pass[t0] = 0;
  if (t0 == 0) *ts.done = 0;
}

// reads of cluster c as frozen at the start of shuffle pass `pass` (pass == npasses: after the last one).  Valid until
// k_tail_final commits them to cl_reads: after that, the deltas would be counted twice.
__device__ __forceinline__ uint32_t frozen_reads(const DevState &st, const TailState &ts, int pass, int c) {
  int v = (int)st.cl_reads[c];
  for (int k = 0; k < pass; k++) v += row_delta(ts, k, c);
  return (uint32_t)v;
}
// cluster c needs a p-update: flagged before the round (new cluster / bud) or touched by a move of passes 0..last_pass
__device__ __forceinline__ bool cluster_updated(const DevState &st, const TailState &ts, int last_pass, int c) {
  int u = st.cl_update_e[c];
  for (int k = 0; k <= last_pass; k++) u |= row_touched(ts, k, c);
  return u != 0;
}
__device__ __forceinline__ void stage_reads(const DevState &st, const TailState &ts, int pass, int nclust, uint32_t *s_reads) {
  for (int c = threadIdx.x; c < nclust; c += blockDim.x) s_reads[c] = frozen_reads(st, ts, pass, c);
  __syncthreads();
}

// TAIL_RPT raws per thread, their chains walked in lockstep: the walk is a chain of dependent DRAM round trips (head -> entry ->
// previous entry ...), so what one thread can overlap is what counts (one raw per thread: several waves of 2048 threads per SM,
// each as long as the chain)
constexpr int TAIL_RPT = 4;
template <bool SMEM>
__global__ void k_tail_pass(DevState st, DevIn in, TailState ts, int pass, int nclust) {
  extern __shared__ uint32_t s_reads[];                               // SMEM: [nclust] frozen reads
  if (pass > 0 && row_nmove(ts, pass - 1) == 0) return;             // previous pass moved nothing (anywhere): b_shuffle2 returned false
  if (SMEM) stage_reads(st, ts, pass, nclust, s_reads);
  int r[TAIL_RPT];
  uint32_t x[TAIL_RPT], best_x[TAIL_RPT];
  double best_e[TAIL_RPT];
#pragma unroll
  for (int u = 0; u < TAIL_RPT; u++) {
    const long long rl = tail_raw(ts, ((long long)blockIdx.x * TAIL_RPT + u) * blockDim.x + threadIdx.x);
    r[u] = rl < in.nraw ? (int)rl : -1;
    best_e[u] = -1.0; best_x[u] = CHAIN_END;
  }
#pragma unroll
  for (int u = 0; u < TAIL_RPT; u++) x[u] = r[u] >= 0 ? ts.head[r[u]] : CHAIN_END;
  for (;;) {                                                            // clusters descending: '>=' keeps the lowest index among ties
    bool any = false;
    double lam[TAIL_RPT]; uint32_t ci[TAIL_RPT], nx[TAIL_RPT];
#pragma unroll
    for (int u = 0; u < TAIL_RPT; u++)
      if (x[u] != CHAIN_END) { lam[u] = st.cs_lambda[x[u]]; ci[u] = st.cs_i[x[u]]; nx[u] = ts.cs_prev[x[u]]; any = true; }
    if (!any) break;
#pragma unroll
    for (int u = 0; u < TAIL_RPT; u++)
      if (x[u] != CHAIN_END) {
        const double e = lam[u] * (double)(SMEM ? s_reads[ci[u]] : frozen_reads(st, ts, pass, ci[u]));
        if (e >= best_e[u]) { best_e[u] = e; best_x[u] = x[u]; }
        x[u] = nx[u];
      }
  }
#pragma unroll
  for (int u = 0; u < TAIL_RPT; u++) {
    if (best_x[u] == CHAIN_END) continue;
    const int rr = r[u];
    const uint32_t to = st.cs_i[best_x[u]], from = st.cluster_of[rr];
    if (to != from && !st.is_center[rr]) {                              // cluster.cpp:248-260
      const unsigned long long s = atomicAdd(&st.ctr[CTR_NMOVE], 1ull);
      if (s < st.move_cap) { st.moves[2 * s] = (uint32_t)rr; st.moves[2 * s + 1] = to; }
      atomicAdd(&ts.nmove_pass[pass], 1u);                              // this rank's moves of the pass (splits the local move list)
      atomicAdd(&row_nmove(ts, pass), 1);                               // all ranks' after the all-reduce
      st.cluster_of[rr] = to;
      st.comp_lambda[rr] = st.cs_lambda[best_x[u]];
      st.comp_ham[rr] = st.cs_ham[best_x[u]];
      const int rd = (int)in.reads[rr];
      atomicAdd(&row_delta(ts, pass, from), -rd);
      atomicAdd(&row_delta(ts, pass, to), rd);
      row_touched(ts, pass, from) = 1; row_touched(ts, pass, to) = 1;   // -> cl_update_e (bi_pop_raw / bi_add_raw set update_e)
    }
  }
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o); v = t < v ? t : v; }
  return v;
}
__device__ __forceinline__ uint32_t warp_max_u32(uint32_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) { const uint32_t t = __shfl_xor_sync(0xffffffffu, v, o); v = t > v ? t : v; }
  return v;
}

// one copy of the incomplete-gamma code for the TAIL_RPT unrolled raws of a thread
__device__ __noinline__ double calc_pA_call(int reads, double E_reads, bool prior) { return calc_pA(reads, E_reads, prior); }

// blockDim.x must be TAIL_BLOCK (a multiple of 32, at most 1024)
// mode 0: p-update + bud scan only if the last launched pass moved nothing (anywhere); otherwise just report and leave the
//         state for further k_tail_pass launches
// mode 2: MAX_SHUFFLE passes are done: proceed as if converged (Rmain.cpp:322-325 stops shuffling there)
template <bool SMEM>
__global__ void k_tail_final(DevState st, DevIn in, TailState ts, BudParams bp, int greedy, int detect_singletons, int last_pass, int nclust,
                             int mode) {
  extern __shared__ uint32_t s_reads[];                 // SMEM: [nclust] reads, then [nclust] bytes: cluster needs a p-update
  uint8_t *s_upd = (uint8_t *)(s_reads + nclust);
  __shared__ unsigned long long s_pb[32], s_pbp[32];
  __shared__ uint32_t s_rd[32], s_rdp[32];
  __shared__ unsigned s_n, s_np, s_last;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nwarp = blockDim.x >> 5;
  const bool moved_nothing = last_pass < 0 || row_nmove(ts, last_pass) == 0;
  const bool converged = moved_nothing || mode == 2;
  // the cluster state after the last pass; it stays valid in the last block until the commit below
  auto reads_of = [&](auto c) { return SMEM ? s_reads[c] : frozen_reads(st, ts, last_pass + 1, c); };
  auto updated = [&](auto c) { return SMEM ? s_upd[c] != 0 : cluster_updated(st, ts, last_pass, c); };
  if (tid == 0) { s_n = 0; s_np = 0; }
  if (SMEM) {
    for (int c = tid; c < nclust; c += blockDim.x) s_upd[c] = cluster_updated(st, ts, last_pass, c) ? 1 : 0;
    stage_reads(st, ts, last_pass + 1, nclust, s_reads);             // also the barrier behind s_n / s_np / s_upd
  } else __syncthreads();
  // TAIL_RPT raws per thread: the per-CTA work around them (staging, five barriers, the block reductions: two thirds of the
  // kernel's instructions with one raw per thread) is paid once per 1024 raws
  int rA[TAIL_RPT];
  unsigned long long pbA[TAIL_RPT];
  uint32_t rdA[TAIL_RPT];
  unsigned eligm = 0, priorm = 0;
  unsigned long long pb = ~0ull, pbp = ~0ull;                           // this thread's minima
#pragma unroll
  for (int u = 0; u < TAIL_RPT; u++) {
    const long long rl = tail_raw(ts, ((long long)blockIdx.x * TAIL_RPT + u) * blockDim.x + tid);
    const int r = (int)(rl < in.nraw ? rl : in.nraw);
    rA[u] = r; pbA[u] = ~0ull; rdA[u] = 0;
    if (converged && r < in.nraw) {
      const uint32_t ci = st.cluster_of[r];
      const uint32_t rd = in.reads[r];
      const bool prior = in.prior[r] != 0;
      const double lambda = st.comp_lambda[r];
      const uint32_t ham = st.comp_ham[r];
      double pval = st.p[r];
      if (updated(ci)) {                                                 // get_pA pval.cpp:67-89
        if (rd == 1 && !prior && !detect_singletons) pval = 1.;
        else if (ham == 0) pval = 1.;
        else if (lambda == 0) pval = 0.;
        else {
          // b_bud only ever asks whether p * nraw < omegaA (or p < omegaP for a raw with a prior), cluster.cpp:313-316, and the
          // p-values of the output are recomputed after the loop (k_final_p).  p >= P(X = reads) = exp(-E) E^reads / reads!  for
          // either normalisation of calc_pA: when that lower bound is already above the threshold (by a factor e), the raw cannot
          // be budded whatever its exact p is, and the bound is stored in its place -- no incomplete-gamma evaluation.
          const double E = lambda * (double)reads_of(ci);
          const double lg = -E + (double)rd * log(E) - lgamma((double)rd + 1.0);
          if (lg >= (prior ? bp.skip_log_prior : bp.skip_log)) pval = exp(lg);
          else pval = calc_pA_call((int)rd, E, prior || detect_singletons);
        }
        st.p[r] = pval;
      }
      if (greedy && st.cl_check_locks[ci]) {                             // pval.cpp:29-38
        const uint32_t cen = st.cl_center[ci];
        if ((double)in.reads[cen] * lambda > (double)rd) st.lock[r] = 1;
        if ((uint32_t)r == cen) st.lock[r] = 1;
      }
      // b_bud candidate (cluster.cpp:285-294)
      const bool elig = !st.slot0[r] && (int)rd >= bp.min_abund && (int)ham >= bp.min_hamming &&
                        (bp.min_fold <= 1 || ((double)rd) >= bp.min_fold * lambda * (double)reads_of(ci));
      rdA[u] = rd;
      if (prior) priorm |= 1u << u;
      if (elig) {
        eligm |= 1u << u;
        pbA[u] = (unsigned long long)__double_as_longlong(pval);
        pb = pbA[u] < pb ? pbA[u] : pb;
        if (prior) pbp = pbA[u] < pbp ? pbA[u] : pbp;
      }
    }
  }
  // block minimum of p, then maximum of reads among the raws attaining it; all of those are tie candidates
  unsigned long long w = warp_min_u64(pb), wp = warp_min_u64(pbp);
  if (lane == 0) { s_pb[wid] = w; s_pbp[wid] = wp; }
  __syncthreads();
  unsigned long long bmin = ~0ull, bminp = ~0ull;
  for (int k = 0; k < nwarp; k++) { bmin = s_pb[k] < bmin ? s_pb[k] : bmin; bminp = s_pbp[k] < bminp ? s_pbp[k] : bminp; }
  uint32_t tr = 0, trp = 0;                                             // this thread's largest reads among its candidates
  unsigned cam = 0, cpm = 0;
#pragma unroll
  for (int u = 0; u < TAIL_RPT; u++) {
    const bool elig = (eligm >> u) & 1u, prior = (priorm >> u) & 1u;
    if (elig && pbA[u] == bmin) { cam |= 1u << u; tr = rdA[u] > tr ? rdA[u] : tr; }
    if (elig && prior && pbA[u] == bminp) { cpm |= 1u << u; trp = rdA[u] > trp ? rdA[u] : trp; }
  }
  uint32_t wr = warp_max_u32(tr), wrp = warp_max_u32(trp);
  if (lane == 0) { s_rd[wid] = wr; s_rdp[wid] = wrp; }
  __syncthreads();
  uint32_t bmax = 0, bmaxp = 0;
  for (int k = 0; k < nwarp; k++) { bmax = s_rd[k] > bmax ? s_rd[k] : bmax; bmaxp = s_rdp[k] > bmaxp ? s_rdp[k] : bmaxp; }
#pragma unroll
  for (int u = 0; u < TAIL_RPT; u++) {
    if (((cam >> u) & 1u) && rdA[u] == bmax) { const unsigned k = atomicAdd(&s_n, 1u); if (k < TIE_MAX) ts.blk_ties[(size_t)blockIdx.x * TIE_MAX + k] = (uint32_t)rA[u]; }
    if (((cpm >> u) & 1u) && rdA[u] == bmaxp) { const unsigned k = atomicAdd(&s_np, 1u); if (k < TIE_MAX) ts.blk_ties_pr[(size_t)blockIdx.x * TIE_MAX + k] = (uint32_t)rA[u]; }
  }
  __syncthreads();
  if (tid == 0) {
    BlkBest b;
    b.pb = bmin; b.pbp = bminp; b.rd = bmax; b.rdp = bmaxp; b.n = s_n; b.np = s_np;
    ts.blk[blockIdx.x] = b;
    __threadfence();                                                   // results visible before the ticket
    s_last = atomicAdd(ts.done, 1u) == gridDim.x - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;

  // ---- the last block to finish: commit, global reduction, report ----
  __threadfence();
  const volatile BlkBest *blk = ts.blk;
  const volatile uint32_t *bt = ts.blk_ties, *btp = ts.blk_ties_pr;
  if (converged)       // the other blocks read cl_reads before they took their tickets
    for (int c = tid; c < nclust; c += blockDim.x) st.cl_reads[c] = reads_of(c);
  // a cluster's reads after the commit: in global memory, cl_reads now holds them (the barriers below make every thread's commit
  // visible to the block)
  auto committed_reads = [&](auto c) { return SMEM ? s_reads[c] : st.cl_reads[c]; };
  if (tid == 0) {
    uint32_t acc = 0;                                                  // pinfo[p+1] = moves recorded up to and including pass p
    st.pinfo[0] = 0;
    for (int p = 0; p <= last_pass; p++) { acc += ts.nmove_pass[p]; st.pinfo[p + 1] = acc; }
  }
  if (converged) {
    unsigned long long gmin = ~0ull, gminp = ~0ull;
    for (unsigned b = tid; b < gridDim.x; b += blockDim.x) {
      const unsigned long long x = blk[b].pb, xp = blk[b].pbp;
      gmin = x < gmin ? x : gmin; gminp = xp < gminp ? xp : gminp;
    }
    gmin = warp_min_u64(gmin); gminp = warp_min_u64(gminp);
    if (lane == 0) { s_pb[wid] = gmin; s_pbp[wid] = gminp; }
    __syncthreads();
    gmin = ~0ull; gminp = ~0ull;
    for (int k = 0; k < nwarp; k++) { gmin = s_pb[k] < gmin ? s_pb[k] : gmin; gminp = s_pbp[k] < gminp ? s_pbp[k] : gminp; }
    uint32_t gmax = 0, gmaxp = 0;
    for (unsigned b = tid; b < gridDim.x; b += blockDim.x) {
      if (blk[b].n && blk[b].pb == gmin) gmax = blk[b].rd > gmax ? blk[b].rd : gmax;
      if (blk[b].np && blk[b].pbp == gminp) gmaxp = blk[b].rdp > gmaxp ? blk[b].rdp : gmaxp;
    }
    gmax = warp_max_u32(gmax); gmaxp = warp_max_u32(gmaxp);
    if (lane == 0) { s_rd[wid] = gmax; s_rdp[wid] = gmaxp; }
    if (tid == 0) { s_n = 0; s_np = 0; }
    __syncthreads();
    gmax = 0; gmaxp = 0;
    for (int k = 0; k < nwarp; k++) { gmax = s_rd[k] > gmax ? s_rd[k] : gmax; gmaxp = s_rdp[k] > gmaxp ? s_rdp[k] : gmaxp; }
    for (unsigned b = tid; b < gridDim.x; b += blockDim.x) {
      if (blk[b].n && blk[b].pb == gmin && blk[b].rd == gmax) {
        const unsigned cnt = blk[b].n, at = atomicAdd(&s_n, cnt);
        for (unsigned k = 0; k < cnt && k < TIE_MAX && at + k < TIE_MAX; k++) {
          const uint32_t rr = bt[(size_t)b * TIE_MAX + k];
          st.report->tie_r[at + k] = rr; st.report->tie_lam[at + k] = st.comp_lambda[rr]; st.report->tie_ham[at + k] = st.comp_ham[rr];
          const uint32_t cc = st.cluster_of[rr];
          st.report->tie_cl[at + k] = cc; st.report->tie_clreads[at + k] = committed_reads(cc);
        }
      }
      if (blk[b].np && blk[b].pbp == gminp && blk[b].rdp == gmaxp) {
        const unsigned cnt = blk[b].np, at = atomicAdd(&s_np, cnt);
        for (unsigned k = 0; k < cnt && k < TIE_MAX && at + k < TIE_MAX; k++) {
          const uint32_t rr = btp[(size_t)b * TIE_MAX + k];
          st.report->tiep_r[at + k] = rr; st.report->tiep_lam[at + k] = st.comp_lambda[rr]; st.report->tiep_ham[at + k] = st.comp_ham[rr];
          const uint32_t cc = st.cluster_of[rr];
          st.report->tiep_cl[at + k] = cc; st.report->tiep_clreads[at + k] = committed_reads(cc);
        }
      }
    }
    for (int c = tid; c < nclust; c += blockDim.x) { st.cl_update_e[c] = 0; st.cl_check_locks[c] = 0; }   // consumed above
    __syncthreads();
    if (tid == 0) {
      st.ctr[CTR_PMIN] = gmin; st.ctr[CTR_RMAX] = gmax; st.ctr[CTR_NTIE] = s_n;
      st.ctr[CTR_PMIN_PR] = gminp; st.ctr[CTR_RMAX_PR] = gmaxp; st.ctr[CTR_NTIE_PR] = s_np;
    }
  }
  __syncthreads();
  if (tid < CTR_N) st.report->ctr[tid] = st.ctr[tid];
  if (tid < MAX_PASS + 2) st.report->pinfo[tid] = st.pinfo[tid];
  if (tid == 0) { st.report->converged = converged ? 1u : 0u; *ts.done = 0; }
  (void)moved_nothing;
}


// ---- per-rank helpers: every rank keeps the comparisons / state of its own raws only (one rank: every raw) ----
// b_bud tie sets larger than TIE_MAX: this rank's candidates at the GLOBAL (p, reads) optimum (ctr[CTR_PMIN..] set by the host).
__global__ void k_bud_collect_owned(DevState st, DevIn in, TailState ts, BudParams bp, uint32_t *ties, uint32_t *ties_pr, unsigned cap) {
  const long long rl = tail_raw(ts, blockIdx.x * (long long)blockDim.x + threadIdx.x);
  if (rl >= in.nraw) return;
  const int r = (int)rl;
  const uint32_t rd = in.reads[r];
  const bool elig = !st.slot0[r] && (int)rd >= bp.min_abund && (int)st.comp_ham[r] >= bp.min_hamming &&
                    (bp.min_fold <= 1 || ((double)rd) >= bp.min_fold * st.comp_lambda[r] * (double)st.cl_reads[st.cluster_of[r]]);
  if (!elig) return;
  const unsigned long long pb = (unsigned long long)__double_as_longlong(st.p[r]);
  if (pb == st.ctr[CTR_PMIN] && (unsigned long long)rd == st.ctr[CTR_RMAX]) {
    const unsigned long long k = atomicAdd(&st.ctr[CTR_NTIE], 1ull);
    if (k < cap) ties[k] = (uint32_t)r;
  }
  if (in.prior[r] && pb == st.ctr[CTR_PMIN_PR] && (unsigned long long)rd == st.ctr[CTR_RMAX_PR]) {
    const unsigned long long k = atomicAdd(&st.ctr[CTR_NTIE_PR], 1ull);
    if (k < cap) ties_pr[k] = (uint32_t)r;
  }
}
// final per-raw results of raws this rank does not own -> 0, so that a sum all-reduce assembles the full arrays
__global__ void k_mask_unowned(double *p, uint8_t *correct, int nraw, int rank, int world) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < nraw && r % world != rank) { p[r] = 0.0; correct[r] = 0; }
}
// Post-hoc expected reads (error.cpp:106-116) over this rank's own stored comparisons: every stored comparison whose raw is the
// centre of another cluster j contributes lambda * reads_i to tot_e[j]; emit (i, j, value) triples, the host adds them in ascending
// i like the reference's cluster-order loop.
__global__ void k_posthoc_owned(DevState st, unsigned long long n, const int *center_cluster, uint32_t *trip_ij, double *trip_v, unsigned cap,
                                unsigned long long *count, int rank, int world, int nraw) {
  const unsigned long long x = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (x >= n) return;
  if (x < (unsigned long long)nraw && (int)(x % (unsigned long long)world) != rank) return;      // cluster-0 slot of somebody else's raw: never written
  const int j = center_cluster[st.cs_index[x]];
  if (j < 0) return;
  const uint32_t i = st.cs_i[x];
  if ((int)i == j) return;
  const unsigned long long s = atomicAdd(count, 1ull);
  if (s < cap) { trip_ij[2 * s] = i; trip_ij[2 * s + 1] = (uint32_t)j; trip_v[s] = st.cs_lambda[x] * (double)st.cl_reads[i]; }
}

// ------------------------------- launch wrappers --------------------------------------
constexpr int TAIL_BLOCK = 256;
constexpr size_t TAIL_SMEM_MAX = 160 * 1024;

int tail_smem_clusters_max() { return (int)((TAIL_SMEM_MAX - 16) / 5); }     // k_tail_final<true>: nclust * 5 + 16 bytes
int tail_grid(int nraw) { return std::max(1, (nraw + TAIL_BLOCK - 1) / TAIL_BLOCK); }
static int tail_grid_owned(const DevIn &in, const TailState &ts) { return tail_grid((in.nraw - ts.rank + ts.world - 1) / ts.world); }

void launch_tail_link(const DevState &st, const TailState &ts, unsigned long long base, uint32_t cluster_i, int nraw, int nclust, cudaStream_t s) {
  count_launch(1);
  const unsigned g = (unsigned)std::min<unsigned long long>(((unsigned long long)nraw + 255) / 256 + 1, 148ull * 8);
  k_tail_link<<<g, 256, 0, s>>>(st, ts, base, cluster_i, nraw, nclust);
}
void launch_tail_pass(const DevState &st, const DevIn &in, const TailState &ts, int pass, int nclust, bool smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) { cudaFuncSetAttribute(k_tail_pass<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TAIL_SMEM_MAX); attr_set = true; }
  count_launch(1);
  const unsigned g = (tail_grid_owned(in, ts) + TAIL_RPT - 1) / TAIL_RPT;
  if (smem) k_tail_pass<true><<<g, TAIL_BLOCK, (size_t)nclust * 4, s>>>(st, in, ts, pass, nclust);
  else k_tail_pass<false><<<g, TAIL_BLOCK, 0, s>>>(st, in, ts, pass, nclust);
}
void launch_tail_final(const DevState &st, const DevIn &in, const TailState &ts, const BudParams &bp, int greedy, int detect_singletons,
                       int last_pass, int nclust, int mode, bool smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) { cudaFuncSetAttribute(k_tail_final<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TAIL_SMEM_MAX); attr_set = true; }
  count_launch(1);
  const unsigned g = (tail_grid_owned(in, ts) + TAIL_RPT - 1) / TAIL_RPT;
  if (smem) k_tail_final<true><<<g, TAIL_BLOCK, (size_t)nclust * 5 + 16, s>>>(st, in, ts, bp, greedy, detect_singletons, last_pass, nclust, mode);
  else k_tail_final<false><<<g, TAIL_BLOCK, 0, s>>>(st, in, ts, bp, greedy, detect_singletons, last_pass, nclust, mode);
}

void launch_bud_collect_owned(const DevState &st, const DevIn &in, const TailState &ts, const BudParams &bp, uint32_t *ties, uint32_t *ties_pr,
                              unsigned cap, cudaStream_t s) {
  count_launch(1);
  k_bud_collect_owned<<<tail_grid_owned(in, ts), TAIL_BLOCK, 0, s>>>(st, in, ts, bp, ties, ties_pr, cap);
}
void launch_mask_unowned(double *p, uint8_t *correct, int nraw, int rank, int world, cudaStream_t s) {
  count_launch(1);
  k_mask_unowned<<<(nraw + 255) / 256, 256, 0, s>>>(p, correct, nraw, rank, world);
}
void launch_posthoc_owned(const DevState &st, int nraw, unsigned long long n_entries, const int *center_cluster, uint32_t *trip_ij, double *trip_v,
                          unsigned cap, unsigned long long *count, int rank, int world, cudaStream_t s) {
  if (!n_entries) return;
  count_launch(1);
  k_posthoc_owned<<<(unsigned)((n_entries + 255) / 256), 256, 0, s>>>(st, n_entries, center_cluster, trip_ij, trip_v, cap, count, rank, world, nraw);
}

}  // namespace dd2
