// k_nwlane<B, G>: the row-sweep NW of dd_nwrow.cu with G lanes per (centre, raw) pair, for rounds with FEW pairs.
// Product code (sm_90a).
//
// Why: one thread per pair is the throughput layout, but a round with a few thousand pairs leaves most of the chip idle
// and then costs the full latency of one thread's 250 x 33 dependent cells (~80 us measured), twice when a bound pass
// and an exact pass follow each other.  Here the band's W = 2B+1 slots are split over G lanes (C = ceil(W/G) slots each),
// the lanes sweep rows in a software pipeline -- lane g works on row t - g at step t, so the left input (lane g-1, same
// row) was produced one step earlier and the up input (lane g+1, previous row) is its first cell of the same step, which
// every lane computes before the exchange -- and ONE launch does everything a pair of the loop needs:
//   DP with recorded moves  ->  nsubs  ->  store-rule bound (lambda <= S_r * rho_r^nsubs, dd_round.cu:k_raw_bounds)
//   ->  for the survivors: traceback, lambda in raw-position order, store rule (cluster.cpp:179-201).
// Two shuffles per lane and row; the dependent chain per step is C cells instead of W.
// Same cell update, same word layout, same boundary rules as dd_nwrow.cu (see there for the reference lines).
// The kernel only runs when the round has at most `lane_max` jobs (device-side count); above that it returns at once and
// the thread-per-pair kernels, which return at once below it, do the work.
#include "dd_common.h"
#include "dd_kernels.h"
#include "dd_nwrow.cuh"
#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace dd2 {

namespace {

struct LaneArgs {
  FwdArgs f;
  uint32_t *uneq_list;                 // raws not as long as the centre -> lane-group forward-carry kernel
  unsigned long long *uneq_count;
  uint32_t *mv_scratch;                // [row][lane g][group] 2-bit moves of the group's current pair
  uint16_t *sub_scratch;               // [k][group] substitutions found by the traceback: raw position | centre base << 14
  unsigned long long lane_max;         // run only if the round has at most this many jobs
};

}  // namespace

// Per-lane state of the pipelined sweep.
template <int C> struct LaneState {
  int S[C];                 // this lane's slots of the current row (clean words)
  uint32_t win;             // 2-bit raw bases under the slots
  uint32_t rw;              // rest of the packed raw word the next window base comes from
  int ridx;                 // index of that base
  int i;                    // row this lane handles in the current step
  int pinval;               // -(i-1) * match << 16: the ends-free zero of column 0 in biased space
  uint32_t *mvp;            // where the moves of row i go
  uint32_t gacc;            // OR of the main-diagonal cells' words (prec field in place): non-zero prec = the traced path leaves the diagonal
};

// One step of one lane: row st.i of its C slots, in place.  CHECKED: boundary rules on (rows near the matrix edges);
// GUARD: the lane may be outside rows 1..L (pipeline fill / drain) and must then leave its state alone.
template <int B, int G, int C, bool CHECKED, bool GUARD>
__device__ __forceinline__ void lane_step(LaneState<C> &st, const RowConsts &c, const uint8_t *s_cen, const uint32_t *rrow, int SW, int L, int g, int klast,
                                          bool act, size_t mv_row_stride) {
  constexpr int SENT = NW_SENT_H * 65536;
  const int i = st.i;
  const bool on = !GUARD || (act && i >= 1 && i <= L);
  const uint32_t cb = s_cen[GUARD ? min(max(i - 1, 0), L - 1) : i - 1];
  const uint32_t x = st.win ^ (cb * 0x55555555u);
  const uint32_t mm = x | (x >> 1);                    // even bits: mismatch flags (only those are read below)
  int left = __shfl_up_sync(0xffffffffu, st.S[C - 1], 1, G);          // lane g-1 finished this row one step ago
  if (g == 0) left = SENT;
  const int dpin = B - i - g * C, dfree = L - i + B - g * C;            // local slot of column 0 / column L in this row
  const int cLrow = (CHECKED && i == L) ? c.cL0 : c.cL;
  const int pin = st.pinval - c.matchS;
  uint32_t mv = 0, mdiag = 0;
  constexpr int GO = B / C, KO = B % C;                                   // lane / local slot of the main diagonal (slot B)
  int S0 = st.S[0];
  {  // cell 0 first: the lane below needs it as its up input of this very step
    const int diag = S0 + (int)__umulhi(mm << 31, 2u) * c.delta;
    const int up = (0 == klast) ? SENT : st.S[1];
    const int cu = (CHECKED && 0 == dfree) ? c.cU0 : c.cU;
    int m = __viaddmax_s32(left, cLrow, __viaddmax_s32(up, cu, diag));
    mv = __funnelshift_r(mv, (uint32_t)m >> 14, 2);
    if (KO == 0) mdiag = (uint32_t)m;
    m &= NW_CLR;
    if (CHECKED && 0 == dpin) m = pin;
    if (on) S0 = m;
    left = m;
  }
  int upin = __shfl_down_sync(0xffffffffu, S0, 1, G);                   // lane g+1's first slot of the previous row
  if (g == G - 1) upin = SENT;
  if (on) st.S[0] = S0;
#pragma unroll
  for (int k = 1; k < C; k++) {
    const int diag = st.S[k] + (int)__umulhi(mm << (31 - 2 * k), 2u) * c.delta;
    int up = (k + 1 < C) ? st.S[k + 1] : upin;
    if (k == klast) up = SENT;                                            // slot W-1: the neighbour above is out of band
    const int cu = (CHECKED && k == dfree) ? c.cU0 : c.cU;
    int m = __viaddmax_s32(left, cLrow, __viaddmax_s32(up, cu, diag));
    mv = __funnelshift_r(mv, (uint32_t)m >> 14, 2);                       // cell k ends at bits 32 - 2 (C - k)
    if (k == KO) mdiag = (uint32_t)m;
    m &= NW_CLR;
    if (CHECKED && k == dpin) m = pin;
    if (on) st.S[k] = m;
    left = m;
  }
  if (on) {
    if (g == GO) st.gacc |= mdiag;
    st.pinval = pin;
    *st.mvp = mv;
    st.mvp += mv_row_stride;
    st.win = (st.win >> 2) | ((st.rw & 3u) << (2 * (C - 1)));            // raw base ridx enters at the top slot for row i+1
    st.rw >>= 2;
    st.ridx++;
    if ((st.ridx & 15) == 0) st.rw = (st.ridx >= 0 && (st.ridx >> 4) < SW) ? rrow[st.ridx >> 4] : 0u;
  }
  st.i = i + 1;
}

template <int B, int G>
__global__ void __launch_bounds__(128) k_nwlane(LaneArgs la) {
  constexpr int W = 2 * B + 1;
  constexpr int C = (W + G - 1) / G;                    // slots per lane
  static_assert(C <= 16 && C >= 2, "one window register and one move word per lane and row");
  constexpr int SENT = NW_SENT_H * 65536;
  const FwdArgs &a = la.f;
  extern __shared__ uint32_t smem[];
  const int ncol = a.P.ncol;
  double *s_err = (double *)smem;
  uint8_t *s_cen = (uint8_t *)(smem + 2 * (16 * ncol));
  const unsigned long long njobs = *a.njobs_ptr;
  constexpr int GPB = 128 / G;                          // groups (pairs) per block
  if (njobs > la.lane_max || (unsigned long long)blockIdx.x * GPB >= njobs) return;
  const int L = (int)a.in.len[a.centre_idx];
  {
    const uint32_t *crow = a.in.seq2 + (size_t)a.centre_idx * a.in.SW;
    for (int p = threadIdx.x; p < L; p += blockDim.x) s_cen[p] = (uint8_t)((crow[p >> 4] >> (2 * (p & 15))) & 3u);
    for (int x = threadIdx.x; x < 16 * ncol; x += blockDim.x) s_err[x] = a.st.err[x];
  }
  __syncthreads();
  const RowConsts c = row_consts(a.P);
  const int lane = threadIdx.x & 31, g = lane % G;
  const size_t TG = (size_t)gridDim.x * GPB, grp = (size_t)blockIdx.x * GPB + threadIdx.x / G;
  const int d0 = g * C;                                 // first slot of this lane
  const int klast = W - 1 - d0;                         // local index of slot W-1 (>= C: not in this lane; < 0: only padding here)
  const int SW = a.in.SW;
  long long cells_lane = 0;
  const long long cells_pair = band_cells_cf(L, L, B, B);
  int errflag = 0;

  for (unsigned long long base = (unsigned long long)blockIdx.x * GPB; base < njobs; base += (unsigned long long)gridDim.x * GPB) {
    const unsigned long long jb = base + threadIdx.x / G;
    bool act = jb < njobs;
    const uint32_t r = act ? a.jobs[jb] : 0u;
    const bool uneq = act && (int)a.in.len[r] != L;
    warp_append(uneq && g == 0, r, la.uneq_list, la.uneq_count);
    act = act && !uneq;
    const uint32_t *rrow = a.in.seq2 + (size_t)r * SW;
    auto raw_base = [&](int p) -> uint32_t { return (p >= 0 && p < L) ? (rrow[p >> 4] >> (2 * (p & 15))) & 3u : 0u; };
    LaneState<C> st;
#pragma unroll
    for (int k = 0; k < C; k++) { const int d = d0 + k; st.S[k] = (d >= B && d < W) ? 0 : SENT; }   // row 0: columns 0..B are the ends-free zeros
    st.win = 0;                                         // row 1: slot d <-> raw base d - B
#pragma unroll
    for (int k = 0; k < C; k++) st.win |= raw_base(d0 + k - B) << (2 * k);
    st.ridx = d0 + C - B;                               // the base that enters at the top slot for row 2
    st.rw = (st.ridx >= 0 && (st.ridx >> 4) < SW) ? rrow[st.ridx >> 4] : 0u;
    st.rw >>= 2 * (st.ridx & 15);
    st.pinval = 0;
    st.gacc = 0u;
    st.i = 1 - g;                                       // software pipeline: lane g handles row t - g at step t
    st.mvp = la.mv_scratch + (size_t)g * TG + grp;
    const size_t mrs = (size_t)G * TG;
    int t = 1;
    // fill (some lanes not started), then boundary rows, interior rows, boundary rows, drain: every branch is block-uniform
    for (; t <= min(B + G - 1, L + G - 1); t++) lane_step<B, G, C, true, true>(st, c, s_cen, rrow, SW, L, g, klast, act, mrs);
    for (; t <= L - B; t++) lane_step<B, G, C, false, false>(st, c, s_cen, rrow, SW, L, g, klast, act, mrs);
    for (; t <= L + G - 1; t++) lane_step<B, G, C, true, true>(st, c, s_cen, rrow, SW, L, g, klast, act, mrs);
    __syncwarp();                                       // the moves written by the other lanes are visible to the owner
    // ---- the lane holding cell (L, L) (slot B) finishes the pair on its own ----
    constexpr int GO = B / C, KO = B % C;
    const bool owner = act && g == GO;
    int ns = 0;
#pragma unroll
    for (int k = 0; k < C; k++) if (k == KO) ns = st.S[k] & NW_NMASK;
    bool survive = owner;
    if (owner && a.cluster_i != 0) {
      const double bound = a.raw_S[r] * pow(a.raw_rho[r], (double)ns) * (double)a.total_reads * (1.0 + 1e-9);
      survive = !(bound <= a.st.E_minmax[r]) || bound < 1e-280;
    }
    if (owner && a.ns_out) a.ns_out[r] = (uint32_t)ns | (survive ? 0x80000000u : 0u);
    if (owner && !a.no_cells) cells_lane += cells_pair;
    // Every main-diagonal cell took the diagonal move strictly: the traced path is the gapless alignment (DESIGN.md 4.2), no walk
    // needed -- and its lambda is formed by the whole lane group: lane g looks up the factor of position p0 + g (bases, quality,
    // table: ~20 instructions), the group then multiplies the G factors IN POSITION ORDER through shuffles, so the owner's chain
    // is one DMUL per position instead of the ~22 dependent instructions of a one-lane loop (x * 1.0 pads the tail exactly).
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
    const int gbase = lane & ~(G - 1);
    const int diag_grp = __shfl_sync(gmask, (int)(survive && !(st.gacc & 0xC000u)), gbase + GO);
    if (diag_grp) {
      const uint32_t rg = __shfl_sync(gmask, r, gbase + GO);
      const uint32_t *rr2 = a.in.seq2 + (size_t)rg * SW;
      const uint8_t *qrow = a.in.qual + (size_t)rg * a.in.QS;
      auto factor = [&](int p, int &mis) -> double {
        if (p >= L) return 1.0;
        const uint32_t b = (rr2[p >> 4] >> (2 * (p & 15))) & 3u, cb = s_cen[p];
        int q = a.P.use_quals ? (int)qrow[p] : 0;
        if (q > ncol - 1) { errflag = ERR_QUAL; q = ncol - 1; }
        mis += (b != cb) ? 1 : 0;
        return s_err[(4u * cb + b) * ncol + q];                               // cb == b: 5 b, the self transition (pval.cpp:158-193)
      };
      double lam = 1.0;
      int mis = 0;
      double f = factor(g, mis);
      for (int p0 = 0; p0 < L; p0 += G) {
        const double fn = factor(p0 + G + g, mis);                           // next block's factor: its loads overlap this block's products
#pragma unroll
        for (int k = 0; k < G; k++) lam = lam * __shfl_sync(gmask, f, gbase + k);
        f = fn;
      }
#pragma unroll
      for (int o = G / 2; o; o >>= 1) mis += __shfl_xor_sync(gmask, mis, o);
      if (survive) {
        if (mis != ns) errflag = ERR_TRACE;     // the forward-carried count and the diagonal's Hamming distance must agree
        if (lam < 0 || lam > 1 || lam != lam) errflag = ERR_LAMBDA;             // pval.cpp:195
        store_comparison(a, r, lam, ns);
      }
    } else if (survive) {
      // traceback over the recorded moves, lambda in raw-position order, store rule (dd_nwrow.cuh)
      const int nsub = trace_moves<G, C, 8, true>(la.mv_scratch + grp, (size_t)G * TG, TG, L, B, s_cen, rrow, la.sub_scratch + grp, TG);
      const double lam = lambda_from_subs(rrow, a.in.qual + (size_t)r * a.in.QS, L, ncol, a.P.use_quals, s_err, la.sub_scratch + grp, TG, nsub, &errflag);
      if (nsub != ns) errflag = ERR_TRACE;
      if (lam < 0 || lam > 1 || lam != lam) errflag = ERR_LAMBDA;               // pval.cpp:195
      store_comparison(a, r, lam, ns);
    }
    __syncwarp();
  }
  if (errflag) atomicMax(&a.st.ctr[CTR_ERR], (unsigned long long)errflag);
#pragma unroll
  for (int o = 16; o; o >>= 1) cells_lane += __shfl_xor_sync(0xffffffffu, cells_lane, o);
  if (lane == 0 && cells_lane) atomicAdd(&a.st.ctr[CTR_CELLS], (unsigned long long)cells_lane);
}

int nwlane_lanes(int band) { return band == 32 ? 16 : (band == 16 ? 8 : 4); }        // 5 slots per lane in every case
// scratch for `groups` pairs in flight
size_t nwlane_mv_words(int band, int maxlen, int groups) { return (size_t)groups * (size_t)maxlen * nwlane_lanes(band); }
size_t nwlane_sub_halfwords(int maxlen, int groups) { return (size_t)groups * (size_t)maxlen; }

// Everything a small round's NW pairs need, in one launch.  Returns false when the configuration is not covered (the
// caller then runs the thread-per-pair kernels for every round size).  lane_max: job-count threshold; groups_cap: pairs
// in flight the scratch was sized for.
bool launch_nwlane(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, uint32_t *mv_scratch, uint16_t *sub_scratch, int len1,
                   unsigned long long lane_max, int groups_cap, cudaStream_t s) {
  if (!nwrow_applicable(f, len1) || !mv_scratch || !sub_scratch) return false;
  LaneArgs a{f, uneq_list, uneq_count, mv_scratch, sub_scratch, lane_max};
  const int G = nwlane_lanes(f.P.band), gpb = 128 / G;
  const int grid = std::max(1, groups_cap / gpb);
  const size_t smem = (size_t)16 * f.P.ncol * 8 + (size_t)((f.in.maxlen + 15) & ~15);
  count_launch(1);
  if (f.P.band == 16) k_nwlane<16, 8><<<grid, 128, smem, s>>>(a);
  else if (f.P.band == 8) k_nwlane<8, 4><<<grid, 128, smem, s>>>(a);
  else k_nwlane<32, 16><<<grid, 128, smem, s>>>(a);
  return true;
}

}  // namespace dd2
