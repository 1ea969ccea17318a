// k_nwrow<B>: banded ends-free NW, ONE THREAD PER (centre, raw) PAIR, the whole band of a DP row in registers.
// Product code (sm_90a).  Replaces the anti-diagonal lane-group kernels for the loop comparisons of equal-length pairs
// (every pair of a fixed-length amplicon run).
//
// What it restates: nwalign_endsfree / nwalign_vectorized2 (/root/reference/src/nwalign_endsfree.cpp:76-216,
// nwalign_vectorized.cpp:71-318), al2subs' substitution count (nwalign_endsfree.cpp:570-639) and, in the exact
// variant, compute_lambda_ts (pval.cpp:144-197) + the store rule of b_compare (cluster.cpp:179-201).
//
// Layout.  Row i of the DP matrix (i over the centre) lives in W = 2*B + 1 registers, slot d <-> column
// j = i + d - B.  A row is swept in place in ascending d: cell (i, j) reads old[d] (diag), old[d + 1] (up) and the
// freshly written new[d - 1] (left).  No lane ever talks to another lane: no shuffles, no shared-memory traffic in the
// sweep, and the dependent chain per cell is one VIADDMNMX + one LOP3.
//
// One 32-bit word per cell carries everything the reference's traceback would need to know about the path into it:
//     V = score << 16  |  prec << 14  |  nsubs          (nsubs < 2^14)
// Candidates are formed by adding a constant to the clean (prec = 0) predecessor words: up gets prec 2, left prec 1,
// diag prec 0 -- so ONE signed max over the three words picks the best score and, among equal scores, the
// reference's precedence up > left > diag (nwalign_endsfree.cpp:147-156), and the substitution count of the chosen
// predecessor rides along in the low bits (+1 on a mismatching diagonal move).  The prec field is cleared after the
// max; it is also exactly the 2-bit move of the cell, which the exact variant records for its traceback.
// Scores are kept relative to i * match (S = V - i * (match << 16)): the diagonal candidate of a matching pair is then
// the stored word itself and a mismatch adds one constant, selected by an integer multiply-add (FMA pipe) so that the
// ALU pipe only sees the two max instructions and the clear: 3 ALU + 3 FMA-pipe instructions per cell.
//
// Boundaries (all warp-uniform, the centre and hence the row index are shared by every pair of a launch):
//   rows i <= B       : the slot of column 0 is pinned to the ends-free value 0 (nwalign_endsfree.cpp:89-92)
//   rows i >  L - B   : the cell in column L takes the up move without a gap cost (:138-142)
//   row  i == L       : left moves are free (:131-135)
//   out-of-band neighbours (slot -1, slot W) are a constant far below any real score (:113-119).
#include "dd_common.h"
#include "dd_kernels.h"
#include "dd_nwrow.cuh"
#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace dd2 {

namespace {

struct RowArgs {
  FwdArgs f;
  uint32_t *uneq_list;                 // jobs this kernel does not take (len2 != len1) -> lane-group kernels
  unsigned long long *uneq_count;
  uint32_t *mv_scratch;                // EXACT: [row][word][thread] 2-bit moves of the thread's current pair
  uint16_t *sub_scratch;               // EXACT: [k][thread] substitutions found by the traceback: raw position | centre base << 14
  unsigned long long lane_max;         // BOUND / EXACT: job lists with at most this many entries belong to k_nwlane (dd_nwlane.cu)
  uint32_t *ns_out;                    // BOUND, test hook only: nsubs per raw (NULL in the product path)
};

enum RowMode : int { ROW_BOUND = 0, ROW_FINAL = 1, ROW_EXACT = 2 };

}  // namespace

// MODE ROW_BOUND  (loop, pass 1 of the two-phase scheme, DESIGN.md 4.2): substitution count of the traced path for every
//                 job, then lambda <= S_r * rho_r^nsubs decides whether the pair can pass the store rule (cluster.cpp:192);
//                 survivors whose path leaves the main diagonal are listed for the exact pass, the others (every main-diagonal
//                 cell took the diagonal move strictly: the traced path IS the gapless alignment) for k_gapless_loop.
// MODE ROW_EXACT  (loop): the moves of every row go to a per-thread scratch column, the thread walks its path back
//                 (nwalign_endsfree.cpp:169-188), notes the substituted raw positions (al2subs) and multiplies lambda in
//                 raw-position order (compute_lambda_ts, pval.cpp:190-193: bit-identical), then applies the store rule
//                 of b_compare (cluster.cpp:179-201).
// MODE ROW_FINAL  (FinalSubsParallel, Rmain.cpp:179-236: every raw against its own centre; all sequences equally long):
//                 nsubs of the final alignment and whether the traced path is the pure diagonal (column list trivial)
//                 or contains gaps (-> traceback kernel k_align<FINAL>).
// Jobs whose raw is not as long as the centre are handed back through uneq_list.
template <int B, int MODE>
__global__ void __launch_bounds__(128) k_nwrow(RowArgs ra) {
  constexpr int W = 2 * B + 1;
  constexpr int NWW = (2 * W + 31) / 32;                 // 32-bit words of the 2-bit raw window / mismatch mask / moves of a row
  constexpr int TOPSH = 4 * B - 32 * (NWW - 1);          // bit offset of slot 2B in the top window word
  const FwdArgs &a = ra.f;
  extern __shared__ uint32_t smem[];
  const int ncol = a.P.ncol;
  double *s_err = (double *)smem;                        // EXACT: 16 x ncol transition table
  uint8_t *s_cen = (uint8_t *)(smem + (MODE == ROW_EXACT ? 2 * (16 * ncol) : 0));
  const unsigned long long njobs = *a.njobs_ptr;
  if ((unsigned long long)blockIdx.x * blockDim.x >= njobs) return;
  if (MODE != ROW_FINAL && njobs <= ra.lane_max) return;       // this many jobs or fewer: k_nwlane's launch does them
  const int L = (MODE == ROW_FINAL) ? a.in.maxlen : (int)a.in.len[a.centre_idx];
  if (MODE != ROW_FINAL) {
    const uint32_t *crow = a.in.seq2 + (size_t)a.centre_idx * a.in.SW;
    for (int p = threadIdx.x; p < L; p += blockDim.x) s_cen[p] = (uint8_t)((crow[p >> 4] >> (2 * (p & 15))) & 3u);
  }
  if (MODE == ROW_EXACT) for (int x = threadIdx.x; x < 16 * ncol; x += blockDim.x) s_err[x] = a.st.err[x];
  __syncthreads();
  const RowConsts c = row_consts(a.P);
  const int lane = threadIdx.x & 31;
  const size_t T = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  long long cells_lane = 0;
  const long long cells_pair = band_cells_cf(L, L, B, B);
  int errflag = 0;

  for (unsigned long long wbase = ((unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u)); wbase < njobs;
       wbase += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long jb = wbase + lane;
    bool act = jb < njobs;
    const uint32_t r = act ? (a.jobs ? a.jobs[jb] : (uint32_t)jb * (uint32_t)a.job_mul + (uint32_t)a.job_add) : 0u;
    uint32_t cidx = a.centre_idx;
    if (MODE == ROW_FINAL && act) cidx = a.st.cl_center[a.st.cluster_of[r]];
    const bool uneq = act && ((int)a.in.len[r] != L || (MODE == ROW_FINAL && (int)a.in.len[cidx] != L));
    warp_append(uneq, r, ra.uneq_list, ra.uneq_count);
    act = act && !uneq;
    int ns = 0;
    bool gapped = false;
    const uint32_t *rrow = a.in.seq2 + (size_t)r * a.in.SW;
    if (act) {
      const uint32_t *crow = a.in.seq2 + (size_t)cidx * a.in.SW;
      int S[W];
      uint32_t win[NWW], mm[NWW], mv[NWW];
      // row 0: columns 0..B are the ends-free zeros (slots B..2B); slots below hold no cell
#pragma unroll
      for (int d = 0; d < W; d++) S[d] = (d >= B) ? 0 : NW_SENT_H * 65536;
      // raw window of row 1: slot d <-> raw base d - B  (slots < B: none)
#pragma unroll
      for (int w = 0; w < NWW; w++) win[w] = 0u;
      uint32_t rw = rrow[0];
#pragma unroll
      for (int k = 0; k <= B; k++) {            // B + 1 <= 33 bases: at most three packed words
        if (k > 0 && (k & 15) == 0) rw = (k >> 4) < a.in.SW ? rrow[k >> 4] : 0u;
        const uint32_t nb = (rw >> (2 * (k & 15))) & 3u;
        const int slot = B + k;
        win[slot >> 4] |= nb << (2 * (slot & 15));
      }
      int idx = B + 1;                          // next raw base to enter the window
      rw = (idx >> 4) < a.in.SW ? rrow[idx >> 4] : 0u;
      rw >>= 2 * (idx & 15);
      int pinval = 0;
      uint32_t cw = 0, gacc = 0;
      for (int i = 1; i <= L; i++) {
        uint32_t cb;
        if (MODE == ROW_FINAL) { if (((i - 1) & 15) == 0) cw = crow[(i - 1) >> 4]; cb = cw & 3u; cw >>= 2; }
        else cb = s_cen[i - 1];
        const uint32_t cen = cb * 0x55555555u;
#pragma unroll
        for (int w = 0; w < NWW; w++) { const uint32_t x = win[w] ^ cen; mm[w] = x | (x >> 1); }   // even bits: mismatch flags (mis_bit reads nothing else; an
                                                                                                   // `& 0x55555555` here is sunk by the compiler into one LOP3 per cell)
        pinval -= c.matchS;
        int mB;
        if (i > B && i <= L - B) mB = nw_row<B, false, MODE == ROW_EXACT>(S, mm, c, c.cL, -1, 0, -1, mv);
        else mB = nw_row<B, true, MODE == ROW_EXACT>(S, mm, c, i == L ? c.cL0 : c.cL, B - i, pinval, L - i + B, mv);
        if (MODE != ROW_EXACT) gacc |= (uint32_t)mB;          // prec of the main-diagonal cell: non-zero = the path leaves the diagonal here
        if (MODE == ROW_EXACT) {
#pragma unroll
          for (int w = 0; w < NWW; w++) ra.mv_scratch[((size_t)(i - 1) * NWW + w) * T + tid] = mv[w];
        }
        // advance the window: drop slot 0, raw base idx enters at slot 2B
#pragma unroll
        for (int w = 0; w + 1 < NWW; w++) win[w] = __funnelshift_r(win[w], win[w + 1], 2);
        win[NWW - 1] = (win[NWW - 1] >> 2) | ((rw & 3u) << TOPSH);
        idx++;
        rw >>= 2;
        if ((idx & 15) == 0) rw = (idx >> 4) < a.in.SW ? rrow[idx >> 4] : 0u;
      }
      ns = S[B] & NW_NMASK;                     // cell (L, L)
      gapped = (gacc & 0xC000u) != 0u;
      if (!(MODE == ROW_EXACT && a.no_cells)) cells_lane += cells_pair;
    }
    if (MODE == ROW_BOUND) {
      if (ra.ns_out && act) ra.ns_out[r] = (uint32_t)ns;
      // lambda <= S_r * rho_r^nsubs for ANY alignment with nsubs substitutions (dd_round.cu:k_raw_bounds)
      bool survive = false;
      if (act) {
        const double bound = a.raw_S[r] * pow(a.raw_rho[r], (double)ns) * (double)a.total_reads * (1.0 + 1e-9);
        survive = !(bound <= a.st.E_minmax[r]) || bound < 1e-280;     // near underflow the fp product is not a safe bound: keep
      }
      // a survivor whose traced path is the pure diagonal is the gapless alignment (same columns, same lambda): it joins the
      // gapless jobs of this round (k_gapless_loop) instead of the exact pass, which then only records moves for real gaps
      const bool diag = survive && !gapped && a.gl_out != nullptr;
      warp_append(diag, r, a.gl_out, a.gl_count);
      warp_append(survive && !diag, r, a.surv_list, a.surv_count);
    } else if (MODE == ROW_FINAL) {
      if (act) a.st.nsubs_final[r] = (uint32_t)ns;
      warp_append(act && !gapped, r, a.gl_out, a.gl_count);
      warp_append(act && gapped, r, a.nw_out, a.nw_count);
    } else if (act) {
      // ---- traceback over the recorded moves, lambda in raw-position order, store rule (dd_nwrow.cuh) ----
      const int nsub = trace_moves<NWW, 16, 8>(ra.mv_scratch + tid, (size_t)NWW * T, T, L, B, s_cen, rrow, ra.sub_scratch + tid, T);
      const double lam = lambda_from_subs(rrow, a.in.qual + (size_t)r * a.in.QS, L, ncol, a.P.use_quals, s_err, ra.sub_scratch + tid, T, nsub, &errflag);
      if (nsub != ns) errflag = ERR_TRACE;      // the forward-carried count and the traced path must agree
      if (lam < 0 || lam > 1 || lam != lam) errflag = ERR_LAMBDA;               // pval.cpp:195
      store_comparison(a, r, lam, ns);
    }
  }
  if (errflag) atomicMax(&a.st.ctr[CTR_ERR], (unsigned long long)errflag);
#pragma unroll
  for (int o = 16; o; o >>= 1) cells_lane += __shfl_xor_sync(0xffffffffu, cells_lane, o);
  if (lane == 0 && cells_lane) atomicAdd(&a.st.ctr[CTR_CELLS], (unsigned long long)cells_lane);
}

template <int B, int MODE> static void launch_row(const RowArgs &a, int grid, size_t smem, cudaStream_t s) {
  k_nwrow<B, MODE><<<grid, 128, smem, s>>>(a);
}
template <int MODE> static void launch_row_band(const RowArgs &a, int grid, size_t smem, cudaStream_t s) {
  if (a.f.P.band == 16) launch_row<16, MODE>(a, grid, smem, s);
  else if (a.f.P.band == 8) launch_row<8, MODE>(a, grid, smem, s);
  else launch_row<32, MODE>(a, grid, smem, s);
}

// Can the thread-per-pair kernels take this launch at all?  (band instantiated, scores inside the 16-bit score field,
// plain gap costs, band narrower than the centre so that the reference fills its band boundaries)
bool nwrow_applicable(const FwdArgs &f, int len1) {
  const AlnParams &P = f.P;
  if (P.homo || P.band < 0) return false;
  if (!(P.band == 8 || P.band == 16 || P.band == 32)) return false;
  if (len1 < P.band + 2 || len1 >= 16000) return false;
  const long amax = std::max(std::max(std::abs(P.match), std::abs(P.mismatch)), std::abs(P.gap));
  const long worst = (long)(std::abs(P.match) + amax) * len1 + 80L * (amax + std::abs(P.match));
  if (worst >= 15000) return false;          // |biased score| stays well inside (NW_SENT_H, 32767 + NW_SENT_H)
  if (P.match < 0) return false;
  return true;
}

static int row_grid(unsigned long long njobs_upper, int num_sms, int per_sm) {
  const unsigned long long blocks = (njobs_upper + 127) / 128;
  return (int)std::min<unsigned long long>(std::max<unsigned long long>(blocks, 1ull), (unsigned long long)num_sms * per_sm);
}


// k_gapless_loop: the loop comparisons raw_align settles WITHOUT a DP (kodist == kdist: nwalign_gapless, nwalign_endsfree.cpp:539-555:
// position i against position i, the shorter sequence padded with '-' at its end).  One thread per pair: the substitution
// count is the Hamming distance of the packed rows over the common length; pairs that cannot pass the store rule leave after
// the bound test; the rest multiply lambda in raw-position order (compute_lambda_ts) and apply the store rule.  Any lengths.
__global__ void __launch_bounds__(128) k_gapless_loop(FwdArgs a, int use_bound) {
  extern __shared__ uint32_t smem[];
  const int ncol = a.P.ncol;
  double *s_err = (double *)smem;
  uint32_t *s_crow = smem + 2 * (16 * ncol);           // the centre's packed row
  const unsigned long long njobs = *a.njobs_ptr;
  if ((unsigned long long)blockIdx.x * blockDim.x >= njobs) return;
  const int SW = a.in.SW, len1 = (int)a.in.len[a.centre_idx];
  for (int x = threadIdx.x; x < SW; x += blockDim.x) s_crow[x] = a.in.seq2[(size_t)a.centre_idx * SW + x];
  for (int x = threadIdx.x; x < 16 * ncol; x += blockDim.x) s_err[x] = a.st.err[x];
  __syncthreads();
  int errflag = 0;
  for (unsigned long long jb = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; jb < njobs; jb += (unsigned long long)gridDim.x * blockDim.x) {
    const uint32_t r = a.jobs[jb];
    const int len2 = (int)a.in.len[r], lc = min(len1, len2);
    const uint32_t *rrow = a.in.seq2 + (size_t)r * SW;
    int ns = 0;
    for (int w = 0; w * 16 < lc; w++) {
      const uint32_t x = rrow[w] ^ s_crow[w];
      uint32_t mis = (x | (x >> 1)) & 0x55555555u;
      const int left = lc - w * 16;
      if (left < 16) mis &= (1u << (2 * left)) - 1u;
      ns += __popc(mis);
    }
    bool survive = true;
    if (use_bound && a.cluster_i != 0) {               // lambda <= S_r * rho_r^nsubs (dd_round.cu:k_raw_bounds): unstorable pairs stop here
      const double bound = a.raw_S[r] * pow(a.raw_rho[r], (double)ns) * (double)a.total_reads * (1.0 + 1e-9);
      survive = !(bound <= a.st.E_minmax[r]) || bound < 1e-280;
    }
    if (a.ns_out) a.ns_out[r] = (uint32_t)ns | (survive ? 0x80000000u : 0u);
    if (!survive) continue;
    const uint8_t *qrow = a.in.qual + (size_t)r * a.in.QS;
    double lam = 1.0;
    uint4 qn = *(const uint4 *)qrow;
    for (int p0 = 0; p0 < len2; p0 += 16) {
      const uint4 qv = qn;
      if (p0 + 16 < len2) qn = *(const uint4 *)(qrow + p0 + 16);
      uint32_t bw = rrow[p0 >> 4], cw = s_crow[p0 >> 4];
      const uint32_t qq[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
      for (int u = 0; u < 16; u++) {
        const int p = p0 + u;
        if (p < len2) {
          const uint32_t b = bw & 3u, c = (p < len1) ? (cw & 3u) : b;       // beyond the centre: raw base against a gap = self transition
          int q = a.P.use_quals ? (int)((qq[u >> 2] >> (8 * (u & 3))) & 0xFFu) : 0;
          if (q > ncol - 1) { errflag = ERR_QUAL; q = ncol - 1; }
          lam = lam * s_err[(4u * c + b) * ncol + q];                        // c == b: 5 b, the self transition
        }
        bw >>= 2; cw >>= 2;
      }
    }
    if (lam < 0 || lam > 1 || lam != lam) errflag = ERR_LAMBDA;               // pval.cpp:195
    store_comparison(a, r, lam, ns);
  }
  if (errflag) atomicMax(&a.st.ctr[CTR_ERR], (unsigned long long)errflag);
}

void launch_gapless_loop(const FwdArgs &f, int use_bound, unsigned long long njobs_upper, int num_sms, cudaStream_t s) {
  const size_t smem = (size_t)16 * f.P.ncol * 8 + (size_t)f.in.SW * 4;
  count_launch(1);
  k_gapless_loop<<<row_grid(njobs_upper, num_sms, 16), 128, smem, s>>>(f, use_bound);
}

// Bound pass over f.jobs; jobs with len2 != len1 come back in uneq_list (count in *uneq_count, zeroed by the caller).
// false: nothing launched (the caller falls back to the lane-group kernels for every job).
bool launch_nwrow_bound(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, int len1, unsigned long long njobs_upper, int num_sms,
                        unsigned long long lane_max, cudaStream_t s, uint32_t *ns_out) {
  if (!nwrow_applicable(f, len1)) return false;
  RowArgs a{f, uneq_list, uneq_count, nullptr, nullptr, lane_max, ns_out};
  const size_t smem = (size_t)((f.in.maxlen + 15) & ~15);
  count_launch(1);
  launch_row_band<ROW_BOUND>(a, row_grid(njobs_upper, num_sms, 16), smem, s);
  return true;
}

// Final pass (every raw against its own centre); needs every sequence to have the same length.
bool launch_nwrow_final(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, unsigned long long njobs_upper, int num_sms,
                        cudaStream_t s) {
  if (f.in.minlen != f.in.maxlen || !nwrow_applicable(f, f.in.maxlen)) return false;
  RowArgs a{f, uneq_list, uneq_count, nullptr, nullptr, 0ull, nullptr};
  count_launch(1);
  launch_row_band<ROW_FINAL>(a, row_grid(njobs_upper, num_sms, 16), 16, s);
  return true;
}

// Exact pass: threads in flight are bounded by the scratch columns (rows x words of moves + substitutions per thread).
int nwrow_exact_grid(int num_sms, int nraw) { return std::max(1, std::min(num_sms * 6, (nraw + 127) / 128)); }
size_t nwrow_mv_words(int band, int maxlen, int grid) {
  const int W = 2 * band + 1, NWW = (2 * W + 31) / 32;
  return (size_t)grid * 128 * (size_t)maxlen * NWW;
}
size_t nwrow_sub_halfwords(int maxlen, int grid) { return (size_t)grid * 128 * (size_t)maxlen; }
bool nwrow_usable(const AlnParams &P, int len1) { FwdArgs f{}; f.P = P; return nwrow_applicable(f, len1); }

bool launch_nwrow_exact(const FwdArgs &f, uint32_t *uneq_list, unsigned long long *uneq_count, uint32_t *mv_scratch, uint16_t *sub_scratch, int len1,
                        unsigned long long njobs_upper, int grid_cap, cudaStream_t s, unsigned long long lane_max) {
  if (!nwrow_applicable(f, len1) || !mv_scratch || !sub_scratch) return false;
  RowArgs a{f, uneq_list, uneq_count, mv_scratch, sub_scratch, lane_max, nullptr};
  const size_t smem = (size_t)16 * f.P.ncol * 8 + (size_t)((f.in.maxlen + 15) & ~15);
  count_launch(1);
  launch_row_band<ROW_EXACT>(a, (int)std::min<unsigned long long>(std::max<unsigned long long>((njobs_upper + 127) / 128, 1ull), (unsigned long long)grid_cap), smem, s);
  return true;
}

}  // namespace dd2
