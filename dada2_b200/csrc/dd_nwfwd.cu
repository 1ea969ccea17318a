// k_nwfwd<G, ND, WL, HM>: register-resident banded ends-free NW for the LOOP comparisons (b_compare),
// G lanes per (centre, raw) pair, ND diagonals per lane.  Product code (sm_90a).
// The GENERAL loop aligner: any pair of lengths (band slots up to 256), homopolymer gap costs (HM).  Pairs as long as
// their centre with plain gap costs -- every pair of a fixed-length amplicon run -- take the thread-per-pair row kernels
// instead (dd_nwrow.cu / dd_nwlane.cu), which hand everything else over to this kernel through a job list.
//
// Replaces, for pairs that need a real alignment inside the divisive loop,
//   nwalign_vectorized2 / nwalign_endsfree   (/root/reference/src/nwalign_vectorized.cpp:71-318,
//                                             nwalign_endsfree.cpp:76-216)
//   al2subs + compute_lambda_ts              (nwalign_endsfree.cpp:570-639, pval.cpp:144-197)
//   the "selectively store" step             (cluster.cpp:179-201)
// The loop only consumes (lambda, nsubs) of each alignment, so no move matrix is stored and
// nothing is traced back: every DP cell carries, next to its score, the lambda product and the
// substitution count of the unique path the reference's traceback would follow to that cell
// (predecessor chosen with the reference's precedence up > left > diag).  lambda is multiplied
// along that path in raw-position order, i.e. in the exact order of pval.cpp:190-193, so it is
// bit-identical to trace-then-multiply.  The final pass (which needs per-position pairs) and
// anything this kernel cannot hold in registers go through k_align (dd_kernels.cu).
//
// Layout: anti-diagonal wavefront.  Band index dd = (j - i) + LB with LB = lb rounded up to even;
// lane gl of a group owns dd in [gl*ND, gl*ND + ND).  Step k = i + j updates the dd of parity k&1
// from neighbours of the other parity (step k-1) and itself (step k-2): ND/2 independent cells
// per lane per step, one neighbour exchange by warp shuffle.  The centre's bases stream up the
// lanes and the raw's bases/qualities stream down, one shuffle each per step (systolic).
#include "dd_common.h"
#include "dd_kernels.h"
#include <math_constants.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace dd2 {

// DP cells of a banded alignment (SURVEY.md 8d): sum_i [min(len2, i + rband) - max(1, i - lband) + 1], closed form.
__device__ __forceinline__ long long band_cells2(int n, int m, int l, int r) {
  const long long k = min(max(m - r, 0), n);
  const long long A = k * (k + 1) / 2 + k * r + (long long)(n - k) * m;
  const long long k2 = min(max(l + 1, 0), n);
  const long long B = k2 + ((long long)n * (n + 1) / 2 - k2 * (k2 + 1) / 2) - (long long)l * (n - k2);
  return A - B + n;
}

// One anti-diagonal step of the register-resident wavefront (cells of parity PAR), updated IN PLACE: a cell of parity
// PAR reads its neighbours of the other parity (unchanged during this step) and its own previous value only.
// FAST = interior step (no boundary cell, no free end gap, every pair running): branch-free, out-of-band slots kept
// below any real score by PEN.  Otherwise every cell is checked against the matrix borders and the band.
// select without a branch: ptxas otherwise turns the rare 'up' move into a divergent branch around the table lookup
__device__ __forceinline__ int sel_i32(bool p, int a, int b) {
#ifdef DADA2B_EMU
  return p ? a : b;
#else
  int r;
  asm("{.reg .pred q; setp.ne.s32 q, %3, 0; selp.s32 %0, %1, %2, q;}" : "=r"(r) : "r"(a), "r"(b), "r"((int)p));
  return r;
#endif
}

struct StepCtx {
  int gl, len1, len2, tlo, thi, nsteps, SENT, match, mismatch, gap, hgap, ncol4, ONE_IDX;
  int b2_off;            // byte offset of the pair's b2 table (entry 0) from the start of dynamic shared memory
};

// HM = homopolymer gap costs (nwalign_endsfree.cpp:220-396): a gap opposite a base that lies in a run >= 3 costs hgap; HA / HB
// carry that flag for the centre / raw base of every slot (bit cc <-> slot cc), like A / B carry the bases.
template <int G, int ND, bool WL, bool HM, int PAR, bool FAST>
__device__ __forceinline__ void nw_step(int (&H)[ND], int (&NSUB)[ND], double (&LAM)[ND], const int (&PEN)[ND], uint32_t A,
                                        uint32_t B, uint32_t HA, uint32_t HB, int I, int J, int k, const StepCtx &c) {
  constexpr int NSL = ND / 2;
  constexpr int BIGPEN = 1 << 20, GAPFLAG = 1 << 30, PADL = 64;
  // neighbour exchange: identical in both paths, unconditional
  int Hn, Nn;
  double Ln = 1.0;
  if (PAR == 0) {           // left neighbour of local t=0 is lane gl-1's t=ND-1
    Hn = __shfl_up_sync(0xffffffffu, H[ND - 1], 1, G);
    Nn = __shfl_up_sync(0xffffffffu, NSUB[ND - 1], 1, G);
    if (WL) Ln = __shfl_up_sync(0xffffffffu, LAM[ND - 1], 1, G);
    if (c.gl == 0) { Hn = FAST ? -BIGPEN : c.SENT; Nn = 0; Ln = 1.0; }
  } else {                  // up neighbour of local t=ND-1 is lane gl+1's t=0
    Hn = __shfl_down_sync(0xffffffffu, H[0], 1, G);
    Nn = __shfl_down_sync(0xffffffffu, NSUB[0], 1, G);
    if (WL) Ln = __shfl_down_sync(0xffffffffu, LAM[0], 1, G);
    if (c.gl == G - 1) { Hn = FAST ? -BIGPEN : c.SENT; Nn = 0; Ln = 1.0; }
  }
  const uint32_t X = A ^ B;
  const int Jp = J + PAR;
  extern __shared__ uint32_t smem[];                     // named directly: no generic-to-shared address conversion per load
  const double *s_err = (const double *)smem;             // the error table sits at offset 0
  const uint16_t *s_b2 = (const uint16_t *)((const unsigned char *)smem + c.b2_off);
  const uint16_t *b2p = s_b2 + (Jp - 1);
#pragma unroll
  for (int cc = 0; cc < NSL; cc++) {
    const int t = 2 * cc + PAR;
    const int hl = (PAR == 0 && cc == 0) ? Hn : H[t - 1 < 0 ? 0 : t - 1];
    const int nl = (PAR == 0 && cc == 0) ? Nn : NSUB[t - 1 < 0 ? 0 : t - 1];
    const double ll = (PAR == 0 && cc == 0) ? Ln : LAM[t - 1 < 0 ? 0 : t - 1];
    const int hu = (PAR == 1 && cc == NSL - 1) ? Hn : H[t + 1 >= ND ? ND - 1 : t + 1];
    const int nu = (PAR == 1 && cc == NSL - 1) ? Nn : NSUB[t + 1 >= ND ? ND - 1 : t + 1];
    const double lu = (PAR == 1 && cc == NSL - 1) ? Ln : LAM[t + 1 >= ND ? ND - 1 : t + 1];
    const uint32_t nt1 = (A >> (2 * cc)) & 3u, nt2 = (B >> (2 * cc)) & 3u;
    const bool eq = ((X >> (2 * cc)) & 3u) == 0u;
    if (FAST) {
      const int gl_ = (HM && ((HB >> cc) & 1u)) ? c.hgap : c.gap, gu_ = (HM && ((HA >> cc) & 1u)) ? c.hgap : c.gap;   // :303-320
      const int left = hl + gl_, up = hu + gu_, diag = H[t] + (eq ? c.match : c.mismatch);
      const int m = __vimax3_s32(left, up, diag);
      const bool isU = up == m;                      // precedence up > left > diag (nwalign_endsfree.cpp:147-156)
      const bool isL = (left == m) && !isU;
      if (WL) {
        const int idx = sel_i32(isU, c.ONE_IDX, (int)b2p[cc] + (int)(isL ? nt2 : nt1) * c.ncol4);
        const double lp = isU ? lu : (isL ? ll : LAM[t]);
        LAM[t] = lp * s_err[idx];
      }
      NSUB[t] = sel_i32(isU, nu | GAPFLAG, sel_i32(isL, nl | GAPFLAG, NSUB[t] + (eq ? 0 : 1)));
      H[t] = m + PEN[t];
    } else {
      const int i = I - cc, j = Jp + cc;
      const bool valid = (t >= c.tlo) && (t <= c.thi) && i >= 0 && j >= 0 && i <= c.len1 && j <= c.len2 && k <= c.nsteps;
      const int gl_ = (HM && ((HB >> cc) & 1u)) ? c.hgap : c.gap, gu_ = (HM && ((HA >> cc) & 1u)) ? c.hgap : c.gap;
      const int left = hl + ((i == c.len1) ? 0 : gl_);                     // nwalign_endsfree.cpp:128-156 (homo :303-320)
      const int up = hu + ((j == c.len2) ? 0 : gu_);
      const int diag = H[t] + (eq ? c.match : c.mismatch);
      const int m = max(max(left, up), diag);
      int pmove = (up == m) ? 3 : ((left == m) ? 2 : 1);
      int val = m;
      if (i == 0) { val = 0; pmove = (j == 0) ? 0 : 2; }                   // top row: ends-free, p=2  (:97-101)
      else if (j == 0) { val = 0; pmove = 0; }                             // left column: p=3, no raw base consumed
      int np = (pmove == 3) ? nu : ((pmove == 2) ? nl : NSUB[t]);
      if (pmove == 0) np = (i > 0) ? GAPFLAG : 0;
      if (pmove == 1 && !eq) np++;
      if (pmove == 2 || pmove == 3) np |= GAPFLAG;
      if (WL) {
        const int b2 = s_b2[min(max(j - 1, -PADL), c.len2 + PADL - 1)];
        const int idx = (pmove == 1 || pmove == 2) ? b2 + (int)((pmove == 1) ? nt1 : nt2) * c.ncol4 : c.ONE_IDX;
        double lp = (pmove == 3) ? lu : ((pmove == 2) ? ll : LAM[t]);
        if (pmove == 0) lp = 1.0;
        LAM[t] = valid ? lp * s_err[idx] : LAM[t];
      }
      H[t] = valid ? val : H[t];
      NSUB[t] = valid ? np : NSUB[t];
    }
  }
}

// bit 2 of a staged base byte = "inside a homopolymer run of length >= 3" (nwalign_endsfree.cpp:230-255).  Writers only touch
// bit 2 and readers of the neighbours only use bits 1:0, so the flags of one sequence can be set concurrently.
__device__ __forceinline__ void homo_flag(uint8_t *seq, int p, int len) {
  const int b = seq[p] & 3;
  int L = 0, R = 0;
  while (L < 2 && p - L - 1 >= 0 && (seq[p - L - 1] & 3) == b) L++;
  while (R < 2 && p + R + 1 < len && (seq[p + R + 1] & 3) == b) R++;
  if (L + R >= 2) seq[p] |= 4;
}

// WL = carry lambda (the exact kernel).  WL = false is the bound pass of the two-phase scheme (DESIGN.md 9.3): scores and
// substitution counts only; pairs that provably fail the store rule are dropped, the rest are listed for the exact kernel.
template <int G, int ND, bool WL, bool HM>
__global__ void __launch_bounds__(128) k_nwfwd(FwdArgs a) {
  constexpr int NSL = ND / 2;             // cells per lane per step
  constexpr int PPW = 32 / G;             // pairs per warp
  static_assert(ND % 2 == 0 && NSL <= 16, "base windows are one 32-bit register each");
  extern __shared__ uint32_t smem[];
  const AlnParams &P = a.P;
  const int ncol = P.ncol;
  double *s_err = (double *)smem;                       // 16*ncol + 1 (last = 1.0)
  uint8_t *s_cen_shared = (uint8_t *)(s_err + 16 * ncol + 2);  // centre bases (LOOP: one centre per launch)
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gid = lane / G, gl = lane % G;
  // per pair: raw bases [seq_bytes] then b2[pos] = nt*ncol + qual as u16 with PAD zeroed entries on both sides
  constexpr int PAD = 64;
  uint8_t *s_grp = s_cen_shared + a.seq_bytes + (size_t)(wid * PPW + gid) * (4 * a.seq_bytes + 4 * PAD);
  uint8_t *s_cen_own = s_grp;                            // FINAL: each pair has its own centre
  uint8_t *s_raw = s_grp + a.seq_bytes;
  uint16_t *s_b2 = (uint16_t *)(s_raw + a.seq_bytes) + PAD;
  const bool final_mode = a.mode == 1;
  const uint8_t *s_cen = final_mode ? s_cen_own : s_cen_shared;
  constexpr int GAPFLAG = 1 << 30;                       // carried in the nsubs word: the path contains a gap move
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gid * G));
  (void)gmask;

  const unsigned long long njobs = *a.njobs_ptr;
  if ((unsigned long long)blockIdx.x * nwarps * PPW >= njobs) return;      // whole block idle (grid is sized for the worst case)
  const int len1_shared = final_mode ? 0 : a.in.len[a.centre_idx];
  for (int x = threadIdx.x; x < 16 * ncol; x += blockDim.x) s_err[x] = a.st.err[x];
  if (threadIdx.x == 0) s_err[16 * ncol] = 1.0;
  if (!final_mode) {
    const uint32_t *crow = a.in.seq2 + (size_t)a.centre_idx * a.in.SW;
    for (int p = threadIdx.x; p < len1_shared; p += blockDim.x) s_cen_shared[p] = (uint8_t)((crow[p >> 4] >> (2 * (p & 15))) & 3u);
    if (HM) {
      __syncthreads();
      for (int p = threadIdx.x; p < len1_shared; p += blockDim.x) homo_flag(s_cen_shared, p, len1_shared);
    }
  }
  __syncthreads();
  const int ONE_IDX = 16 * ncol, ncol4 = 4 * ncol;
  const int SENT = P.sentinel, match = P.match, mismatch = P.mismatch, gap = P.gap;
  int errflag = 0;
  long long cells_lane = 0;

  for (unsigned long long base = (unsigned long long)(blockIdx.x * nwarps + wid) * PPW; base < njobs;
       base += (unsigned long long)gridDim.x * nwarps * PPW) {
    const unsigned long long jb = base + gid;
    bool act = jb < njobs;
    const uint32_t r = act ? (a.jobs ? a.jobs[jb] : (uint32_t)jb * (uint32_t)a.job_mul + (uint32_t)a.job_add) : 0;
    uint32_t c = a.centre_idx, cluster = 0;
    if (final_mode && act) { cluster = a.st.cluster_of[r]; c = a.st.cl_center[cluster]; }
    const int len1 = final_mode ? (act ? (int)a.in.len[c] : 16) : len1_shared;
    const int len2 = act ? a.in.len[r] : len1;     // idle groups run a benign geometry (their lanes still execute)
    if (final_mode && act) {
      const uint32_t *crow = a.in.seq2 + (size_t)c * a.in.SW;
      for (int p = gl; p < len1; p += G) s_cen_own[p] = (uint8_t)((crow[p >> 4] >> (2 * (p & 15))) & 3u);
    }
    if (HM && final_mode) {
      __syncwarp();
      if (act) for (int p = gl; p < len1; p += G) homo_flag(s_cen_own, p, len1);
    }
    // ---- stage raw bases + qualities (group-cooperative) ----
    if (act) {
      const uint32_t *rrow = a.in.seq2 + (size_t)r * a.in.SW;
      const uint8_t *qrow = a.in.qual + (size_t)r * a.in.QS;
      for (int p = gl; p < len2; p += G) {
        const uint32_t b = (rrow[p >> 4] >> (2 * (p & 15))) & 3u;
        s_raw[p] = (uint8_t)b;
        int q = P.use_quals ? qrow[p] : 0;
        if (q > ncol - 1) { errflag = ERR_QUAL; q = ncol - 1; }             // pval.cpp:169-171
        s_b2[p] = (uint16_t)(b * ncol + q);
      }
      for (int p = gl; p < PAD; p += G) { s_b2[-1 - p] = 0; s_b2[len2 + p] = 0; }
    } else {   // idle group: its lanes still execute the DP; keep their table indices in range
      for (int p = gl; p < a.seq_bytes + 2 * PAD; p += G) s_b2[p - PAD] = 0;
    }
    __syncwarp();
    if (HM) {
      if (act) for (int p = gl; p < len2; p += G) homo_flag(s_raw, p, len2);
      __syncwarp();
    }
    // ---- band geometry (nwalign_endsfree.cpp:101-111) ----
    int lband, rband;
    if (len2 > len1) { lband = P.band; rband = P.band + len2 - len1; }
    else if (len1 > len2) { lband = P.band + len1 - len2; rband = P.band; }
    else { lband = P.band; rband = P.band; }
    const int lb = min(lband, len1), rb = min(rband, len2);
    const int LB = (lb + 1) & ~1;
    const int lo = LB - lb, hi = LB + rb;          // in-band dd range [lo, hi]
    if (act && (P.band < 0 || hi >= G * ND)) {     // does not fit this instantiation: hand over to k_align
      if (gl == 0) { unsigned long long s = atomicAdd(a.fb_count, 1ull); a.fb_list[s] = r; }
      act = false;
    }
    const int tlo = lo - gl * ND, thi = hi - gl * ND;   // in-band local t range for this lane
    const int D = gl * ND - LB;                          // delta of local t = 0 (even)
    const int nsteps = act ? len1 + len2 : 0;
    int maxsteps = nsteps;
#pragma unroll
    for (int o = 16; o; o >>= 1) maxsteps = max(maxsteps, __shfl_xor_sync(0xffffffffu, maxsteps, o));

    int H[ND], NSUB[ND];
    double LAM[ND];
#pragma unroll
    for (int t = 0; t < ND; t++) { H[t] = SENT; NSUB[t] = 0; LAM[t] = 1.0; }
    // windows for step k = 0: I = -D/2, J = D/2 ; slot c: s1[I-1-c], s2[J-1+c]
    int I = -(D / 2), J = D / 2;      // D even; exact
    uint32_t A = 0, B = 0, HA = 0, HB = 0;
#pragma unroll
    for (int cc = 0; cc < NSL; cc++) {
      const int i1 = I - 1 - cc, j1 = J - 1 + cc;
      const uint32_t b1 = (i1 >= 0 && i1 < len1) ? s_cen[i1] : 0u;
      const uint32_t b2 = (act && j1 >= 0 && j1 < len2) ? s_raw[j1] : 0u;
      A |= (b1 & 3u) << (2 * cc); B |= (b2 & 3u) << (2 * cc);
      if (HM) { HA |= (b1 >> 2) << cc; HB |= (b2 >> 2) << cc; }
    }

    // Interior steps (no boundary cell, no free end gap, every pair still running) take a branch-free path;
    // out-of-band slots are kept far below any real score by an additive penalty instead of a mask.
    int kf_lo = act ? max(lb, rb) + 2 : 0, kf_hi = act ? min(2 * len1 - lb, 2 * len2 - rb) - 1 : 0x3fffffff;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      kf_lo = max(kf_lo, __shfl_xor_sync(0xffffffffu, kf_lo, o));
      kf_hi = min(kf_hi, __shfl_xor_sync(0xffffffffu, kf_hi, o));
    }
    if (!a.fast_ok) kf_hi = -1;
    constexpr int BIGPEN = 1 << 20;
    int PEN[ND];
#pragma unroll
    for (int t = 0; t < ND; t++) {
      PEN[t] = (t >= tlo && t <= thi) ? 0 : -BIGPEN;
      PEN[t] = __shfl_sync(0xffffffffu, PEN[t], lane);   // opaque to ptxas: stays an addend (one IADD per cell), not a predicate + select
    }

    // ---- main loop in three phases: checked prologue, branch-free interior, checked epilogue ----
    auto advB = [&]() {            // even -> odd: raw window moves one base (J -> J+1)
      uint32_t nbB = __shfl_down_sync(0xffffffffu, B, 1, G);
      uint32_t newb = nbB & 3u, newh = 0;
      if (HM) newh = __shfl_down_sync(0xffffffffu, HB, 1, G) & 1u;
      if (gl == G - 1) { const int jn = J + NSL - 1; const uint32_t v = (act && jn >= 0 && jn < len2) ? s_raw[jn] : 0u; newb = v & 3u; newh = v >> 2; }
      B = (B >> 2) | (newb << (2 * (NSL - 1)));
      if (HM) HB = (HB >> 1) | (newh << (NSL - 1));
    };
    auto advA = [&]() {            // odd -> even: centre window moves one base (I -> I+1), J -> J+1 completes
      uint32_t nbA = __shfl_up_sync(0xffffffffu, A, 1, G);
      uint32_t newa = (nbA >> (2 * (NSL - 1))) & 3u, newh = 0;
      if (HM) newh = (__shfl_up_sync(0xffffffffu, HA, 1, G) >> (NSL - 1)) & 1u;
      if (gl == 0) { const uint32_t v = (I >= 0 && I < len1) ? s_cen[I] : 0u; newa = v & 3u; newh = v >> 2; }
      A = ((A << 2) | newa) & (NSL == 16 ? 0xffffffffu : ((1u << (2 * NSL)) - 1u));
      if (HM) HA = ((HA << 1) | newh) & ((1u << NSL) - 1u);
      I += 1; J += 1;
    };
    const StepCtx cx{gl, len1, len2, tlo, thi, nsteps, SENT, match, mismatch, gap, P.hgap, ncol4, ONE_IDX, (int)((const unsigned char *)s_b2 - (const unsigned char *)smem)};
    int kk = 0;
    const int kfa = (kf_lo + 1) & ~1;                       // first even step index inside the interior range
    for (; kk < kfa && kk <= maxsteps; kk += 2) {
      nw_step<G, ND, WL, HM, 0, false>(H, NSUB, LAM, PEN, A, B, HA, HB, I, J, kk, cx); advB();
      nw_step<G, ND, WL, HM, 1, false>(H, NSUB, LAM, PEN, A, B, HA, HB, I, J, kk + 1, cx); advA();
    }
    for (; kk + 1 <= kf_hi && kk <= maxsteps; kk += 2) {
      nw_step<G, ND, WL, HM, 0, true>(H, NSUB, LAM, PEN, A, B, HA, HB, I, J, kk, cx); advB();
      nw_step<G, ND, WL, HM, 1, true>(H, NSUB, LAM, PEN, A, B, HA, HB, I, J, kk + 1, cx); advA();
    }
    for (; kk <= maxsteps; kk += 2) {
      nw_step<G, ND, WL, HM, 0, false>(H, NSUB, LAM, PEN, A, B, HA, HB, I, J, kk, cx); advB();
      nw_step<G, ND, WL, HM, 1, false>(H, NSUB, LAM, PEN, A, B, HA, HB, I, J, kk + 1, cx); advA();
    }
    // ---- result: cell (len1, len2) on dd = len2 - len1 + LB ----
    const int ddf = len2 - len1 + LB;
    const int tf = ddf - gl * ND;
    double lam = 0.0; int ns = 0;
#pragma unroll
    for (int t = 0; t < ND; t++) if (t == tf) { lam = LAM[t]; ns = NSUB[t]; }
    const bool owner = act && tf >= 0 && tf < ND;
    if (owner && !a.no_cells) cells_lane += band_cells2(len1, len2, lband, rband);
    if (final_mode) {
      // FinalSubsParallel (Rmain.cpp:179-236): nsubs of the final alignment; pairs whose optimal path is the pure
      // diagonal get the trivial (gapless) column list, the rest go to the traceback kernel.
      const bool pure = owner && !(ns & GAPFLAG);
      const bool gapped = owner && (ns & GAPFLAG);
      if (owner) a.st.nsubs_final[r] = (uint32_t)(ns & (GAPFLAG - 1));
      const unsigned mp = __ballot_sync(0xffffffffu, pure), mg = __ballot_sync(0xffffffffu, gapped);
      unsigned long long bp = 0, bg = 0;
      if (lane == 0) { if (mp) bp = atomicAdd(a.gl_count, (unsigned long long)__popc(mp)); if (mg) bg = atomicAdd(a.nw_count, (unsigned long long)__popc(mg)); }
      bp = __shfl_sync(0xffffffffu, bp, 0); bg = __shfl_sync(0xffffffffu, bg, 0);
      if (pure) a.gl_out[bp + __popc(mp & ((1u << lane) - 1u))] = r;
      if (gapped) a.nw_out[bg + __popc(mg & ((1u << lane) - 1u))] = r;
    } else if (!WL) {
      // bound pass: lambda <= S_r * rho_r^nsubs for ANY alignment with nsubs substitutions (S_r = product of the raw's
      // self-transition factors, rho_r = largest substitution/self ratio at the raw's own (base, quality) positions), so
      // bound * total_reads <= E_minmax proves the comparison fails cluster.cpp:192 and can never matter again.
      bool survive = false;
      if (owner) {
        const double bound = a.raw_S[r] * pow(a.raw_rho[r], (double)(ns & (GAPFLAG - 1))) * (double)a.total_reads * (1.0 + 1e-9);
        survive = !(bound <= a.st.E_minmax[r]) || bound < 1e-280;     // near underflow the fp product is not a safe bound: keep
      }
      if (owner && a.ns_out) a.ns_out[r] = (uint32_t)(ns & (GAPFLAG - 1)) | (survive ? 0x80000000u : 0u);
      const unsigned ms = __ballot_sync(0xffffffffu, survive);
      unsigned long long bs = 0;
      if (lane == 0 && ms) bs = atomicAdd(a.surv_count, (unsigned long long)__popc(ms));
      bs = __shfl_sync(0xffffffffu, bs, 0);
      if (survive) a.surv_list[bs + __popc(ms & ((1u << lane) - 1u))] = r;
    } else if (owner) {
      ns &= (GAPFLAG - 1);
      if (lam < 0 || lam > 1 || lam != lam) errflag = ERR_LAMBDA;                 // pval.cpp:195
      const double emm = a.st.E_minmax[r];                                          // cluster.cpp:192-200
      if (lam * (double)a.total_reads > emm) {
        const double ec = lam * (double)a.centre_reads;
        if (ec > emm) a.st.E_minmax[r] = ec;
        {
          const unsigned long long slot = a.cluster_i == 0 ? (unsigned long long)r : atomicAdd(&a.st.ctr[CTR_CS_COUNT], 1ull);
          if (slot < a.st.cs_cap) {
            a.st.cs_index[slot] = r; a.st.cs_i[slot] = a.cluster_i; a.st.cs_lambda[slot] = lam; a.st.cs_ham[slot] = (uint32_t)ns;
          }
          if (a.cluster_i == 0 || r == c) { a.st.comp_lambda[r] = lam; a.st.comp_ham[r] = (uint32_t)ns; }
        }
      }
    }
    __syncwarp();
  }
  if (errflag) atomicMax(&a.st.ctr[CTR_ERR], (unsigned long long)errflag);
#pragma unroll
  for (int o = 16; o; o >>= 1) cells_lane += __shfl_xor_sync(0xffffffffu, cells_lane, o);
  if (lane == 0 && cells_lane) atomicAdd(&a.st.ctr[CTR_CELLS], (unsigned long long)cells_lane);
}

template <int G, int ND, bool WL, bool HM> static void launch_one(const FwdArgs &a, int grid, size_t smem, cudaStream_t s) {
  static bool attr_set = false;
  if (!attr_set) { cudaFuncSetAttribute(k_nwfwd<G, ND, WL, HM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024); attr_set = true; }
  k_nwfwd<G, ND, WL, HM><<<grid, 128, smem, s>>>(a);
}
template <int G, int ND> static void launch_wl(const FwdArgs &a, bool bound_only, int grid, size_t smem, cudaStream_t s) {
  if (a.P.homo) launch_one<G, ND, true, true>(a, grid, smem, s);        // homopolymer costs: exact kernel only (no bound pass)
  else if (bound_only) launch_one<G, ND, false, false>(a, grid, smem, s);
  else launch_one<G, ND, true, false>(a, grid, smem, s);
}

// Picks the instantiation: smallest G*ND >= needed band slots, preferring few lanes per pair for
// large batches (throughput) and many lanes for small batches (latency).
bool launch_nwfwd(const FwdArgs &a, int slots_needed, unsigned long long njobs_upper, unsigned long long njobs_hint, int num_sms, cudaStream_t s,
                  bool bound_only) {
  if (a.P.homo && bound_only) return false;
  int G, ND;
  const bool big = njobs_hint > (unsigned long long)num_sms * 512;
  if (slots_needed <= 40) { G = big ? 4 : 8; ND = big ? 10 : 6; }
  else if (slots_needed <= 48) { G = 8; ND = 6; }
  else if (slots_needed <= 64) { G = 8; ND = 8; }
  else if (slots_needed <= 128) { G = 16; ND = 8; }
  else if (slots_needed <= 256) { G = 32; ND = 8; }
  else return false;
  if (G * ND < slots_needed) return false;
  const int PPW = 32 / G;
  const size_t smem = (size_t)(16 * a.P.ncol + 2) * 8 + a.seq_bytes + (size_t)4 * PPW * (4 * a.seq_bytes + 4 * 64);
  if (smem > 160 * 1024) return false;
  unsigned long long warps = (njobs_upper + PPW - 1) / PPW;
  int grid = (int)std::min<unsigned long long>((warps + 3) / 4, (unsigned long long)num_sms * 16);
  if (grid < 1) grid = 1;
  count_launch(1);
  if (G == 4 && ND == 10) launch_wl<4, 10>(a, bound_only, grid, smem, s);
  else if (G == 8 && ND == 6) launch_wl<8, 6>(a, bound_only, grid, smem, s);
  else if (G == 8 && ND == 8) launch_wl<8, 8>(a, bound_only, grid, smem, s);
  else if (G == 16 && ND == 8) launch_wl<16, 8>(a, bound_only, grid, smem, s);
  else if (G == 32 && ND == 8) launch_wl<32, 8>(a, bound_only, grid, smem, s);
  else return false;
  return true;
}

}  // namespace dd2
