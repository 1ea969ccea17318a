// C_eval_pair (evaluate.cpp:73-120) on the 2-bit move string of nw_warp, shared by mergePairs' kernel (dd_merge.cu) and
// collapseNoMismatch's alignment kernel (dd_collapse.cu).  Product code.
#pragma once
#include "dd_nw_warp.cuh"
#include "dd_bimera.cuh"

namespace dd2 {

struct EvalPair { int match, mismatch, indel, leadQ, trailP; };

// One warp, warp-uniform result.  s1 / s2: the unpacked rows that nw_warp aligned; opw / nops: its moves (reverse order).
// Writes the column masks, forward order: mQ = gap in s1's row, mP = gap in s2's row, mE = equal bases (nops + 32 bits each).
// The internal part lies between the leading and the trailing end-gap run: start is the first column by which both rows
// have begun, end the last column before both have ended.  leadQ / trailP: s1's leading and s2's trailing gap runs.
__device__ inline EvalPair eval_pair_warp(const uint8_t *s1, const uint8_t *s2, const uint32_t *opw, int nops, uint32_t *mQ,
                                         uint32_t *mP, uint32_t *mE) {
  const int lane = lane_id();
  int i0b = 0, i1b = 0, neq = 0, ngap = 0;
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
    neq += __popc(be); ngap += __popc(bq) + __popc(bp);
    i0b += __popc(b0); i1b += __popc(b1);
  }
  if (lane == 0) { mQ[nch] = 0; mP[nch] = 0; mE[nch] = 0; }
  __syncwarp();
  const int n = nops;
  const int leadQ = run_fwd(mQ, 0, n), leadP = run_fwd(mP, 0, n);
  const int trailQ = run_bwd(mQ, n - 1), trailP = run_bwd(mP, n - 1);
  const int start = leadQ ? leadQ : leadP, end = n - 1 - (trailQ ? trailQ : trailP);
  EvalPair r{0, 0, 0, leadQ, trailP};
  if (start <= end) {
    r.match = neq;                                           // equal columns never lie in an end-gap run
    r.indel = ngap - (leadQ ? leadQ : leadP) - (trailQ ? trailQ : trailP);
    r.mismatch = (end - start + 1) - r.match - r.indel;
  }
  return r;
}

}  // namespace dd2
