// Warp-per-pair banded ends-free Needleman-Wunsch with traceback (device functions shared by dd_kernels.cu and
// dd_bimera.cu).  Product code.
#pragma once
#include "dd_common.h"

namespace dd2 {

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31u; }
__device__ __forceinline__ unsigned lanemask_lt() { return (1u << lane_id()) - 1u; }

__device__ __forceinline__ unsigned base_at(const uint32_t *row, int p) { return (row[p >> 4] >> (2 * (p & 15))) & 3u; }


// =====================================================================================
// Banded ends-free Needleman-Wunsch, one warp per pair, anti-diagonal wavefront.
//   s1 = centre (rows i), s2 = raw (columns j); recurrence, tie order (up > left > diag),
//   free end gaps on the last row/column and band geometry follow nwalign_endsfree.cpp:101-160
//   (and :230-330 for homopolymer gap costs).  State: one live score per diagonal
//   (delta = j - i) in shared memory; a step k = i + j updates the diagonals with the
//   parity of k from their neighbours (k-1) and themselves (k-2).  2-bit move codes are
//   written per step with two warp ballots.
// =====================================================================================
struct BandGeom { int lb, rb, W, nchunk; };

__device__ __forceinline__ BandGeom band_geom(int len1, int len2, int band) {
  int lband, rband;
  if (band < 0) { lband = len1; rband = len2; }
  else if (len2 > len1) { lband = band; rband = band + len2 - len1; }
  else if (len1 > len2) { lband = band + len1 - len2; rband = band; }
  else { lband = band; rband = band; }
  BandGeom g;
  g.lb = min(lband, len1);
  g.rb = min(rband, len2);
  g.W = g.lb + g.rb + 1;
  g.nchunk = (((g.W + 1) >> 1) + 31) >> 5;
  return g;
}
__device__ __forceinline__ int step_dlo(int k, int len1, const BandGeom &g) {
  // max(-lb, -k, k - 2*len1), written as a negated min of non-negated terms: ptxas for sm_90a fuses the max form into one
  // VIMNMX3 that drops the negation of -k (dlo = k at the last step on an H100, so the traceback reads outside the move rows)
  int dlo = -min(min(g.lb, k), 2 * len1 - k);
  if ((dlo - k) & 1) dlo++;
  return dlo;
}

// s1/s2: bytes, bits 1:0 = base, bit 2 = "inside a homopolymer run >= 3".  H: W+2 ints.
// ptr: 2*nchunk words per step, (len1+len2+1) steps.  Returns number of ops; ops (1 diag, 2 gap in
// centre row, 3 gap in raw row) are packed 2 bits each into opw in traceback (reverse) order.
// GLOBAL: nwalign() of nwalign_endsfree.cpp:403-537 (endsfree=FALSE): row 0 and column 0 hold cumulative gap penalties
// (:417-427) and the last row and column pay for their gaps.  With a band, the reference overwrites (lband+1, 0) and
// (0, rband+1) with -9999 (:446-447); those are the cells of diagonals -lb-1 and rb+1, which keep the sentinel here.
// Homopolymer costs do not apply (evaluate.cpp:49-52).
template <bool GLOBAL = false>
__device__ inline int nw_warp(const uint8_t *s1, int len1, const uint8_t *s2, int len2, const AlnParams &P, int *H,
                       uint32_t *ptr, uint32_t *opw, unsigned long long *cells, int *err) {
  const int lane = lane_id();
  const BandGeom g = band_geom(len1, len2, P.band);
  const int SENT = P.sentinel;
  for (int x = lane; x < g.W + 2; x += 32) H[x] = (x == g.lb + 1) ? 0 : SENT;   // cell (0,0) = 0 on diagonal 0
  __syncwarp();
  const int nsteps = len1 + len2;
  unsigned long long ncell_tot = 0;
  for (int k = 1; k <= nsteps; k++) {
    const int dlo = step_dlo(k, len1, g);
    const int dhi = min(min(g.rb, k), 2 * len2 - k);
    const int ncell = dhi >= dlo ? ((dhi - dlo) >> 1) + 1 : 0;
    uint32_t *row = ptr + (size_t)k * 2 * g.nchunk;
    for (int m = 0; m * 32 < ncell; m++) {
      const int cidx = m * 32 + lane;
      const bool active = cidx < ncell;
      int p = 0;
      if (active) {
        const int dl = dlo + 2 * cidx;
        const int i = (k - dl) >> 1, j = (k + dl) >> 1;
        int *h = H + dl + g.lb + 1;
        int val;
        if (i == 0) { val = GLOBAL ? j * P.gap : 0; p = 2; }     // nwalign_endsfree.cpp:97-101
        else if (j == 0) { val = GLOBAL ? i * P.gap : 0; p = 3; } // :91-95
        else {
          const int c1 = s1[i - 1], c2 = s2[j - 1];
          int left, up, diag;
          if (!GLOBAL && i == len1) left = h[-1];                        // :130-137 (homo :303-311)
          else left = h[-1] + ((!GLOBAL && P.homo && (c2 & 4)) ? P.hgap : P.gap);
          if (!GLOBAL && j == len2) up = h[1];                           // :139-144 (homo :313-320)
          else up = h[1] + ((!GLOBAL && P.homo && (c1 & 4)) ? P.hgap : P.gap);
          diag = h[0] + (((c1 ^ c2) & 3) ? P.mismatch : P.match);
          if (up >= diag && up >= left) { val = up; p = 3; }             // :147-156
          else if (left >= diag) { val = left; p = 2; }
          else { val = diag; p = 1; }
          ncell_tot++;
        }
        h[0] = val;
      }
      const unsigned b0 = __ballot_sync(0xffffffffu, p & 1), b1 = __ballot_sync(0xffffffffu, p & 2);
      if (lane == 0) { row[2 * m] = b0; row[2 * m + 1] = b1; }
    }
    __syncwarp();
  }
  // ---- traceback (warp-uniform), nwalign_endsfree.cpp:166-190 ----
  int i = len1, j = len2, nops = 0;
  uint32_t acc = 0;
  while (i > 0 || j > 0) {
    int p;
    if (i == 0) p = 2;
    else if (j == 0) p = 3;
    else {
      const int k = i + j, dl = j - i;
      const int cidx = (dl - step_dlo(k, len1, g)) >> 1;
      const uint32_t *row = ptr + (size_t)k * 2 * g.nchunk + 2 * (cidx >> 5);
      const unsigned bit = cidx & 31;
      p = ((row[0] >> bit) & 1u) | (((row[1] >> bit) & 1u) << 1);
    }
    if (p == 1) { i--; j--; }
    else if (p == 2) { j--; }
    else if (p == 3) { i--; }
    else { *err = ERR_TRACE; break; }
    acc |= (uint32_t)p << (2 * (nops & 15));
    if ((nops & 15) == 15) { if (lane == 0) opw[nops >> 4] = acc; acc = 0; }
    nops++;
  }
  if ((nops & 15) && lane == 0) opw[nops >> 4] = acc;
  __syncwarp();
  if (cells) *cells += ncell_tot;         // per-lane running total, reduced once per warp by the caller
  return nops;
}

// Unpack a 2-bit row into bytes; bit 2 flags "inside a homopolymer run of length >= 3"
// (nwalign_endsfree.cpp:230-255).  Flag writes only touch bit 2, concurrent readers only use bits 1:0.
__device__ inline void unpack_row(const uint32_t *grow, int len, uint8_t *dst, bool homo) {
  const int lane = lane_id();
  for (int p = lane; p < len; p += 32) dst[p] = (uint8_t)base_at(grow, p);
  __syncwarp();
  if (homo) {
    for (int p = lane; p < len; p += 32) {
      const int b = dst[p] & 3;
      int L = 0, R = 0;
      while (L < 2 && p - L - 1 >= 0 && (dst[p - L - 1] & 3) == b) L++;
      while (R < 2 && p + R + 1 < len && (dst[p + R + 1] & 3) == b) R++;
      if (L + R >= 2) dst[p] |= 4;
    }
    __syncwarp();
  }
}

}  // namespace dd2
