// Read filtering on the H100 (include/dada2b_filter.h).  Product code.
//
// Replaces stages 1-12 of fastqFilter / fastqPairedFilter (R/filter.R:613-730, :878-1141) for every chunk of a file, plus
// C_matchRef / C_matrixEE (src/filter.cpp) and seqComplexity (R/filter.R:1248-1275).  Byte work, but not bandwidth-bound:
// measured on an H100 the kernels reach ~8 % of the HBM roofline for the bytes they move; the per-read warp work
// (sequential EE adds, hash probes) bounds them (DESIGN.md 18).
// Launch sequence of one call (dada2b_filter and the stage hook run the same one):
//   k_flt_alpha   one thread per base: letters must be upper-case IUPAC, qualities 0..93; the host reads its flags and
//                 stops the call before any kernel indexes the EE table with a quality
//   k_flt_stage   one warp per read (pair): orientation, the trim window of stages 2-7 (the truncQ cut from ballots and
//                 ffs), then one pass over the window: the non-ACGT count (popc of ballots), min(q), the expected errors
//                 (sequential fp64 adds of a table computed on the host), the phiX hits of both strands (rolling 2-bit
//                 keys built from ballots, a hash table of the genome's k-mers, the greedy non-overlapping walk over the
//                 hit bitmask) and the 2-mer histogram of the complexity
//   k_flt_decide  one thread per read (pair): thresholds of stages 8-12 -> reason code, survivor counts and lengths
//   scans         exclusive u64 scans of the survivor counts / lengths, split by orientation (output order per chunk:
//                 reads kept as they are first, then the flipped ones)
//   k_flt_emit    one warp per survivor: the trimmed window, reverse-complemented where flipped, at its output offset
#include "../../include/dada2b_filter.h"
#include "dd_flt.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace dd2 {

constexpr int FLT_WARPS = 8;                    // warps per block of the per-read kernels

__device__ __forceinline__ int flt_code(char c) {            // A C G T -> 0..3, anything else 4
  switch (c) { case 'A': return 0; case 'C': return 1; case 'G': return 2; case 'T': return 3; default: return 4; }
}

// Open-addressing table of k-mer keys (2 bits per base, base j at bits 2j..2j+1), entry = strand mask << 32 | key.
__device__ __forceinline__ unsigned flt_find(const unsigned long long *t, int lg, unsigned key) {
  const unsigned mask = (1u << lg) - 1u;
  unsigned h = (key * 0x9E3779B1u) >> (32 - lg);
  for (;;) {
    const unsigned long long e = __ldg(t + h);
    if (!(e >> 32)) return 0u;
    if ((unsigned)e == key) return (unsigned)(e >> 32);
    h = (h + 1u) & mask;
  }
}
static unsigned host_hash(unsigned key, int lg) { return (key * 0x9E3779B1u) >> (32 - lg); }

__device__ __forceinline__ unsigned flt_spread(unsigned x) {  // bit j -> bit 2j (16 bits)
  x = (x | (x << 8)) & 0x00FF00FFu; x = (x | (x << 4)) & 0x0F0F0F0Fu;
  x = (x | (x << 2)) & 0x33333333u; x = (x | (x << 1)) & 0x55555555u;
  return x;
}

// Greedy left-to-right hit count of C_matchRef (src/filter.cpp:24-29): after a hit at j the next window tested is
// j + skip (word_size + 1 when non-overlapping, else 1).  bits: hits of windows b .. b+31; uniform over the warp.
__device__ __forceinline__ void flt_walk(unsigned bits, int b, int skip, int &next, int &cnt) {
  while (bits) {
    const int k = __ffs((int)bits) - 1;
    bits &= bits - 1u;
    if (b + k >= next) { cnt++; next = b + k + skip; }
  }
}

struct FltPass {                       // what one pass over a window computes
  const double *ee_tab;                // shared-memory copy of the EE terms, NULL: no quality statistics
  const unsigned long long *tab; int lg, word, skip;   // k-mer table (NULL: no screen)
  unsigned *hist; int kmer;            // warp's histogram (kmer 0: none)
};
struct FltVals { int n_other, min_q, hf, hr; double ee; };

// One warp, one pass over [s0, e) of v, 32 positions per step.  Codes of positions [b, b + 64) sit in three 64-bit
// masks (low bit, high bit, not-ACGT), so the window starting at lane l is bits l .. l+w-1 of each; positions >= e load
// as not-ACGT, which invalidates every window that does not fit.
__device__ void flt_pass(const FltView &v, int s0, int e, int lane, const FltPass &P, FltVals &r) {
  int n_other = 0, minq = 1 << 30, nf = 0, nr = 0, hf = 0, hr = 0;
  double ee = 0.0;
  const unsigned wmask = P.word >= 32 ? FULL : (1u << P.word) - 1u;
  const unsigned kmask = (1u << P.kmer) - 1u;
  unsigned lo[2], hi[2], inv[2];
  auto load = [&](int p0, int slot) {
    const int p = p0 + lane;
    const bool in = p < e;
    const int c = in ? flt_code(v.base(p)) : 4;
    lo[slot] = __ballot_sync(FULL, c & 1);
    hi[slot] = __ballot_sync(FULL, (c >> 1) & 1);
    inv[slot] = __ballot_sync(FULL, c >> 2);
    if (p0 < e) {
      n_other += __popc(inv[slot] & __ballot_sync(FULL, in));
      if (P.ee_tab) {
        const int q = in ? v.qual(p) : 0;
        if (in) minq = min(minq, q);
        const double t = in ? P.ee_tab[q] : 0.0;
        const int m = min(32, e - p0);
        for (int j = 0; j < m; j++) ee += __shfl_sync(FULL, t, j);     // C_matrixEE: ascending positions, one add at a time
      }
    }
  };
  if (s0 < e) load(s0, 0);
  for (int b = s0; b < e; b += 32) {
    load(b + 32, 1);
    const unsigned long long L = lo[0] | ((unsigned long long)lo[1] << 32), H = hi[0] | ((unsigned long long)hi[1] << 32),
                             I = inv[0] | ((unsigned long long)inv[1] << 32);
    if (P.tab) {
      const unsigned x = (unsigned)(L >> lane) & wmask, y = (unsigned)(H >> lane) & wmask;
      const bool ok = ((unsigned)(I >> lane) & wmask) == 0u;
      const unsigned m = ok ? flt_find(P.tab, P.lg, flt_spread(x) | (flt_spread(y) << 1)) : 0u;
      flt_walk(__ballot_sync(FULL, m & 1u), b, P.skip, nf, hf);
      flt_walk(__ballot_sync(FULL, m & 2u), b, P.skip, nr, hr);
    }
    if (P.kmer && ((unsigned)(I >> lane) & kmask) == 0u) {
      unsigned idx = 0;                                     // lexical order: first base most significant
      for (int j = 0; j < P.kmer; j++) idx = idx * 4u + (unsigned)(((L >> (lane + j)) & 1u) | (((H >> (lane + j)) & 1u) << 1));
      atomicAdd(&P.hist[idx], 1u);
    }
    lo[0] = lo[1]; hi[0] = hi[1]; inv[0] = inv[1];
  }
  for (int o = 16; o; o >>= 1) minq = min(minq, __shfl_xor_sync(FULL, minq, o));
  r.n_other = n_other; r.min_q = minq; r.ee = ee; r.hf = hf; r.hr = hr;
}

// sindex(x) = exp(sum(-y*log(y))), y = x/sum(x) > 0, in lexical k-mer order (R/filter.R:1271-1275).  R adds in long double;
// here the sum is compensated (Neumaier) in fp64.  Resets the histogram.  NaN where no k-mer was counted (R's NA).
__device__ double flt_sindex(unsigned *hist, int kmer, int lane) {
  __syncwarp();
  const int nb = 1 << (2 * kmer);
  unsigned tot = 0;
  for (int x = lane; x < nb; x += 32) tot += hist[x];
  for (int o = 16; o; o >>= 1) tot += __shfl_xor_sync(FULL, tot, o);
  double s = 0.0, c = 0.0;
  for (int x0 = 0; x0 < nb; x0 += 32) {
    const int x = x0 + lane;
    const unsigned cnt = x < nb ? hist[x] : 0u;
    double t = 0.0;
    if (cnt) { const double y = (double)cnt / (double)tot; t = -y * log(y); }
    const unsigned has = __ballot_sync(FULL, cnt != 0u);
    for (int j = 0; j < 32; j++) {
      const double u = __shfl_sync(FULL, t, j);
      if (!((has >> j) & 1u)) continue;
      const double n = s + u;
      c += fabs(s) >= fabs(u) ? (s - n) + u : (u - n) + s;
      s = n;
    }
    if (x < nb) hist[x] = 0u;
  }
  __syncwarp();
  if (!tot) return __longlong_as_double(0x7FF8000000000000LL);
  return exp(s + c);
}

// ---------------------------------------------------------------------------------------------------------------------
struct FltMateOpt {
  int trunc_q, start, trim_right, end, max_len, min_len, max_n, min_q, use_min_q, use_ee, phix, lowc;
  double max_ee, lowc_thr;
};
struct FltReads { const char *seq; const uint8_t *qual; const long long *off; };
struct FltArgs {
  int n, nm;                            // reads (pairs), mates (1 or 2)
  FltReads in[2];
  FltMateOpt o[2];
  const char *primer; int barlen;       // orient.fwd (barlen < 0: off)
  const unsigned long long *tab; int lg, word;
  int calc_phix[2], calc_cplx[2];
  dada2b_filter_stage *st;              // [n][nm]
  unsigned *err;                        // bit 0: a read shorter than orient.fwd; bit 1: NA complexity at rm.lowcomplex
  double ee_tab[94];                    // pow(10, -q/10) from the host's C library, kernel parameters = constant memory
};

__global__ void __launch_bounds__(256) k_flt_alpha(const char *seq, const uint8_t *qual, long long nbytes, unsigned *err) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= nbytes) return;
  bool ok;
  switch (seq[x]) {
    case 'A': case 'C': case 'G': case 'T': case 'R': case 'Y': case 'S': case 'W': case 'K': case 'M': case 'B': case 'D':
    case 'H': case 'V': case 'N': ok = true; break;
    default: ok = false;
  }
  if (!ok) atomicOr(err, 4u);
  if (qual[x] > 93) atomicOr(err, 8u);
}

__device__ bool flt_prefix(const FltView &v, const char *pr, int bl, int lane) {
  for (int j0 = 0; j0 < bl; j0 += 32) {
    const int j = j0 + lane;
    if (__any_sync(FULL, j < bl && v.base(j) != pr[j])) return false;
  }
  return true;
}

// Stages 2-7 of one mate: the trim window [start, end) of the oriented read, or the stage that removed it.
__device__ int flt_trim(const FltView &v, const FltMateOpt &o, int lane, int &s0, int &e) {
  const int L = v.L;
  if (o.max_len >= 0 && L > o.max_len) return 2;
  if (L < o.start) return 3;
  s0 = o.start - 1; e = L;
  if (o.trim_right > 0) {
    if (e - s0 <= o.trim_right) return 4;
    e -= o.trim_right;
  }
  for (int p0 = s0; p0 < e; p0 += 32) {                  // trimTails(k = 1): cut before the first base with q <= truncQ
    const int p = p0 + lane;
    const unsigned b = __ballot_sync(FULL, p < e && v.qual(p) <= o.trunc_q);
    if (b) { e = p0 + __ffs((int)b) - 1; break; }
  }
  if (e == s0) return 5;
  if (o.end >= 0) {
    if (e - s0 < o.end) return 6;
    e = s0 + o.end;
  }
  if (e - s0 < o.min_len) return 7;
  return 0;
}

__global__ void __launch_bounds__(FLT_WARPS * 32) k_flt_stage(FltArgs a) {
  __shared__ double s_ee[94];
  __shared__ unsigned s_hist[FLT_WARPS][16];
  for (int x = threadIdx.x; x < 94; x += blockDim.x) s_ee[x] = a.ee_tab[x];
  for (int x = threadIdx.x; x < FLT_WARPS * 16; x += blockDim.x) s_hist[x / 16][x % 16] = 0u;
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int nw = gridDim.x * FLT_WARPS;
  for (int i = blockIdx.x * FLT_WARPS + wib; i < a.n; i += nw) {
    FltView raw[2];
    for (int m = 0; m < a.nm; m++) {
      const long long o = a.in[m].off[i];
      raw[m] = FltView{a.in[m].seq + o, a.in[m].qual + o, (int)(a.in[m].off[i + 1] - o), false};
    }
    // stage 1, orient.fwd (R/filter.R:649-658, :994-1007)
    int fail = 0, flip = 0;
    if (a.barlen >= 0) {
      bool short_read = false;
      for (int m = 0; m < a.nm; m++) short_read |= raw[m].L < a.barlen;
      if (short_read) {                                   // narrow() beyond the read's end: an error in R
        if (lane == 0) atomicOr(a.err, 1u);
        fail = 1;
      } else if (a.nm == 1) {
        if (!flt_prefix(raw[0], a.primer, a.barlen, lane)) {
          FltView rc = raw[0]; rc.flip = true;
          if (flt_prefix(rc, a.primer, a.barlen, lane)) flip = 1; else fail = 1;
        }
      } else if (!flt_prefix(raw[0], a.primer, a.barlen, lane)) {
        if (flt_prefix(raw[1], a.primer, a.barlen, lane)) flip = 1; else fail = 1;
      }
    }
    for (int m = 0; m < a.nm; m++) {
      FltView v = raw[a.nm == 2 && flip ? 1 - m : m];     // paired: swapped mates; single-end: reverse complement
      if (a.nm == 1) v.flip = flip;
      dada2b_filter_stage r{};
      r.flipped = flip;
      int s0 = 0, e = 0;
      r.trim_fail = fail ? fail : flt_trim(v, a.o[m], lane, s0, e);
      if (!r.trim_fail) {
        r.start = s0; r.end = e;
        FltPass P{s_ee, a.calc_phix[m] ? a.tab : nullptr, a.lg, a.word, a.word + 1, s_hist[wib], a.calc_cplx[m] ? 2 : 0};
        FltVals vals;
        flt_pass(v, s0, e, lane, P, vals);
        r.n_other = vals.n_other; r.min_q = vals.min_q; r.ee = vals.ee; r.hits_fwd = vals.hf; r.hits_rc = vals.hr;
        r.complexity = P.kmer ? flt_sindex(s_hist[wib], 2, lane) : 0.0;
      }
      if (lane == 0) a.st[(size_t)i * a.nm + m] = r;
    }
  }
}

// Stages 8-12 and the survivors.  acc rows of n+1 u64 (last entry 0): 0 kept as is, 1 kept flipped, then per mate m
// 2+2m / 3+2m the lengths of the same reads.
__global__ void __launch_bounds__(256) k_flt_decide(FltArgs a, uint8_t *reason, uint8_t *flags, unsigned long long *acc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t R = (size_t)a.n + 1;
  if (i > a.n) return;
  if (i == a.n) { for (int k = 0; k < 2 + 2 * a.nm; k++) acc[k * R + i] = 0ull; return; }
  int f[2] = {0, 0}, low[2] = {0, 0};                     // low: 0 no, 1 yes, 2 NA
  const dada2b_filter_stage *st = a.st + (size_t)i * a.nm;
  for (int m = 0; m < a.nm; m++) {
    const dada2b_filter_stage &r = st[m];
    const FltMateOpt &o = a.o[m];
    if (r.trim_fail) f[m] = r.trim_fail;
    else if (r.n_other > o.max_n) f[m] = 8;
    else if (o.use_min_q && !(r.min_q > o.min_q)) f[m] = 9;
    else if (o.use_ee && r.ee > o.max_ee) f[m] = 10;
    else if (o.phix && (r.hits_fwd >= 2 || r.hits_rc >= 2)) f[m] = 11;
    else if (o.lowc) low[m] = isnan(r.complexity) ? 2 : (r.complexity < o.lowc_thr ? 1 : 0);
  }
  int why = 0;
  for (int m = 0; m < a.nm; m++) if (f[m] && (!why || f[m] < why)) why = f[m];
  unsigned fl = st[0].flipped ? 4u : 0u;
  if (why) {
    for (int m = 0; m < a.nm; m++) if (f[m] == why) fl |= 1u << m;
  } else {
    const bool any = low[0] == 1 || low[1] == 1;           // is.lowc of both mates or'ed, NA | TRUE == TRUE
    if (any) { why = 12; for (int m = 0; m < a.nm; m++) if (low[m] == 1) fl |= 1u << m; }
    else if (low[0] == 2 || low[1] == 2) { atomicOr(a.err, 2u); why = 12; }
  }
  reason[i] = (uint8_t)why; flags[i] = (uint8_t)fl;
  const bool keep = !why, fp = st[0].flipped != 0;
  acc[0 * R + i] = keep && !fp; acc[1 * R + i] = keep && fp;
  for (int m = 0; m < a.nm; m++) {
    const unsigned long long len = keep ? (unsigned long long)(st[m].end - st[m].start) : 0ull;
    acc[(2 + 2 * m) * R + i] = fp ? 0ull : len; acc[(3 + 2 * m) * R + i] = fp ? len : 0ull;
  }
}

// ---- exclusive scan of u64 (three kernels, in place): the byte offsets of a run exceed 32 bits ----
__global__ void __launch_bounds__(256) k_flt_scan1(unsigned long long *v, unsigned long long *sums, size_t n) {
  __shared__ unsigned long long wtot[8];
  const size_t b0 = (size_t)blockIdx.x * 1024 + threadIdx.x * 4;
  unsigned long long x[4], s = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { x[k] = (b0 + k < n) ? v[b0 + k] : 0ull; s += x[k]; }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) wtot[w] = inc;
  __syncthreads();
  unsigned long long wbase = 0;
  for (int k = 0; k < w; k++) wbase += wtot[k];
  unsigned long long run = wbase + inc - s;
#pragma unroll
  for (int k = 0; k < 4; k++) { if (b0 + k < n) v[b0 + k] = run; run += x[k]; }
  if (threadIdx.x == 255) sums[blockIdx.x] = wbase + inc;
}
__global__ void __launch_bounds__(1024) k_flt_scan2(unsigned long long *sums, size_t nblocks) {
  __shared__ unsigned long long wtot[32];
  __shared__ unsigned long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (size_t c0 = 0; c0 < nblocks; c0 += 1024) {
    const size_t i = c0 + threadIdx.x;
    const unsigned long long x = i < nblocks ? sums[i] : 0ull;
    unsigned long long inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) wtot[w] = inc;
    __syncthreads();
    unsigned long long wbase = 0;
    for (int k = 0; k < w; k++) wbase += wtot[k];
    const unsigned long long c = carry;
    if (i < nblocks) sums[i] = c + wbase + inc - x;
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + wbase + inc;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(256) k_flt_scan3(unsigned long long *v, const unsigned long long *sums, size_t n) {
  const size_t b0 = (size_t)blockIdx.x * 1024 + threadIdx.x * 4;
  const unsigned long long add = sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < 4; k++) if (b0 + k < n) v[b0 + k] += add;
}

// Output position of survivor i of chunk [c0, c1): survivors of earlier chunks, then within the chunk the reads kept as
// they are (input order), then the flipped ones (input order) -- from the exclusive scans A (as is) and B (flipped).
__device__ __forceinline__ unsigned long long flt_place(const unsigned long long *A, const unsigned long long *B, int i, int c0, int c1,
                                                        bool fp) {
  return fp ? A[c1] + B[i] : B[c0] + A[i];
}

struct FltOut { char *seq[2]; uint8_t *qual[2]; long long *off[2]; int32_t *src; };

__global__ void __launch_bounds__(FLT_WARPS * 32) k_flt_emit(FltArgs a, const uint8_t *reason, const unsigned long long *acc, long long chunk_n,
                                                             FltOut out) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * FLT_WARPS;
  const size_t R = (size_t)a.n + 1;
  for (int i = blockIdx.x * FLT_WARPS + (threadIdx.x >> 5); i < a.n; i += nw) {
    if (reason[i]) continue;
    const dada2b_filter_stage *st = a.st + (size_t)i * a.nm;
    const bool fp = st[0].flipped != 0;
    const int c0 = chunk_n > 0 ? (int)((i / chunk_n) * chunk_n) : 0;
    const int c1 = chunk_n > 0 && (long long)c0 + chunk_n < (long long)a.n ? (int)(c0 + chunk_n) : a.n;
    const unsigned long long pos = flt_place(acc, acc + R, i, c0, c1, fp);
    if (lane == 0) out.src[pos] = i;
    for (int m = 0; m < a.nm; m++) {
      const unsigned long long off = flt_place(acc + (2 + 2 * m) * R, acc + (3 + 2 * m) * R, i, c0, c1, fp);
      const int sm = a.nm == 2 && fp ? 1 - m : m;
      const long long o = a.in[sm].off[i];
      const FltView v{a.in[sm].seq + o, a.in[sm].qual + o, (int)(a.in[sm].off[i + 1] - o), a.nm == 1 && fp};
      const int s0 = st[m].start, len = st[m].end - st[m].start;
      flt_copy_window(v, s0, len, out.seq[m] + off, out.qual[m] + off, lane);
      if (lane == 0) out.off[m][pos] = (long long)off;
    }
  }
}

// C_matchRef and seqComplexity on whole sequences (one warp each).
__global__ void __launch_bounds__(FLT_WARPS * 32) k_flt_match(const char *seq, const long long *off, int n, const unsigned long long *tab, int lg,
                                                              int word, int skip, int32_t *hits) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * FLT_WARPS;
  for (int i = blockIdx.x * FLT_WARPS + (threadIdx.x >> 5); i < n; i += nw) {
    const FltView v{seq + off[i], nullptr, (int)(off[i + 1] - off[i]), false};
    FltPass P{nullptr, tab, lg, word, skip, nullptr, 0};
    FltVals r;
    flt_pass(v, 0, v.L, lane, P, r);
    if (lane == 0) hits[i] = r.hf;
  }
}
__global__ void __launch_bounds__(FLT_WARPS * 32) k_flt_cplx(const char *seq, const long long *off, int n, int kmer, double *out) {
  __shared__ unsigned s_hist[FLT_WARPS][256];
  for (int x = threadIdx.x; x < FLT_WARPS * 256; x += blockDim.x) s_hist[x / 256][x % 256] = 0u;
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int nw = gridDim.x * FLT_WARPS;
  for (int i = blockIdx.x * FLT_WARPS + wib; i < n; i += nw) {
    const FltView v{seq + off[i], nullptr, (int)(off[i + 1] - off[i]), false};
    FltPass P{nullptr, nullptr, 4, 16, 17, s_hist[wib], kmer};
    FltVals r;
    flt_pass(v, 0, v.L, lane, P, r);
    const double c = flt_sindex(s_hist[wib], kmer, lane);
    if (lane == 0) out[i] = c;
  }
}

}  // namespace dd2

using namespace dd2;

void dd2::flt_check_reads(const char *seq, const uint8_t *qual, long long nbytes, unsigned *err, cudaStream_t s) {
  k_flt_alpha<<<(unsigned)((nbytes + 255) / 256), 256, 0, s>>>(seq, qual, nbytes, err);
}

void dd2::FltScan::operator()(unsigned long long *v, size_t n) {
  const size_t nb = (n + 1023) / 1024;
  if (sums.n < nb) sums.alloc(nb);
  unsigned long long *sp = sums.p;
  k_flt_scan1<<<(unsigned)nb, 256, 0, s>>>(v, sp, n);
  k_flt_scan2<<<1, 1024, 0, s>>>(sp, nb);
  k_flt_scan3<<<(unsigned)nb, 256, 0, s>>>(v, sp, n);
  launches += 3;
}

namespace {

// The word-mers of the circularised ref (ref + ref[0:w], C_matchRef's phash) and, with both, of its reverse complement
// (isPhiX's rc.phix), as the device's hash table: strand mask 1 = ref, 2 = reverse complement.
std::vector<unsigned long long> build_table(const std::string &ref, int w, bool both, int &lg) {
  if (w < 1 || w > 16) throw BErr{"dada2b: word_size must be 1..16."};
  if ((int)ref.size() < w) throw BErr{"dada2b: the reference is shorter than word_size."};
  if (!is_acgt(ref)) throw BErr{"dada2b: the reference must be A/C/G/T."};
  std::vector<std::pair<unsigned, unsigned>> keys;
  auto add = [&](const std::string &r, unsigned mask) {
    const std::string c = r + r.substr(0, w);
    for (size_t i = 0; i < r.size(); i++) {
      unsigned k = 0;
      for (int j = 0; j < w; j++) {
        const char b = c[i + j];
        k |= (unsigned)(b == 'C' ? 1 : b == 'G' ? 2 : b == 'T' ? 3 : 0) << (2 * j);
      }
      keys.push_back({k, mask});
    }
  };
  add(ref, 1u);
  if (both) {
    std::string rc(ref.rbegin(), ref.rend());
    for (char &c : rc) c = flt_comp(c);
    add(rc, 2u);
  }
  lg = 4;
  while ((size_t(1) << lg) < 2 * keys.size()) lg++;
  std::vector<unsigned long long> t(size_t(1) << lg, 0ull);
  const unsigned mask = (1u << lg) - 1u;
  for (auto &km : keys) {
    unsigned h = host_hash(km.first, lg);
    for (;;) {
      unsigned long long &e = t[h];
      if (!(e >> 32)) { e = ((unsigned long long)km.second << 32) | km.first; break; }
      if ((unsigned)e == km.first) { e |= (unsigned long long)km.second << 32; break; }
      h = (h + 1u) & mask;
    }
  }
  return t;
}

FltMateOpt mate_opt(const dada2b_filter_mate_opts &m, bool paired) {
  if (m.trunc_q < 0 || m.trunc_q > 93) throw BErr{"Encoding for this truncQ value not found."};
  if (m.max_len < -1) throw BErr{"dada2b: max_len must be -1 (Inf) or >= 0."};
  FltMateOpt o{};
  o.trunc_q = m.trunc_q;
  o.start = std::max(1, m.trim_left + 1);                               // R/filter.R:622
  o.trim_right = m.trim_right;
  o.end = m.trunc_len < o.start ? -1 : m.trunc_len - o.start + 1;      // :623-625, NA when truncLen < start
  o.max_len = m.max_len; o.min_len = m.min_len; o.max_n = m.max_n; o.min_q = m.min_q;
  o.use_min_q = m.min_q > m.trunc_q;                                    // :690
  o.use_ee = m.max_ee < INFINITY;                                      // :691 maxEE < Inf
  o.max_ee = m.max_ee;
  o.phix = m.rm_phix != 0;
  o.lowc = paired ? m.rm_lowcomplex != 0.0 : m.rm_lowcomplex > 0.0;    // :703 `> 0`, :1100 used as a logical
  o.lowc_thr = m.rm_lowcomplex;
  return o;
}

// The one launch sequence of dada2b_filter and dada2b_test_filter_stages (hook != NULL: every per-stage value is computed
// -- phiX hits when a genome is given, complexity always -- and the stage records are copied out).
int run_filter(const dada2b_derep_in *fwd, const dada2b_derep_in *rev, const dada2b_filter_opts *opts, int32_t device,
               dada2b_filter_out **out, dada2b_filter_stage *hook, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  dada2b_filter_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!fwd || !opts || (!out && !hook)) throw BErr{"dada2b: NULL argument."};
    if (out) *out = nullptr;
    need_device(device);
    const int nm = rev ? 2 : 1;
    const int n = fwd->nreads;
    if (n < 0 || (rev && rev->nreads < 0)) throw BErr{"dada2b: negative read count."};
    if (rev && rev->nreads != n)
      throw BErr{"Mismatched forward and reverse sequence files: " + std::to_string(n) + ", " + std::to_string(rev->nreads) + "."};
    FltArgs a{};
    a.n = n; a.nm = nm;
    bool need_phix = false;
    for (int m = 0; m < nm; m++) {
      a.o[m] = mate_opt(opts->mate[m], nm == 2);
      a.calc_phix[m] = hook ? opts->phix != nullptr : a.o[m].phix;
      a.calc_cplx[m] = hook ? 1 : a.o[m].lowc;
      need_phix |= a.calc_phix[m] || a.o[m].phix;
    }
    std::string primer;
    a.barlen = -1;
    if (opts->orient_fwd) {
      primer = opts->orient_fwd;
      if (!is_acgt(primer)) throw BErr{"Non-ACGT characters detected in orient.fwd"};
      a.barlen = (int)primer.size();
    }
    if (need_phix && !opts->phix) throw BErr{"dada2b: rm_phix needs the phiX genome (opts->phix)."};
    for (int q = 0; q < 94; q++) a.ee_tab[q] = pow(10.0, -q / 10.0);     // C_matrixEE's terms (src/filter.cpp:44)
    res = (dada2b_filter_out *)calloc(1, sizeof(dada2b_filter_out));
    res->nreads = n; res->paired = nm == 2;
    res->reason = (uint8_t *)malloc(std::max(n, 1)); res->flags = (uint8_t *)malloc(std::max(n, 1));
    if (n == 0) {
      res->src = (int32_t *)malloc(4);
      for (int m = 0; m < nm; m++) {
        res->seq_concat[m] = (char *)malloc(1); res->qual_concat[m] = (uint8_t *)malloc(1);
        res->seq_off[m] = (int64_t *)calloc(1, 8);
      }
      res->ms_total = bnow_ms() - t0;
      if (out) { *out = res; res = nullptr; }
      else { dada2b_filter_free(res); res = nullptr; }
      return 0;
    }
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
    long long h2d = 0, d2h = 0, kbytes = 0, launches = 0;
    BBuf<char> d_seq[2]; BBuf<uint8_t> d_qual[2]; BBuf<long long> d_off[2];
    std::vector<long long> off[2];
    long long nbytes[2] = {0, 0};
    const dada2b_derep_in *ins[2] = {fwd, rev};
    BCK(cudaEventRecord(ev[0], s));
    for (int m = 0; m < nm; m++) {
      nbytes[m] = rebase(n, ins[m]->seq_off, off[m]);
      const long long o0 = ins[m]->seq_off[0];
      d_seq[m].alloc(std::max<long long>(nbytes[m], 1)); d_qual[m].alloc(std::max<long long>(nbytes[m], 1)); d_off[m].alloc((size_t)n + 1);
      BCK(cudaMemcpyAsync(d_seq[m].p, ins[m]->seq_concat + o0, nbytes[m], cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_qual[m].p, ins[m]->qual_concat + o0, nbytes[m], cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_off[m].p, off[m].data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, s));
      h2d += 2 * nbytes[m] + ((long long)n + 1) * 8;
      a.in[m] = FltReads{d_seq[m].p, d_qual[m].p, d_off[m].p};
    }
    BBuf<char> d_primer; BBuf<unsigned long long> d_tab; BBuf<unsigned> d_err;
    if (a.barlen > 0) {
      d_primer.alloc(a.barlen);
      BCK(cudaMemcpyAsync(d_primer.p, primer.data(), a.barlen, cudaMemcpyHostToDevice, s));
      h2d += a.barlen;
      a.primer = d_primer.p;
    }
    std::vector<unsigned long long> tab;
    if (need_phix) {
      tab = build_table(opts->phix, 16, true, a.lg);                  // isPhiX: wordSize 16 on both strands
      d_tab.alloc(tab.size());
      BCK(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, s));
      h2d += (long long)tab.size() * 8;
      a.tab = d_tab.p; a.word = 16;
    }
    d_err.alloc(1);
    BCK(cudaMemsetAsync(d_err.p, 0, 4, s));
    a.err = d_err.p;
    BCK(cudaEventRecord(ev[1], s));
    BBuf<dada2b_filter_stage> d_st; BBuf<uint8_t> d_reason, d_flags; BBuf<unsigned long long> d_acc;
    d_st.alloc((size_t)n * nm); d_reason.alloc(n); d_flags.alloc(n);
    const size_t R = (size_t)n + 1;
    const int K = 2 + 2 * nm;
    d_acc.alloc(R * K);
    a.st = d_st.p;
    for (int m = 0; m < nm; m++) {
      if (nbytes[m]) {
        const char *sp = d_seq[m].p; const uint8_t *qp = d_qual[m].p; unsigned *ep = d_err.p; const long long nb = nbytes[m];
        flt_check_reads(sp, qp, nb, ep, s);
        launches++; kbytes += 2 * nb;
      }
    }
    {                                                       // k_flt_stage indexes the EE table with the qualities: check them first
      unsigned bad = 0;
      BCK(cudaMemcpyAsync(&bad, d_err.p, 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      if (bad & 4u) throw BErr{"dada2b: reads must be upper-case IUPAC letters (A C G T R Y S W K M B D H V N)."};
      if (bad & 8u) throw BErr{"dada2b: quality values must be 0..93."};
    }
    int nsm = 0;
    BCK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    const unsigned wgrid = (unsigned)std::max(1, std::min((n + FLT_WARPS - 1) / FLT_WARPS, nsm * 16));
    uint8_t *reason_p = d_reason.p, *flags_p = d_flags.p;
    unsigned long long *acc_p = d_acc.p;
    k_flt_stage<<<wgrid, FLT_WARPS * 32, 0, s>>>(a);
    k_flt_decide<<<(unsigned)((R + 255) / 256), 256, 0, s>>>(a, reason_p, flags_p, acc_p);
    launches += 2;
    kbytes += (nbytes[0] + nbytes[1]) * 2 + (long long)n * nm * (long long)sizeof(dada2b_filter_stage) * 2 + (long long)R * K * 8 + 2LL * n;
    FltScan scan; scan.s = s;
    for (int k = 0; k < K; k++) scan(acc_p + k * R, R);
    launches += scan.launches; kbytes += (long long)R * K * 8 * 4;
    // totals: reads out and bytes out per mate
    std::vector<unsigned long long> tot((size_t)K);
    for (int k = 0; k < K; k++) BCK(cudaMemcpyAsync(&tot[k], d_acc.p + k * R + n, 8, cudaMemcpyDeviceToHost, s));
    unsigned err = 0;
    BCK(cudaMemcpyAsync(&err, d_err.p, 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    if (err & 1u) throw BErr{"dada2b: a read is shorter than orient.fwd (R's narrow() fails on it)."};
    if (err & 2u) throw BErr{"dada2b: rm.lowcomplex met a read without any A/C/G/T 2-mer (seqComplexity is NA; R stops here)."};
    const long long nout = (long long)(tot[0] + tot[1]);
    res->nout = (int32_t)nout;
    BBuf<char> o_seq[2]; BBuf<uint8_t> o_qual[2]; BBuf<long long> o_off[2]; BBuf<int32_t> o_src;
    FltOut fo{};
    long long obytes[2] = {0, 0};
    o_src.alloc(std::max<long long>(nout, 1)); fo.src = o_src.p;
    for (int m = 0; m < nm; m++) {
      obytes[m] = (long long)(tot[2 + 2 * m] + tot[3 + 2 * m]);
      o_seq[m].alloc(std::max<long long>(obytes[m], 1)); o_qual[m].alloc(std::max<long long>(obytes[m], 1)); o_off[m].alloc((size_t)nout + 1);
      fo.seq[m] = o_seq[m].p; fo.qual[m] = o_qual[m].p; fo.off[m] = o_off[m].p;
    }
    const long long chunk_n = opts->chunk_n;
    k_flt_emit<<<wgrid, FLT_WARPS * 32, 0, s>>>(a, reason_p, acc_p, chunk_n, fo);
    launches++;
    kbytes += (long long)n + (long long)nout * (16 + 4 + 8 * K) + 4 * (obytes[0] + obytes[1]);
    BCK(cudaEventRecord(ev[2], s));
    BCK(cudaMemcpyAsync(res->reason, d_reason.p, n, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->flags, d_flags.p, n, cudaMemcpyDeviceToHost, s));
    res->src = (int32_t *)malloc((size_t)std::max<long long>(nout, 1) * 4);
    BCK(cudaMemcpyAsync(res->src, o_src.p, (size_t)nout * 4, cudaMemcpyDeviceToHost, s));
    d2h += 2LL * n + nout * 4;
    for (int m = 0; m < nm; m++) {
      res->seq_concat[m] = (char *)malloc(std::max<long long>(obytes[m], 1));
      res->qual_concat[m] = (uint8_t *)malloc(std::max<long long>(obytes[m], 1));
      res->seq_off[m] = (int64_t *)malloc(((size_t)nout + 1) * 8);
      BCK(cudaMemcpyAsync(res->seq_concat[m], o_seq[m].p, obytes[m], cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(res->qual_concat[m], o_qual[m].p, obytes[m], cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(res->seq_off[m], o_off[m].p, (size_t)nout * 8, cudaMemcpyDeviceToHost, s));
      d2h += 2 * obytes[m] + nout * 8;
    }
    if (hook) {
      BCK(cudaMemcpyAsync(hook, d_st.p, (size_t)n * sizeof(dada2b_filter_stage), cudaMemcpyDeviceToHost, s));
      d2h += (long long)n * sizeof(dada2b_filter_stage);
    }
    BCK(cudaEventRecord(ev[3], s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    for (int m = 0; m < nm; m++) res->seq_off[m][nout] = obytes[m];
    float ms = 0;
    BCK(cudaEventElapsedTime(&ms, ev[0], ev[1])); res->ms_h2d = ms;
    BCK(cudaEventElapsedTime(&ms, ev[1], ev[2])); res->ms_kernels = ms;
    BCK(cudaEventElapsedTime(&ms, ev[2], ev[3])); res->ms_d2h = ms;
    BCK(cudaEventElapsedTime(&ms, ev[0], ev[3])); res->ms_device = ms;
    res->gpu_launches = launches; res->h2d_bytes = h2d; res->d2h_bytes = d2h; res->kernel_bytes = kbytes;
    res->ms_total = bnow_ms() - t0;
    if (out) { *out = res; res = nullptr; }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (auto &e : ev) if (e) cudaEventDestroy(e);
  if (s) cudaStreamDestroy(s);
  if (res) dada2b_filter_free(res);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

// Whole sequences of one set, uploaded as they are (any letters).
struct SeqUpload {
  BBuf<char> seq; BBuf<long long> off;
  void put(int n, const char *seq_concat, const int64_t *seq_off, cudaStream_t s) {
    std::vector<long long> o;
    const long long nb = rebase(n, seq_off, o);
    seq.alloc(std::max<long long>(nb, 1)); off.alloc((size_t)n + 1);
    BCK(cudaMemcpyAsync(seq.p, seq_concat + seq_off[0], nb, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(off.p, o.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaStreamSynchronize(s));                       // `o` is pageable and goes out of scope
  }
};

}  // namespace

extern "C" {

void dada2b_filter_default_opts(dada2b_filter_opts *o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  for (auto &m : o->mate) {                               // filterAndTrim (R/filter.R:402-406)
    m.trunc_q = 2; m.trunc_len = 0; m.trim_left = 0; m.trim_right = 0; m.max_len = -1; m.min_len = 20; m.max_n = 0; m.min_q = 0;
    m.max_ee = INFINITY; m.rm_phix = 1; m.rm_lowcomplex = 0.0;
  }
  o->orient_fwd = nullptr; o->phix = nullptr; o->chunk_n = 100000;
}

void dada2b_filter_free(dada2b_filter_out *o) {
  if (!o) return;
  free(o->reason); free(o->flags); free(o->src);
  for (int m = 0; m < 2; m++) { free(o->seq_concat[m]); free(o->seq_off[m]); free(o->qual_concat[m]); }
  free(o);
}

int dada2b_filter(const dada2b_derep_in *fwd, const dada2b_derep_in *rev, const dada2b_filter_opts *opts, int32_t device,
                  dada2b_filter_out **out, char errbuf[DADA2B_ERRLEN]) {
  if (!out) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "dada2b: NULL argument."); return 1; }
  return run_filter(fwd, rev, opts, device, out, nullptr, errbuf);
}

int dada2b_test_filter_stages(const dada2b_derep_in *reads, const dada2b_filter_opts *opts, int32_t device, dada2b_filter_stage *out,
                              char errbuf[DADA2B_ERRLEN]) {
  if (!out) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "dada2b: NULL argument."); return 1; }
  return run_filter(reads, nullptr, opts, device, nullptr, out, errbuf);
}

int dada2b_match_ref(int32_t nseq, const char *seq_concat, const int64_t *seq_off, const char *ref, int32_t word_size, int32_t non_overlapping,
                     int32_t device, int32_t *hits, char errbuf[DADA2B_ERRLEN]) {
  cudaStream_t s = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!seq_off || !ref || (nseq > 0 && !hits)) throw BErr{"dada2b: NULL argument."};
    if (nseq < 0) throw BErr{"dada2b: negative sequence count."};
    need_device(device);
    int lg = 4;
    const std::vector<unsigned long long> tab = build_table(ref, word_size, false, lg);
    if (nseq > 0) {
      BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      SeqUpload up; up.put(nseq, seq_concat, seq_off, s);
      BBuf<unsigned long long> d_tab; BBuf<int32_t> d_hits;
      d_tab.alloc(tab.size()); d_hits.alloc(nseq);
      BCK(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, s));
      int nsm = 0;
      BCK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
      const unsigned grid = (unsigned)std::max(1, std::min((nseq + FLT_WARPS - 1) / FLT_WARPS, nsm * 16));
      const char *sp = up.seq.p; const long long *op = up.off.p; const unsigned long long *tp = d_tab.p; int32_t *hp = d_hits.p;
      const int skip = non_overlapping ? word_size + 1 : 1;
      k_flt_match<<<grid, FLT_WARPS * 32, 0, s>>>(sp, op, nseq, tp, lg, word_size, skip, hp);
      BCK(cudaMemcpyAsync(hits, d_hits.p, (size_t)nseq * 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      BCK(cudaGetLastError());
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  if (s) cudaStreamDestroy(s);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

int dada2b_seq_complexity(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t kmer_size, int32_t window, int32_t device,
                          double *out, char errbuf[DADA2B_ERRLEN]) {
  cudaStream_t s = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!seq_off || (nseq > 0 && !out)) throw BErr{"dada2b: NULL argument."};
    if (nseq < 0) throw BErr{"dada2b: negative sequence count."};
    if (window > 0) throw BErr{"dada2b: seqComplexity with a window is not supported (only the whole-sequence form)."};
    if (kmer_size < 1 || kmer_size > 4) throw BErr{"dada2b: kmerSize must be 1..4."};
    need_device(device);
    if (nseq > 0) {
      BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      SeqUpload up; up.put(nseq, seq_concat, seq_off, s);
      BBuf<double> d_out; d_out.alloc(nseq);
      int nsm = 0;
      BCK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
      const unsigned grid = (unsigned)std::max(1, std::min((nseq + FLT_WARPS - 1) / FLT_WARPS, nsm * 16));
      const char *sp = up.seq.p; const long long *op = up.off.p; double *dp = d_out.p;
      k_flt_cplx<<<grid, FLT_WARPS * 32, 0, s>>>(sp, op, nseq, kmer_size, dp);
      BCK(cudaMemcpyAsync(out, d_out.p, (size_t)nseq * 8, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      BCK(cudaGetLastError());
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  if (s) cudaStreamDestroy(s);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

}  // extern "C"
