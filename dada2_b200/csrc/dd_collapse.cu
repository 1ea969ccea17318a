// collapseNoMismatch's inner loop on the H100 (include/dada2b_collapse.h).  Product code.
//
// Replaces the double loop of R/multiSample.R:125-144 (grepl prefix screen, then nwhamming(query, ref) == 0 through
// C_nwvec / C_nwalign and C_eval_pair, R/misc.R:216-220).  The device decides zero(j, i) = "screen passes and
// nwhamming(seq j, seq i) == 0" for every candidate pair i < j of the query-ordered sequences; the host then resolves the
// greedy loop: j collapses into the smallest i with zero(j, i) that is itself a representative (DESIGN.md 17).
//
//   k_col_keys / k_col_insert   hash table: minOverlap-prefix key -> list of the sequences with that prefix
//   k_col_screen<EMIT>          warp per sequence e: every lane hashes windows of e, probes the table and verifies each hit
//                               exactly on the packed rows; sequences shorter than minOverlap scan the table's rows directly.
//                               Each unordered pair {i, j} that passes either grepl is produced by exactly one warp.  Run once
//                               to count per sequence, then per block of sequences whose pairs fit the memory budget to emit.
//   k_col_allpairs              minOverlap <= 0: every pair passes the screen
//   k_col_filter                thread per candidate: max over all shifts of the gapless ends-free score, and whether a
//                               shift attaining it is an exact overlap; proves nwhamming > 0 for most candidates
//   k_col_align                 warp per survivor: nw_warp (dd_nw_warp.cuh, unbanded or banded) + C_eval_pair (dd_evalpair.cuh)
//
// isShiftDenovo (include/dada2b_align.h; R/chimeras.R:384-415) runs the same screen and filter (DESIGN.md 24):
//   k_shift_direct              drops screened pairs of equal abundance, directs the rest (less abundant = query)
//   k_col_filter                with E restricted to the overlaps a shift can have
//   k_nwalign                   (dd_align.cu) warp per survivor, unbanded ends-free, flags the query of every shift
// Integer and bit work only.  There is no CPU fallback.
#include "../../include/dada2b_collapse.h"
#include "dd_align.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <unordered_set>

namespace dd2 {

namespace {

// k <= 32 bases of a packed row from position p, 2 bits each, base p in bits 1:0.  Words past the row read as 0.
__device__ __forceinline__ unsigned long long win64(const uint32_t *row, int SW, int p, int k) {
  const int w = p >> 4, sh = 2 * (p & 15);
  const unsigned long long lo = (unsigned long long)row[w] | (w + 1 < SW ? (unsigned long long)row[w + 1] << 32 : 0ull);
  unsigned long long v = lo >> sh;
  if (sh && w + 2 < SW) v |= (unsigned long long)row[w + 2] << (64 - sh);
  return k >= 32 ? v : v & ((1ull << (2 * k)) - 1ull);
}
__device__ __forceinline__ int mism64(unsigned long long a, unsigned long long b) {
  const unsigned long long t = a ^ b;
  return __popcll((t | (t >> 1)) & 0x5555555555555555ull);
}
// bases [pa, pa + k) of row a equal bases [pb, pb + k) of row b
__device__ __forceinline__ bool eq_at(const uint32_t *ra, int pa, const uint32_t *rb, int pb, int k, int SW) {
  for (int c = 0; c < k; c += 32) {
    const int n = min(32, k - c);
    if (win64(ra, SW, pa + c, n) != win64(rb, SW, pb + c, n)) return false;
  }
  return true;
}
// grepl(needle, hay, fixed=TRUE) for a needle of nlen >= 1 bases
__device__ inline bool contains(const uint32_t *hay, int hlen, const uint32_t *ndl, int nlen, int SW) {
  for (int p = 0; p + nlen <= hlen; p++)
    if (eq_at(hay, p, ndl, 0, nlen, SW)) return true;
  return false;
}
// key of the m-base window at p: the bases themselves for m <= 32, a hash of them beyond (hits are verified exactly)
__device__ __forceinline__ unsigned long long key_at(const uint32_t *row, int SW, int p, int m) {
  if (m <= 32) return win64(row, SW, p, m);
  unsigned long long h = 0x243F6A8885A308D3ull;
  for (int c = 0; c < m; c += 32) { h = (h ^ win64(row, SW, p + c, min(32, m - c))) * 0x9E3779B97F4A7C15ull; h ^= h >> 31; }
  return h;
}
__device__ __forceinline__ unsigned slot_of(unsigned long long key, unsigned mask) {
  unsigned long long h = key * 0xD6E8FEB86659FD93ull;
  h ^= h >> 32;
  return (unsigned)h & mask;
}

struct ColScreenArgs {
  BimSeqs sq;
  int m;                                     // minOverlap >= 1
  unsigned long long *pkey;                  // [n] prefix key of every sequence with len >= m
  int32_t *tab_rep, *tab_head, *next;        // hash table: first sequence that claimed a slot (its key), list head; list links
  unsigned mask;
  int e0, e1;                                // sequences (warps) of this launch
  int32_t *cnt;                              // COUNT: pairs produced per sequence
  int32_t *pr, *pq;                          // EMIT: ref (smaller index) and query (larger index) of each candidate ...
  unsigned long long *npairs, cap;           // ... appended here, never past cap
  unsigned long long *ctr;                   // [2] overflow flag
};

__global__ void k_col_keys(ColScreenArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.sq.n) a.pkey[i] = a.sq.len[i] >= a.m ? key_at(a.sq.seq2 + (size_t)i * a.sq.SW, a.sq.SW, 0, a.m) : 0ull;
}

__global__ void k_col_insert(ColScreenArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.sq.n || a.sq.len[i] < a.m) return;
  const unsigned long long k = a.pkey[i];
  for (unsigned s = slot_of(k, a.mask);; s = (s + 1) & a.mask) {
    const int old = atomicCAS(&a.tab_rep[s], -1, i);
    if (old == -1 || a.pkey[old] == k) { a.next[i] = atomicExch(&a.tab_head[s], i); return; }
  }
}

// Pair {i < j} passes iff pre(i) occurs in j or pre(j) occurs in i, pre(x) = the first min(m, len x) bases.  Producer:
//   both lengths >= m: warp j if pre(i) occurs in j, else warp i (it finds pre(j) in i); each at the first occurrence only;
//   a shorter sequence s: its warp checks s against every row y (pre(y) cannot occur in s when y is at least m long, and
//   when both are shorter the longer one contains the other; equal lengths mean identical rows: the smaller index emits).
template <bool EMIT>
__global__ void __launch_bounds__(256) k_col_screen(ColScreenArgs a) {
  const int lane = threadIdx.x & 31, SW = a.sq.SW, m = a.m;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, tw = (gridDim.x * blockDim.x) >> 5;
  for (int e = a.e0 + gw; e < a.e1; e += tw) {
    const uint32_t *re = a.sq.seq2 + (size_t)e * SW;
    const int le = a.sq.len[e];
    int cnt = 0;
    auto emit = [&](int x) {
      if (EMIT) {
        const unsigned long long t = atomicAdd(a.npairs, 1ull);
        if (t < a.cap) { a.pr[t] = min(x, e); a.pq[t] = max(x, e); }
        else atomicMax(&a.ctr[1], 1ull);
      } else cnt++;
    };
    if (le >= m) {
      for (int p = lane; p + m <= le; p += 32) {
        const unsigned long long wk = key_at(re, SW, p, m);
        int x = -1;
        for (unsigned s = slot_of(wk, a.mask);; s = (s + 1) & a.mask) {
          const int r = a.tab_rep[s];
          if (r < 0) break;
          if (a.pkey[r] == wk) { x = a.tab_head[s]; break; }
        }
        for (; x >= 0; x = a.next[x]) {
          if (x == e) continue;
          const uint32_t *rx = a.sq.seq2 + (size_t)x * SW;
          if (!eq_at(rx, 0, re, p, m, SW)) continue;                 // exact check: a key collision never makes a candidate
          bool first = true;
          for (int q = 0; q < p && first; q++) first = !eq_at(re, q, rx, 0, m, SW);
          if (!first) continue;
          if (x > e && contains(rx, a.sq.len[x], re, m, SW)) continue;   // warp x produces it
          emit(x);
        }
      }
    } else {
      for (int y = lane; y < a.sq.n; y += 32) {
        const int ly = a.sq.len[y];
        if (y == e || ly < le || (ly == le && y < e)) continue;
        if (contains(a.sq.seq2 + (size_t)y * SW, ly, re, le, SW)) emit(y);
      }
    }
    if (!EMIT) {
#pragma unroll
      for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      if (lane == 0) a.cnt[e] = cnt;
    }
  }
}

// minOverlap <= 0: the empty prefix matches everywhere (R's grepl("", x) is TRUE), so every pair (i < e) is a candidate
__global__ void __launch_bounds__(256) k_col_allpairs(ColScreenArgs a) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, tw = (gridDim.x * blockDim.x) >> 5;
  for (int e = a.e0 + gw; e < a.e1; e += tw) {
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(a.npairs, (unsigned long long)e);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base + e > a.cap) { if (lane == 0) atomicMax(&a.ctr[1], 1ull); continue; }
    for (int i = lane; i < e; i += 32) { a.pr[base + i] = i; a.pq[base + i] = e; }
  }
}

struct ColFilterArgs {
  BimSeqs sq;
  int match, mismatch, unbanded;
  int o_lo, o_trim;                         // E counts overlaps in [o_lo, min(l1, l2) - o_trim]: 1, 0 for collapse; max(m, 1), 1 for isShiftDenovo
  const int32_t *pq, *pr;                   // s1 = query, s2 = ref of each pair
  const unsigned long long *np_ptr;         // pair count (device)
  uint32_t *alist; unsigned long long *nalign;   // pairs that need alignment
  int32_t *verdict;                         // test hook: 1 = needs alignment (may be NULL)
};

// Exact overlap filter (DESIGN.md 17, 24).  For every shift s (query base i against ref base i + s) with overlap o(s) > 0:
// g(s) = match * m(s) + mismatch * x(s).  LB = max g, E = some shift attaining LB has x = 0 and o(s) in [o_lo, o_hi],
// o_hi = min(l1, l2) - o_trim.
// Unbanded, LB > 0 and not E prove nwhamming > 0 (collapse, [1, INT_MAX]) or that the pair is no shift (isShiftDenovo).  Shifts go from the full-overlap plateau outwards, so o(s) only falls, and a shift whose best
// possible score o(s) * max(match, mismatch) is below LB can neither raise LB nor tie it exactly: the scan stops there.
__global__ void __launch_bounds__(256) k_col_filter(ColFilterArgs a) {
  const unsigned long long np = *a.np_ptr;
  const int lane = threadIdx.x & 31, SW = a.sq.SW;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const long long gmax = max(a.match, a.mismatch);
  for (unsigned long long x0 = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); x0 < np; x0 += stride) {
    const unsigned long long x = x0 + lane;
    bool need = false;
    if (x < np) {
      need = true;
      if (a.unbanded) {
        const int q = a.pq[x], r = a.pr[x];
        const uint32_t *rq = a.sq.seq2 + (size_t)q * SW, *rr = a.sq.seq2 + (size_t)r * SW;
        const int l1 = a.sq.len[q], l2 = a.sq.len[r];
        long long best = LLONG_MIN;
        bool exact = false;
        auto shift = [&](int s) -> bool {                 // false once no later shift can matter
          const int lo = max(0, -s), o = min(l1, l2 - s) - lo;
          if (o <= 0 || (long long)o * gmax < best) return false;
          int mm = 0;
          for (int c = 0; c < o; c += 32) {
            const int n = min(32, o - c);
            mm += mism64(win64(rq, SW, lo + c, n), win64(rr, SW, lo + s + c, n));
          }
          const long long g = (long long)a.match * (o - mm) + (long long)a.mismatch * mm;
          const bool ex = mm == 0 && o >= a.o_lo && o <= min(l1, l2) - a.o_trim;
          if (g > best) { best = g; exact = ex; }
          else if (g == best && ex) exact = true;
          return true;
        };
        const int slo = min(0, l2 - l1), shi = max(0, l2 - l1);      // o(s) = min(l1, l2) on [slo, shi]
        for (int s = slo; s <= shi; s++) shift(s);
        bool left = true, right = true;
        for (int d = 1; left || right; d++) {
          if (left) left = slo - d > -l1 && shift(slo - d);
          if (right) right = shi + d < l2 && shift(shi + d);
        }
        need = !(best > 0 && !exact);
      }
      if (a.verdict) a.verdict[x] = need ? 1 : 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, need);
    unsigned long long base = 0;
    if (lane == 0 && b && a.alist) base = atomicAdd(a.nalign, (unsigned long long)__popc(b));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (need && a.alist) a.alist[base + __popc(b & lanemask_lt())] = (uint32_t)x;
  }
}

struct ColAlignArgs {
  BimSeqs sq;
  AlnParams P;
  const int32_t *pq, *pr;
  const uint32_t *alist;                    // pairs to align (NULL: every pair x < *nalign)
  const unsigned long long *nalign;
  int32_t *ham;                             // test hook: nwhamming per pair (may be NULL)
  int32_t *zq, *zr; unsigned long long *nzero;   // pairs with nwhamming == 0 (may be NULL)
  unsigned long long *ctr;                  // [0] cells, [2] error flag
  int warp_words, seq_bytes, H_words, ops_words, mask_words, ptr_in_smem;
  uint32_t *ptr_scratch; unsigned long long ptr_words;
};

__global__ void __launch_bounds__(128) k_col_align(ColAlignArgs a) {
  extern __shared__ uint32_t smem[];
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = lane_id();
  const unsigned long long na = *a.nalign;
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
  for (unsigned long long t = gw; t < na; t += tw) {
    const unsigned long long x = a.alist ? a.alist[t] : t;
    const int q = a.pq[x], r = a.pr[x];
    const int len1 = a.sq.len[q], len2 = a.sq.len[r];
    unpack_row(a.sq.seq2 + (size_t)q * a.sq.SW, len1, s1, false);       // s1 = query (nwhamming's s1, al[0])
    unpack_row(a.sq.seq2 + (size_t)r * a.sq.SW, len2, s2, false);       // s2 = ref
    const int nops = nw_warp(s1, len1, s2, len2, a.P, H, ptr, opw, &cells_lane, &errflag);
    const EvalPair ev = eval_pair_warp(s1, s2, opw, nops, mQ, mP, mE);
    const int h = ev.mismatch + ev.indel;
    if (lane == 0) {
      if (a.ham) a.ham[x] = h;
      if (a.zq && h == 0) { const unsigned long long z = atomicAdd(a.nzero, 1ull); a.zq[z] = q; a.zr[z] = r; }
    }
    __syncwarp();
  }
  if (errflag && lane == 0) atomicMax(&a.ctr[2], (unsigned long long)errflag);
  unsigned cl = (unsigned)cells_lane;
#pragma unroll
  for (int o = 16; o; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
  if (lane == 0 && cl) atomicAdd(&a.ctr[0], (unsigned long long)cl);
}

// ---------------------------------------------------------------------------------------------------------------------
// host side

constexpr unsigned long long PAIR_BUDGET = 1ull << 24;          // candidates per block (about 20 bytes of device memory each)
constexpr unsigned long long SCRATCH_BUDGET = 1ull << 31;       // bytes of move-matrix scratch for the alignment kernel

struct Ctx {
  cudaStream_t s = nullptr;
  int num_sms = 132;
  long long launches = 0;
  float ms_align = 0;
  ~Ctx() { if (s) cudaStreamDestroy(s); }
};

void check_opts(const dada2b_collapse_opts &o, const BimSeqs &sq) {
  if (o.vec) check_int16(o.match, o.mismatch, o.gap_p, 1, sq.maxlen, 0);
}

// nw_warp's per-warp shared-memory layout and scratch, as in dd_merge.cu
struct ColAlignPlan { ColAlignArgs a; size_t smem; int grid; BBuf<uint32_t> d_ptr; };

void plan_align(ColAlignPlan &pl, const BimSeqs &sq, const dada2b_collapse_opts &o, int num_sms) {
  ColAlignArgs &a = pl.a;
  a = ColAlignArgs{};
  AlnParams &P = a.P;
  P.match = o.match; P.mismatch = o.mismatch; P.gap = o.gap_p; P.hgap = o.gap_p; P.band = o.band; P.homo = 0;
  if (o.vec) {
    const int m = std::min(std::min(o.mismatch, o.gap_p), std::min(o.match, 0));
    P.sentinel = (int)(int16_t)(INT16_MIN - m);                          // nwalign_vectorized.cpp:106
  } else P.sentinel = -9999;                                             // nwalign_endsfree.cpp:116-117
  const NwWarpLayout L = nw_warp_layout(sq.maxlen, sq.minlen, P.band);
  a.sq = sq;
  set_layout(a, L);
  pl.smem = L.smem;
  BCK(cudaFuncSetAttribute(k_col_align, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(pl.smem, 48 * 1024)));
  pl.grid = num_sms * 8;
  if (!a.ptr_in_smem) {
    const unsigned long long per_block = 4ull * a.ptr_words * 4;
    pl.grid = (int)std::max<unsigned long long>(1, std::min<unsigned long long>(pl.grid, SCRATCH_BUDGET / per_block));
    pl.d_ptr.alloc((size_t)pl.grid * 4 * a.ptr_words);
    a.ptr_scratch = pl.d_ptr.p;
  }
}

// The prefix screen's hash table (minOverlap >= 1)
struct Screen {
  ColScreenArgs a{};
  BBuf<unsigned long long> d_pkey;
  BBuf<int32_t> d_tab, d_next, d_cnt;
  void build(Ctx &c, const BimSeqs &sq, int m) {
    a.sq = sq; a.m = m;
    unsigned cap = 1024;
    while (cap < 2u * (unsigned)sq.n) cap <<= 1;
    a.mask = cap - 1;
    d_pkey.alloc(sq.n); d_tab.alloc(2 * (size_t)cap); d_next.alloc(sq.n); d_cnt.alloc(sq.n);
    a.pkey = d_pkey.p; a.tab_rep = d_tab.p; a.tab_head = d_tab.p + cap; a.next = d_next.p; a.cnt = d_cnt.p;
    BCK(cudaMemsetAsync(d_tab.p, 0xFF, 2 * (size_t)cap * 4, c.s));
    const int g = (sq.n + 255) / 256;
    k_col_keys<<<g, 256, 0, c.s>>>(a);
    k_col_insert<<<g, 256, 0, c.s>>>(a);
    c.launches += 2;
  }
  int warp_grid(const Ctx &c, int nwarp) const { return std::max(1, std::min(c.num_sms * 16, (nwarp + 7) / 8)); }
  // pairs produced by every sequence
  void count(Ctx &c, std::vector<int32_t> &cnt) {
    a.e0 = 0; a.e1 = a.sq.n;
    k_col_screen<false><<<warp_grid(c, a.sq.n), 256, 0, c.s>>>(a);
    c.launches++;
    cnt.resize(a.sq.n);
    BCK(cudaMemcpyAsync(cnt.data(), d_cnt.p, (size_t)a.sq.n * 4, cudaMemcpyDeviceToHost, c.s));
    BCK(cudaStreamSynchronize(c.s));
  }
};

// Candidate pairs of sequences [e0, e1) (m >= 1: the screen's producers; m <= 0: queries) -> pr / pq, count in *npairs
void emit_block(Ctx &c, Screen &scr, const BimSeqs &sq, int m, int e0, int e1, int32_t *pr, int32_t *pq,
                unsigned long long *npairs, unsigned long long cap, unsigned long long *ctr) {
  ColScreenArgs a = scr.a;
  a.sq = sq; a.e0 = e0; a.e1 = e1; a.pr = pr; a.pq = pq; a.npairs = npairs; a.cap = cap; a.ctr = ctr;
  const int g = std::max(1, std::min(c.num_sms * 16, (e1 - e0 + 7) / 8));
  if (m >= 1) k_col_screen<true><<<g, 256, 0, c.s>>>(a);
  else k_col_allpairs<<<g, 256, 0, c.s>>>(a);
  c.launches++;
}

// Blocks of producers whose pairs fit the budget (a single producer with more pairs gets a block of its own)
void plan_blocks(const std::vector<int32_t> &cnt, std::vector<std::pair<int, int>> &blocks, unsigned long long &maxblk,
                 unsigned long long &ncand) {
  const int nseq = (int)cnt.size();
  unsigned long long tot = 0;
  for (int e = 0, b0 = 0; e < nseq; e++) {
    if (tot && tot + (unsigned long long)cnt[e] > PAIR_BUDGET) { blocks.push_back({b0, e}); maxblk = std::max(maxblk, tot); b0 = e; tot = 0; }
    tot += (unsigned long long)cnt[e]; ncand += (unsigned long long)cnt[e];
    if (e == nseq - 1) { blocks.push_back({b0, nseq}); maxblk = std::max(maxblk, tot); }
  }
}

// Test hooks: the screen over the whole set in one block -> every candidate {i < j} as (i << 32 | j), each exactly once
std::unordered_set<unsigned long long> screen_set(Ctx &c, const BimSeqs &sq, int m, unsigned long long *d_ctr) {
  std::unordered_set<unsigned long long> cand;
  Screen scr;
  std::vector<int32_t> cnt;
  scr.build(c, sq, m);
  scr.count(c, cnt);
  unsigned long long want = 0;
  for (int e = 0; e < sq.n; e++) want += (unsigned long long)cnt[e];
  BBuf<int32_t> d_pr, d_pq;
  d_pr.alloc(std::max(want, 1ull)); d_pq.alloc(std::max(want, 1ull));
  emit_block(c, scr, sq, m, 0, sq.n, d_pr.p, d_pq.p, d_ctr + 4, want, d_ctr);
  unsigned long long h[8];
  std::vector<int32_t> pr(want), pq(want);
  BCK(cudaMemcpyAsync(h, d_ctr, sizeof h, cudaMemcpyDeviceToHost, c.s));
  if (want) {
    BCK(cudaMemcpyAsync(pr.data(), d_pr.p, want * 4, cudaMemcpyDeviceToHost, c.s));
    BCK(cudaMemcpyAsync(pq.data(), d_pq.p, want * 4, cudaMemcpyDeviceToHost, c.s));
  }
  BCK(cudaStreamSynchronize(c.s));
  if (h[1] || h[4] != want) throw BErr{"dada2b: collapse screen produced a different number of pairs than it counted."};
  for (unsigned long long t = 0; t < want; t++) {
    if (!(pr[t] < pq[t])) throw BErr{"dada2b: collapse screen produced a pair out of order."};
    if (!cand.insert((unsigned long long)pr[t] << 32 | (uint32_t)pq[t]).second) throw BErr{"dada2b: collapse screen produced a pair twice."};
  }
  return cand;
}

// isShiftDenovo: drops screened pairs of equal abundance (R compares strictly, R/chimeras.R:389) and directs the others
// as (query = the less abundant, parent = the more abundant), compacted into dq / dp
struct ShiftDirectArgs {
  const int32_t *pr, *pq;
  const unsigned long long *np_ptr;
  const int64_t *ab;
  int32_t *dq, *dp;
  unsigned long long *ndir, *nequal;
};

__global__ void __launch_bounds__(256) k_shift_direct(ShiftDirectArgs a) {
  const unsigned long long np = *a.np_ptr;
  const int lane = threadIdx.x & 31;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long x0 = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); x0 < np; x0 += stride) {
    const unsigned long long x = x0 + lane;
    int i = 0, j = 0;
    bool keep = false, eq = false;
    if (x < np) {
      i = a.pr[x]; j = a.pq[x];
      const int64_t ai = a.ab[i], aj = a.ab[j];
      eq = ai == aj;
      keep = !eq;
      if (ai > aj) { const int t = i; i = j; j = t; }                  // i: query (less abundant), j: parent
    }
    const unsigned b = __ballot_sync(0xffffffffu, keep), be = __ballot_sync(0xffffffffu, eq);
    unsigned long long base = 0;
    if (lane == 0) {
      if (b) base = atomicAdd(a.ndir, (unsigned long long)__popc(b));
      if (be) atomicAdd(a.nequal, (unsigned long long)__popc(be));
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    if (keep) { const unsigned long long t = base + __popc(b & lanemask_lt()); a.dq[t] = i; a.dp[t] = j; }
  }
}

dada2b_nwalign_opts shift_align_opts(const dada2b_shift_opts &o) {   // isShiftedPair: nwalign(sq, par, band=-1), :407
  dada2b_nwalign_opts n;
  dada2b_nwalign_default_opts(&n);
  n.match = o.match; n.mismatch = o.mismatch; n.gap_p = o.gap_p; n.homo_gap_p = o.gap_p;
  return n;
}

}  // namespace

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_collapse_default_opts(dada2b_collapse_opts *o) {     // R/multiSample.R:104, R/misc.R:216 + getDadaOpt defaults
  o->min_overlap = 20; o->match = 5; o->mismatch = -4; o->gap_p = -8; o->band = -1; o->vec = 1;
}

int dada2b_collapse_nomismatch(int32_t nseq, const char *seq_concat, const int64_t *seq_off, const dada2b_collapse_opts *opts,
                               int32_t device, int32_t *rep, dada2b_collapse_stats *stats, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ka = nullptr, kb = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!opts || !rep) throw BErr{"dada2b: NULL argument."};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    Ctx c;
    BCK(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&c.s, cudaStreamNonBlocking));
    BCK(cudaEventCreate(&ev0)); BCK(cudaEventCreate(&ev1)); BCK(cudaEventCreate(&ka)); BCK(cudaEventCreate(&kb));
    BCK(cudaEventRecord(ev0, c.s));
    long long h2d = 0;
    BimSeqs sq{};
    BBuf<uint32_t> d_seq2; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
    upload_packed_seqs(nseq, seq_concat, seq_off, c.s, d_seq2, d_len, len, sq, h2d, "collapseNoMismatch");
    check_opts(*opts, sq);
    const int m = opts->min_overlap;
    ColAlignPlan pl;
    plan_align(pl, sq, *opts, c.num_sms);
    Screen scr;
    std::vector<int32_t> cnt;
    if (m >= 1) { scr.build(c, sq, m); scr.count(c, cnt); }
    else { cnt.resize(nseq); for (int e = 0; e < nseq; e++) cnt[e] = e; }
    std::vector<std::pair<int, int>> blocks;
    unsigned long long maxblk = 1, ncand = 0;
    plan_blocks(cnt, blocks, maxblk, ncand);
    BBuf<int32_t> d_pr, d_pq, d_zq, d_zr; BBuf<uint32_t> d_alist; BBuf<unsigned long long> d_ctr;
    d_pr.alloc(maxblk); d_pq.alloc(maxblk); d_alist.alloc(maxblk); d_zq.alloc(maxblk); d_zr.alloc(maxblk); d_ctr.alloc(8);
    // d_ctr: [0] cells, [1] overflow, [2] error, [4] pairs, [5] aligned, [6] zero
    BCK(cudaMemsetAsync(d_ctr.p, 0, 64, c.s));
    ColFilterArgs fa{sq, opts->match, opts->mismatch, opts->band < 0 ? 1 : 0, 1, 0, d_pq.p, d_pr.p, d_ctr.p + 4, d_alist.p, d_ctr.p + 5, nullptr};
    ColAlignArgs &aa = pl.a;
    aa.pq = d_pq.p; aa.pr = d_pr.p; aa.alist = d_alist.p; aa.nalign = d_ctr.p + 5; aa.ham = nullptr;
    aa.zq = d_zq.p; aa.zr = d_zr.p; aa.nzero = d_ctr.p + 6; aa.ctr = d_ctr.p;
    std::vector<std::pair<int32_t, int32_t>> zero;                       // (query, ref)
    unsigned long long naligned = 0, ncells = 0;
    for (auto &b : blocks) {
      unsigned long long want = 0;
      for (int e = b.first; e < b.second; e++) want += (unsigned long long)cnt[e];
      if (!want) continue;
      BCK(cudaMemsetAsync(d_ctr.p + 4, 0, 24, c.s));
      emit_block(c, scr, sq, m, b.first, b.second, d_pr.p, d_pq.p, d_ctr.p + 4, want, d_ctr.p);
      k_col_filter<<<(int)std::max<unsigned long long>(1, std::min<unsigned long long>((unsigned long long)c.num_sms * 16, (want + 255) / 256)), 256, 0, c.s>>>(fa);
      BCK(cudaEventRecord(ka, c.s));
      k_col_align<<<pl.grid, 128, pl.smem, c.s>>>(aa);
      BCK(cudaEventRecord(kb, c.s));
      c.launches += 3;
      unsigned long long h[8];
      BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaStreamSynchronize(c.s));
      BCK(cudaGetLastError());
      if (h[1] || h[4] != want) throw BErr{"dada2b: collapse screen produced a different number of pairs than it counted."};
      if (h[2]) throw BErr{"N-W Align out of range."};                                   // nwalign_endsfree.cpp:184
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ka, kb)); c.ms_align += ms;
      naligned += h[5];
      const size_t nz = (size_t)h[6], z0 = zero.size();
      if (nz) {
        std::vector<int32_t> zq(nz), zr(nz);
        BCK(cudaMemcpyAsync(zq.data(), d_zq.p, nz * 4, cudaMemcpyDeviceToHost, c.s));
        BCK(cudaMemcpyAsync(zr.data(), d_zr.p, nz * 4, cudaMemcpyDeviceToHost, c.s));
        BCK(cudaStreamSynchronize(c.s));
        zero.resize(z0 + nz);
        for (size_t z = 0; z < nz; z++) zero[z0 + z] = {zq[z], zr[z]};
      }
    }
    unsigned long long h[8];
    BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, c.s));
    BCK(cudaEventRecord(ev1, c.s));
    BCK(cudaStreamSynchronize(c.s));
    ncells = h[0];
    // the greedy loop (R/multiSample.R:125-141): query j joins the first kept sequence, in keeping order, with zero(j, i)
    std::sort(zero.begin(), zero.end());
    for (int j = 0; j < nseq; j++) rep[j] = j;
    for (size_t z = 0; z < zero.size();) {
      const int j = zero[z].first;
      for (; z < zero.size() && zero[z].first == j; z++) {
        const int i = zero[z].second;
        if (rep[j] == j && rep[i] == i) rep[j] = i;
      }
    }
    if (stats) {
      memset(stats, 0, sizeof *stats);
      stats->n_candidates = (int64_t)ncand; stats->n_aligned = (int64_t)naligned; stats->n_filtered = (int64_t)(ncand - naligned);
      stats->n_zero = (int64_t)zero.size(); stats->n_cells = (int64_t)ncells; stats->n_blocks = (int64_t)blocks.size();
      stats->gpu_launches = c.launches;
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ev0, ev1)); stats->ms_device = ms;
      stats->ms_k_align = c.ms_align;
      stats->ms_total = bnow_ms() - t0;
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (cudaEvent_t e : {ev0, ev1, ka, kb}) if (e) cudaEventDestroy(e);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

int dada2b_test_collapse_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *query,
                               const int32_t *ref, const dada2b_collapse_opts *opts, int32_t device, int32_t *out3,
                               char errbuf[DADA2B_ERRLEN]) {
  int rc = 0;
  std::string msg;
  try {
    if (!opts || (npairs && (!query || !ref || !out3))) throw BErr{"dada2b: NULL argument."};
    if (npairs < 0) throw BErr{"dada2b: negative pair count."};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    Ctx c;
    BCK(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&c.s, cudaStreamNonBlocking));
    long long h2d = 0;
    BimSeqs sq{};
    BBuf<uint32_t> d_seq2; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
    upload_packed_seqs(nseq, seq_concat, seq_off, c.s, d_seq2, d_len, len, sq, h2d, "collapseNoMismatch");
    for (int x = 0; x < npairs; x++)
      if (query[x] < 0 || query[x] >= nseq || ref[x] < 0 || ref[x] >= nseq) throw BErr{"dada2b: bad pair index."};
    check_opts(*opts, sq);
    const int m = opts->min_overlap;
    BBuf<unsigned long long> d_ctr;
    d_ctr.alloc(8);
    BCK(cudaMemsetAsync(d_ctr.p, 0, 64, c.s));
    // 1. the product's screen over the whole set, in one block: the candidate set, each unordered pair exactly once
    std::unordered_set<unsigned long long> cand;
    if (m >= 1) cand = screen_set(c, sq, m, d_ctr.p);
    for (int x = 0; x < npairs; x++) {
      const int a = std::min(query[x], ref[x]), b = std::max(query[x], ref[x]);
      out3[3 * (size_t)x] = m < 1 ? (a != b) : (int)cand.count((unsigned long long)a << 32 | (uint32_t)b);
    }
    if (npairs) {
      // 2. the filter's verdict and 3. the aligned nwhamming of every given pair
      BBuf<int32_t> d_q, d_r, d_ver, d_ham;
      d_q.alloc(npairs); d_r.alloc(npairs); d_ver.alloc(npairs); d_ham.alloc(npairs);
      BCK(cudaMemcpyAsync(d_q.p, query, (size_t)npairs * 4, cudaMemcpyHostToDevice, c.s));
      BCK(cudaMemcpyAsync(d_r.p, ref, (size_t)npairs * 4, cudaMemcpyHostToDevice, c.s));
      const unsigned long long np = (unsigned long long)npairs;
      BCK(cudaMemcpyAsync(d_ctr.p + 4, &np, 8, cudaMemcpyHostToDevice, c.s));
      ColFilterArgs fa{sq, opts->match, opts->mismatch, opts->band < 0 ? 1 : 0, 1, 0, d_q.p, d_r.p, d_ctr.p + 4, nullptr, nullptr, d_ver.p};
      k_col_filter<<<std::max(1, std::min(c.num_sms * 16, (npairs + 255) / 256)), 256, 0, c.s>>>(fa);
      ColAlignPlan pl;
      plan_align(pl, sq, *opts, c.num_sms);
      ColAlignArgs &aa = pl.a;
      aa.pq = d_q.p; aa.pr = d_r.p; aa.alist = nullptr; aa.nalign = d_ctr.p + 4; aa.ham = d_ham.p; aa.zq = nullptr; aa.ctr = d_ctr.p;
      k_col_align<<<pl.grid, 128, pl.smem, c.s>>>(aa);
      std::vector<int32_t> ver(npairs), ham(npairs);
      unsigned long long h[8];
      BCK(cudaMemcpyAsync(ver.data(), d_ver.p, (size_t)npairs * 4, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaMemcpyAsync(ham.data(), d_ham.p, (size_t)npairs * 4, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaStreamSynchronize(c.s));
      BCK(cudaGetLastError());
      if (h[2]) throw BErr{"N-W Align out of range."};
      for (int x = 0; x < npairs; x++) { out3[3 * (size_t)x + 1] = ver[x]; out3[3 * (size_t)x + 2] = ham[x]; }
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

void dada2b_shift_default_opts(dada2b_shift_opts *o) {          // R/chimeras.R:384 + getDadaOpt defaults
  o->min_overlap = 20; o->match = 5; o->mismatch = -4; o->gap_p = -8;
}

// isShiftDenovo (R/chimeras.R:384-400): every pair the screen passes, of different abundances, directed, filtered, aligned
int dada2b_shift_denovo(int32_t nseq, const char *seq_concat, const int64_t *seq_off, const int64_t *abund,
                        const dada2b_shift_opts *opts, int32_t device, uint8_t *flag, dada2b_shift_stats *stats,
                        char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ka = nullptr, kb = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!opts || !flag || !abund) throw BErr{"dada2b: NULL argument."};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    Ctx c;
    BCK(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&c.s, cudaStreamNonBlocking));
    BCK(cudaEventCreate(&ev0)); BCK(cudaEventCreate(&ev1)); BCK(cudaEventCreate(&ka)); BCK(cudaEventCreate(&kb));
    BCK(cudaEventRecord(ev0, c.s));
    long long h2d = 0;
    BimSeqs sq{};
    BBuf<uint32_t> d_seq2; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
    upload_packed_seqs(nseq, seq_concat, seq_off, c.s, d_seq2, d_len, len, sq, h2d, "isShiftDenovo");
    const int m = opts->min_overlap;
    NwAlignPlan pl;
    nwalign_plan(pl, sq, shift_align_opts(*opts), c.num_sms);
    Screen scr;
    std::vector<int32_t> cnt;
    if (m >= 1) { scr.build(c, sq, m); scr.count(c, cnt); }
    else { cnt.resize(nseq); for (int e = 0; e < nseq; e++) cnt[e] = e; }
    std::vector<std::pair<int, int>> blocks;
    unsigned long long maxblk = 1, nscreen = 0;
    plan_blocks(cnt, blocks, maxblk, nscreen);
    BBuf<int32_t> d_pr, d_pq, d_dq, d_dp; BBuf<uint32_t> d_alist; BBuf<unsigned long long> d_ctr; BBuf<int64_t> d_ab; BBuf<uint8_t> d_flag;
    d_pr.alloc(maxblk); d_pq.alloc(maxblk); d_dq.alloc(maxblk); d_dp.alloc(maxblk); d_alist.alloc(maxblk); d_ctr.alloc(8);
    d_ab.alloc(nseq); d_flag.alloc(nseq);
    BCK(cudaMemcpyAsync(d_ab.p, abund, (size_t)nseq * 8, cudaMemcpyHostToDevice, c.s));
    BCK(cudaMemsetAsync(d_flag.p, 0, (size_t)nseq, c.s));
    // d_ctr: [0] cells, [1] overflow, [2] error, [4] pairs, [5] aligned, [6] directed, [7] equal
    BCK(cudaMemsetAsync(d_ctr.p, 0, 64, c.s));
    const ShiftDirectArgs da{d_pr.p, d_pq.p, d_ctr.p + 4, d_ab.p, d_dq.p, d_dp.p, d_ctr.p + 6, d_ctr.p + 7};
    // the filter's E counts the overlaps a shift can have: match in [max(m, 1), min(l1, l2) - 1] (:409-410)
    const ColFilterArgs fa{sq, opts->match, opts->mismatch, 1, std::max(m, 1), 1, d_dq.p, d_dp.p, d_ctr.p + 6, d_alist.p, d_ctr.p + 5, nullptr};
    NwAlignArgs &aa = pl.a;
    aa.s1 = d_dq.p; aa.s2 = d_dp.p; aa.alist = d_alist.p; aa.npairs_ptr = d_ctr.p + 5; aa.flag = d_flag.p; aa.min_overlap = m;
    aa.ctr = d_ctr.p;
    unsigned long long naligned = 0, nequal = 0, ncand = 0;
    for (auto &b : blocks) {
      unsigned long long want = 0;
      for (int e = b.first; e < b.second; e++) want += (unsigned long long)cnt[e];
      if (!want) continue;
      BCK(cudaMemsetAsync(d_ctr.p + 4, 0, 32, c.s));
      emit_block(c, scr, sq, m, b.first, b.second, d_pr.p, d_pq.p, d_ctr.p + 4, want, d_ctr.p);
      const int g = (int)std::max<unsigned long long>(1, std::min<unsigned long long>((unsigned long long)c.num_sms * 16, (want + 255) / 256));
      k_shift_direct<<<g, 256, 0, c.s>>>(da);
      k_col_filter<<<g, 256, 0, c.s>>>(fa);
      BCK(cudaEventRecord(ka, c.s));
      nwalign_launch(pl, c.s);
      BCK(cudaEventRecord(kb, c.s));
      c.launches += 4;
      unsigned long long h[8];
      BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaStreamSynchronize(c.s));
      BCK(cudaGetLastError());
      if (h[1] || h[4] != want) throw BErr{"dada2b: collapse screen produced a different number of pairs than it counted."};
      if (h[2]) throw BErr{"N-W Align out of range."};                                   // nwalign_endsfree.cpp:184
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ka, kb)); c.ms_align += ms;
      naligned += h[5]; ncand += h[6]; nequal += h[7];
    }
    BCK(cudaMemcpyAsync(flag, d_flag.p, (size_t)nseq, cudaMemcpyDeviceToHost, c.s));
    unsigned long long h[8];
    BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, c.s));
    BCK(cudaEventRecord(ev1, c.s));
    BCK(cudaStreamSynchronize(c.s));
    if (stats) {
      memset(stats, 0, sizeof *stats);
      stats->n_screened = (int64_t)nscreen; stats->n_equal = (int64_t)nequal; stats->n_candidates = (int64_t)ncand;
      stats->n_aligned = (int64_t)naligned; stats->n_filtered = (int64_t)(ncand - naligned);
      int64_t nf = 0;
      for (int i = 0; i < nseq; i++) nf += flag[i] != 0;
      stats->n_flagged = nf; stats->n_cells = (int64_t)h[0]; stats->n_blocks = (int64_t)blocks.size();
      stats->gpu_launches = c.launches;
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ev0, ev1)); stats->ms_device = ms;
      stats->ms_k_align = c.ms_align;
      stats->ms_total = bnow_ms() - t0;
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (cudaEvent_t e : {ev0, ev1, ka, kb}) if (e) cudaEventDestroy(e);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

int dada2b_test_shift_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *query,
                            const int32_t *parent, const dada2b_shift_opts *opts, int32_t device, int32_t *out5,
                            char errbuf[DADA2B_ERRLEN]) {
  int rc = 0;
  std::string msg;
  try {
    if (!opts || (npairs && (!query || !parent || !out5))) throw BErr{"dada2b: NULL argument."};
    if (npairs < 0) throw BErr{"dada2b: negative pair count."};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    Ctx c;
    BCK(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&c.s, cudaStreamNonBlocking));
    long long h2d = 0;
    BimSeqs sq{};
    BBuf<uint32_t> d_seq2; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
    upload_packed_seqs(nseq, seq_concat, seq_off, c.s, d_seq2, d_len, len, sq, h2d, "isShiftDenovo");
    for (int x = 0; x < npairs; x++)
      if (query[x] < 0 || query[x] >= nseq || parent[x] < 0 || parent[x] >= nseq) throw BErr{"dada2b: bad pair index."};
    const int m = opts->min_overlap;
    BBuf<unsigned long long> d_ctr;
    d_ctr.alloc(8);
    BCK(cudaMemsetAsync(d_ctr.p, 0, 64, c.s));
    std::unordered_set<unsigned long long> cand;
    if (m >= 1) cand = screen_set(c, sq, m, d_ctr.p);
    for (int x = 0; x < npairs; x++) {
      const int a = std::min(query[x], parent[x]), b = std::max(query[x], parent[x]);
      out5[5 * (size_t)x] = m < 1 ? (a != b) : (int)cand.count((unsigned long long)a << 32 | (uint32_t)b);
    }
    if (npairs) {
      BBuf<int32_t> d_q, d_p, d_ver, d_cnt;
      d_q.alloc(npairs); d_p.alloc(npairs); d_ver.alloc(npairs); d_cnt.alloc(3 * (size_t)npairs);
      BCK(cudaMemcpyAsync(d_q.p, query, (size_t)npairs * 4, cudaMemcpyHostToDevice, c.s));
      BCK(cudaMemcpyAsync(d_p.p, parent, (size_t)npairs * 4, cudaMemcpyHostToDevice, c.s));
      const unsigned long long np = (unsigned long long)npairs;
      BCK(cudaMemcpyAsync(d_ctr.p + 4, &np, 8, cudaMemcpyHostToDevice, c.s));
      const ColFilterArgs fa{sq, opts->match, opts->mismatch, 1, std::max(m, 1), 1, d_q.p, d_p.p, d_ctr.p + 4, nullptr, nullptr, d_ver.p};
      k_col_filter<<<std::max(1, std::min(c.num_sms * 16, (npairs + 255) / 256)), 256, 0, c.s>>>(fa);
      NwAlignPlan pl;
      nwalign_plan(pl, sq, shift_align_opts(*opts), c.num_sms);
      NwAlignArgs &aa = pl.a;
      aa.s1 = d_q.p; aa.s2 = d_p.p; aa.npairs = np; aa.counts = d_cnt.p; aa.ctr = d_ctr.p;
      nwalign_launch(pl, c.s);
      std::vector<int32_t> ver(npairs), cn(3 * (size_t)npairs);
      unsigned long long h[8];
      BCK(cudaMemcpyAsync(ver.data(), d_ver.p, (size_t)npairs * 4, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaMemcpyAsync(cn.data(), d_cnt.p, (size_t)npairs * 12, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, c.s));
      BCK(cudaStreamSynchronize(c.s));
      BCK(cudaGetLastError());
      if (h[2]) throw BErr{"N-W Align out of range."};
      for (int x = 0; x < npairs; x++) {
        int32_t *o = out5 + 5 * (size_t)x;
        o[1] = ver[x]; o[2] = cn[3 * (size_t)x]; o[3] = cn[3 * (size_t)x + 1]; o[4] = cn[3 * (size_t)x + 2];
      }
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

}  // extern "C"
