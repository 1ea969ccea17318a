// nwalign batched over pairs on the H100 (include/dada2b_align.h).  Product code.
//
// Replaces, per pair (under R/misc.R:179-191):
//   C_nwalign -> nwalign_endsfree / nwalign_endsfree_homo / nwalign (endsfree=FALSE)   evaluate.cpp:18-61,
//                                                                                      nwalign_endsfree.cpp:76-537
//   C_nwvec   -> nwalign_vectorized2 (end_gap 0, or end_gap = gap with endsfree=FALSE)  nwalign_vectorized.cpp:321-343
// and optionally C_eval_pair (evaluate.cpp:73-120).  One warp per pair: nw_warp (dd_nw_warp.cuh; its GLOBAL instantiation
// for endsfree=FALSE), then one lane-parallel pass over the move string that writes both aligned rows, and
// eval_pair_warp (dd_evalpair.cuh) for the counts.  The vectorized aligner differs from the scalar one only in its int16
// scores and out-of-band fill value (DESIGN.md 17, 24).  Integer / byte work only.  There is no CPU fallback.
#include "dd_align.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace dd2 {

template <bool GLOBAL>
__global__ void __launch_bounds__(128) k_nwalign(NwAlignArgs a) {
  extern __shared__ uint32_t smem[];
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = lane_id();
  const unsigned long long np = a.npairs_ptr ? *a.npairs_ptr : a.npairs;
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
  auto nt = [](int b) { return (char)((0x54474341u >> (8 * (b & 3))) & 0xFFu); };      // 'A','C','G','T'
  for (unsigned long long t = gw; t < np; t += tw) {
    const unsigned long long x = a.alist ? a.alist[t] : t;
    const int q = a.s1[x], r = a.s2[x];
    const int len1 = a.sq.len[q], len2 = a.sq.len[r];
    unpack_row(a.sq.seq2 + (size_t)q * a.sq.SW, len1, s1, !GLOBAL && a.P.homo != 0);
    unpack_row(a.sq.seq2 + (size_t)r * a.sq.SW, len2, s2, !GLOBAL && a.P.homo != 0);
    const int nops = nw_warp<GLOBAL>(s1, len1, s2, len2, a.P, H, ptr, opw, &cells_lane, &errflag);
    if (a.al1) {
      // the moves in forward order: column col consumes a base of s1 unless it is a gap there (op 2), of s2 unless op 3
      char *o1 = a.al1 + (a.al_off[x] - a.al_base), *o2 = a.al2 + (a.al_off[x] - a.al_base);
      int i0b = 0, i1b = 0;
      for (int ch = 0; ch * 32 < nops; ch++) {
        const int col = ch * 32 + lane;
        int op = 0;
        if (col < nops) { const int e = nops - 1 - col; op = (opw[e >> 4] >> (2 * (e & 15))) & 3; }
        const unsigned b0 = __ballot_sync(0xffffffffu, op == 1 || op == 3), b1 = __ballot_sync(0xffffffffu, op == 1 || op == 2);
        const int i0 = i0b + __popc(b0 & lanemask_lt()), i1 = i1b + __popc(b1 & lanemask_lt());
        if (op) { o1[col] = op == 2 ? '-' : nt(s1[i0]); o2[col] = op == 3 ? '-' : nt(s2[i1]); }
        i0b += __popc(b0); i1b += __popc(b1);
      }
      if (lane == 0) a.al_len[x] = nops;
    }
    if (a.counts || a.flag) {
      const EvalPair ev = eval_pair_warp(s1, s2, opw, nops, mQ, mP, mE);
      if (lane == 0) {
        if (a.counts) { int32_t *o = a.counts + (size_t)x * 3; o[0] = ev.match; o[1] = ev.mismatch; o[2] = ev.indel; }
        // isShiftedPair (R/chimeras.R:406-411), flagSubseqs never set (:391)
        if (a.flag && ev.match < len1 && ev.match < len2 && ev.match >= a.min_overlap && ev.mismatch == 0 && ev.indel == 0)
          a.flag[q] = 1;
      }
    }
    __syncwarp();
  }
  if (errflag && lane == 0) atomicMax(&a.ctr[2], (unsigned long long)errflag);
  unsigned cl = (unsigned)cells_lane;
#pragma unroll
  for (int o = 16; o; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
  if (lane == 0 && cl) atomicAdd(&a.ctr[0], (unsigned long long)cl);
}

constexpr unsigned long long SCRATCH_BUDGET = 1ull << 31;       // bytes of move-matrix scratch for the alignment kernel
constexpr unsigned long long ROW_BUDGET = 1ull << 28;           // bytes of aligned rows (both) per block of pairs
constexpr unsigned long long PAIRS_PER_BLOCK = 1ull << 24;

void check_int16(int match, int mismatch, int gap_p, int endsfree, int maxlen, long long maxsum) {
  // nwalign_vectorized2 keeps scores in int16 (DESIGN.md 24): beyond 32767 the reference would wrap around
  const long long A = std::max(std::llabs(match), std::llabs(mismatch)), G = std::llabs(gap_p);
  if (endsfree) {
    // every cell of the ends-free matrix lies within A * minlen of 0 (a diagonal path from the free first row or column
    // reaches it), and a candidate adds one more score or gap
    const long long bound = A * maxlen + std::max(A, G);
    if (bound > 32767 || G > 32767)
      throw BErr{"dada2b: sequences too long for the vectorized aligner's 16-bit scores (max(|match|, |mismatch|) * maxlen + "
                 "max(|match|, |mismatch|, |gap|) must stay <= 32767); use vec=FALSE."};
  } else {
    // every cell of the global matrix is the score of a path of at most len1 + len2 scored steps
    if (std::max(A, G) * (maxsum + 1) > 32767)
      throw BErr{"dada2b: sequences too long for the vectorized aligner's 16-bit scores (max(|match|, |mismatch|, |gap|) * "
                 "(len1 + len2 + 1) must stay <= 32767); use vec=FALSE."};
  }
}

void nwalign_plan(NwAlignPlan &pl, const BimSeqs &sq, const dada2b_nwalign_opts &o, int num_sms) {
  NwAlignArgs &a = pl.a;
  a = NwAlignArgs{};
  AlnParams &P = a.P;
  pl.global = o.endsfree == 0;
  P.match = o.match; P.mismatch = o.mismatch; P.gap = o.gap_p; P.hgap = o.homo_gap_p; P.band = o.band;
  P.homo = (!o.vec && o.endsfree && o.homo_gap_p != o.gap_p) ? 1 : 0;   // evaluate.cpp:40-46
  if (o.vec) {
    const int m = std::min(std::min(o.mismatch, o.gap_p), std::min(o.match, 0));
    P.sentinel = (int)(int16_t)(INT16_MIN - m);                          // nwalign_vectorized.cpp:106
  } else P.sentinel = -9999;                                             // nwalign_endsfree.cpp:116-117, :446-447
  const NwWarpLayout L = nw_warp_layout(sq.maxlen, sq.minlen, P.band);
  a.sq = sq;
  set_layout(a, L);
  pl.smem = L.smem;
  const int smax = (int)std::max<size_t>(pl.smem, 48 * 1024);
  BCK(cudaFuncSetAttribute(k_nwalign<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
  BCK(cudaFuncSetAttribute(k_nwalign<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
  pl.grid = num_sms * 8;
  if (!a.ptr_in_smem) {
    const unsigned long long per_block = 4ull * a.ptr_words * 4;
    pl.grid = (int)std::max<unsigned long long>(1, std::min<unsigned long long>(pl.grid, SCRATCH_BUDGET / per_block));
    pl.d_ptr.alloc((size_t)pl.grid * 4 * a.ptr_words);
    a.ptr_scratch = pl.d_ptr.p;
  }
}

void nwalign_launch(const NwAlignPlan &pl, cudaStream_t s) {
  const NwAlignArgs a = pl.a;
  if (pl.global) k_nwalign<true><<<pl.grid, 128, pl.smem, s>>>(a);
  else k_nwalign<false><<<pl.grid, 128, pl.smem, s>>>(a);
}

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_nwalign_default_opts(dada2b_nwalign_opts *o) {       // R/misc.R:179 + getDadaOpt defaults
  o->match = 5; o->mismatch = -4; o->gap_p = -8; o->homo_gap_p = -8; o->band = -1; o->endsfree = 1; o->vec = 0;
}

int dada2b_nwalign(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *s1_idx,
                   const int32_t *s2_idx, const dada2b_nwalign_opts *opts, int32_t device, char *al1, char *al2,
                   int32_t *al_len, int32_t *counts, dada2b_nwalign_stats *stats, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ka = nullptr, kb = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!opts || (npairs && (!s1_idx || !s2_idx))) throw BErr{"dada2b: NULL argument."};
    if (npairs < 0) throw BErr{"dada2b: negative pair count."};
    if (!al1 != !al2 || (al1 && !al_len)) throw BErr{"dada2b: aligned rows need al1, al2 and al_len."};
    if (opts->vec && opts->homo_gap_p != opts->gap_p)
      throw BErr{"Homopolymer gap penalties are not implemented in the vectorized aligner."};      // R/misc.R:183
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    int num_sms = 132;
    BCK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    BCK(cudaEventCreate(&ev0)); BCK(cudaEventCreate(&ev1)); BCK(cudaEventCreate(&ka)); BCK(cudaEventCreate(&kb));
    BCK(cudaEventRecord(ev0, s));
    long long h2d = 0;
    BimSeqs sq{};
    BBuf<uint32_t> d_seq2; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
    upload_packed_seqs(nseq, seq_concat, seq_off, s, d_seq2, d_len, len, sq, h2d, "nwalign");
    std::vector<int64_t> off((size_t)npairs + 1, 0);
    long long maxsum = 0;
    for (int x = 0; x < npairs; x++) {
      if (s1_idx[x] < 0 || s1_idx[x] >= nseq || s2_idx[x] < 0 || s2_idx[x] >= nseq) throw BErr{"dada2b: bad pair index."};
      const long long l = (long long)len[s1_idx[x]] + len[s2_idx[x]];
      maxsum = std::max(maxsum, l);
      off[x + 1] = off[x] + l;
    }
    if (opts->vec) check_int16(opts->match, opts->mismatch, opts->gap_p, opts->endsfree, sq.maxlen, maxsum);
    NwAlignPlan pl;
    nwalign_plan(pl, sq, *opts, num_sms);
    // blocks of consecutive pairs whose rows fit the budget (a single pair always fits: 2 * 2 * 9998 bytes)
    std::vector<std::pair<int, int>> blocks;
    for (int b0 = 0, x = 0; x < npairs; x++) {
      if (x > b0 && ((unsigned long long)(off[x + 1] - off[b0]) * (al1 ? 2 : 0) > ROW_BUDGET || (unsigned long long)(x - b0) >= PAIRS_PER_BLOCK)) {
        blocks.push_back({b0, x}); b0 = x;
      }
      if (x == npairs - 1) blocks.push_back({b0, npairs});
    }
    unsigned long long maxrow = 1;
    for (auto &b : blocks) maxrow = std::max<unsigned long long>(maxrow, (unsigned long long)(off[b.second] - off[b.first]));
    const size_t np1 = std::max(npairs, 1);
    BBuf<int32_t> d_s1, d_s2, d_counts, d_alen; BBuf<int64_t> d_off; BBuf<char> d_al1, d_al2; BBuf<unsigned long long> d_ctr;
    d_s1.alloc(np1); d_s2.alloc(np1); d_ctr.alloc(8);
    if (counts) d_counts.alloc(np1 * 3);
    if (al1) { d_alen.alloc(np1); d_off.alloc(np1 + 1); d_al1.alloc(maxrow); d_al2.alloc(maxrow); }
    BCK(cudaMemsetAsync(d_ctr.p, 0, 64, s));
    if (npairs) {
      BCK(cudaMemcpyAsync(d_s1.p, s1_idx, (size_t)npairs * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_s2.p, s2_idx, (size_t)npairs * 4, cudaMemcpyHostToDevice, s));
      if (al1) BCK(cudaMemcpyAsync(d_off.p, off.data(), ((size_t)npairs + 1) * 8, cudaMemcpyHostToDevice, s));
    }
    NwAlignArgs &a = pl.a;
    a.ctr = d_ctr.p;
    float ms_align = 0;
    for (auto &b : blocks) {
      a.s1 = d_s1.p + b.first; a.s2 = d_s2.p + b.first; a.npairs = (unsigned long long)(b.second - b.first);
      a.counts = counts ? d_counts.p + 3 * (size_t)b.first : nullptr;
      if (al1) { a.al_off = d_off.p + b.first; a.al_base = off[b.first]; a.al1 = d_al1.p; a.al2 = d_al2.p; a.al_len = d_alen.p + b.first; }
      BCK(cudaEventRecord(ka, s));
      nwalign_launch(pl, s);
      BCK(cudaEventRecord(kb, s));
      if (al1) {
        const size_t nb = (size_t)(off[b.second] - off[b.first]);
        BCK(cudaMemcpyAsync(al1 + off[b.first], d_al1.p, nb, cudaMemcpyDeviceToHost, s));
        BCK(cudaMemcpyAsync(al2 + off[b.first], d_al2.p, nb, cudaMemcpyDeviceToHost, s));
      }
      BCK(cudaStreamSynchronize(s));
      BCK(cudaGetLastError());
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ka, kb)); ms_align += ms;
    }
    if (npairs) {
      if (counts) BCK(cudaMemcpyAsync(counts, d_counts.p, (size_t)npairs * 12, cudaMemcpyDeviceToHost, s));
      if (al1) BCK(cudaMemcpyAsync(al_len, d_alen.p, (size_t)npairs * 4, cudaMemcpyDeviceToHost, s));
    }
    unsigned long long h[8];
    BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, s));
    BCK(cudaEventRecord(ev1, s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    if (h[2]) throw BErr{"N-W Align out of range."};                     // nwalign_endsfree.cpp:184, :499
    if (stats) {
      memset(stats, 0, sizeof *stats);
      stats->n_pairs = npairs; stats->n_cells = (int64_t)h[0]; stats->n_blocks = (int64_t)blocks.size();
      stats->gpu_launches = (int64_t)blocks.size();
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ev0, ev1)); stats->ms_device = ms;
      stats->ms_k_align = ms_align;
      stats->ms_total = bnow_ms() - t0;
    }
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (cudaEvent_t e : {ev0, ev1, ka, kb}) if (e) cudaEventDestroy(e);
  if (s) cudaStreamDestroy(s);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

}  // extern "C"
