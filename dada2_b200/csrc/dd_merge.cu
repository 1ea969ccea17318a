// mergePairs' alignment / evaluation / consensus step on the H100 (include/dada2b_merge.h).  Product code.
//
// Replaces, fused per pairing and batched over all pairings of a sample (under /root/reference/src):
//   C_nwalign (endsfree)  -> nwalign_endsfree / nwalign_endsfree_homo      evaluate.cpp:18-61, nwalign_endsfree.cpp:76-396
//   C_eval_pair                                                             evaluate.cpp:73-120
//   C_pair_consensus                                                        evaluate.cpp:131-174
// One warp per pairing: the warp-per-pair NW with traceback of dd_nw_warp.cuh (unbanded for mergePairs: the move matrix
// lives in a per-warp global scratch row), then two lane-parallel passes over the alignment columns -- column masks and
// end-gap runs for the counts, consensus characters written straight to the output row.  Integer / byte work only.
#include "dd_merge.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace dd2 {

__global__ void __launch_bounds__(128) k_merge_pairs(MergeArgs a) {
  extern __shared__ uint32_t smem[];
  const int nwarps = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = lane_id();
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
  for (int jb = gw; jb < a.npairs; jb += tw) {
    const uint32_t q = (uint32_t)a.s1_idx[jb], k = (uint32_t)a.s2_idx[jb];
    const int prefer = a.prefer[jb];
    const int len1 = a.sq.len[q], len2 = a.sq.len[k];
    unpack_row(a.sq.seq2 + (size_t)q * a.sq.SW, len1, s1, a.P.homo != 0);     // s1 = forward ASV       (al[0])
    unpack_row(a.sq.seq2 + (size_t)k * a.sq.SW, len2, s2, a.P.homo != 0);     // s2 = rc(reverse ASV)   (al[1])
    const int nops = nw_warp(s1, len1, s2, len2, a.P, H, ptr, opw, &cells_lane, &errflag);
    // pass 1: column masks and C_eval_pair's counts (dd_evalpair.cuh)
    const EvalPair ev = eval_pair_warp(s1, s2, opw, nops, mQ, mP, mE);
    const int n = nops, nch = (nops + 31) >> 5, leadQ = ev.leadQ, trailP = ev.trailP;
    int i0b, i1b;
    if (lane == 0) { int32_t *o = a.counts + (size_t)jb * 3; o[0] = ev.match; o[1] = ev.mismatch; o[2] = ev.indel; }
    // pass 2: C_pair_consensus (evaluate.cpp:131-174); with trim_overhang the leading columns where s1 has a gap and the
    // trailing columns where s2 has a gap are dropped (:152-160); no other column is a double gap, so the kept range is contiguous
    const int drop_lo = a.trim_overhang ? leadQ : 0, drop_hi = a.trim_overhang ? trailP : 0;
    char *out = a.cons + (size_t)jb * a.cons_stride;
    i0b = 0; i1b = 0;
    for (int ch = 0; ch < nch; ch++) {
      const int col = ch * 32 + lane;
      int op = 0;
      if (col < nops) { const int e = nops - 1 - col; op = (opw[e >> 4] >> (2 * (e & 15))) & 3; }
      const unsigned b0 = __ballot_sync(0xffffffffu, op == 1 || op == 3), b1 = __ballot_sync(0xffffffffu, op == 1 || op == 2);
      const int i0 = i0b + __popc(b0 & lanemask_lt()), i1 = i1b + __popc(b1 & lanemask_lt());
      if (op && col >= drop_lo && col < n - drop_hi) {
        char c;
        if (op == 3) c = nt(s1[i0]);                                       // s2 has a gap: s1's base (:141-142)
        else if (op == 2) c = nt(s2[i1]);                                  // s1 has a gap: s2's base (:143-144)
        else {
          const int c1 = s1[i0] & 3, c2 = s2[i1] & 3;
          c = (c1 == c2) ? nt(c1) : (prefer == 1 ? nt(c1) : (prefer == 2 ? nt(c2) : 'N'));      // :139-150
        }
        out[col - drop_lo] = c;
      }
      i0b += __popc(b0); i1b += __popc(b1);
    }
    if (lane == 0) a.cons_len[jb] = n - drop_lo - drop_hi;
    __syncwarp();
  }
  if (errflag && lane == 0) atomicMax(&a.ctr[2], (unsigned long long)errflag);
  {
    unsigned cl = (unsigned)cells_lane;
#pragma unroll
    for (int o = 16; o; o >>= 1) cl += __shfl_xor_sync(0xffffffffu, cl, o);
    if (lane == 0 && cl) atomicAdd(&a.ctr[1], (unsigned long long)cl);
  }
}

void merge_setup(const BimSeqs &sq, const dada2b_merge_opts *opts, int num_sms, int npairs, MergeArgs &a, size_t &smem, int &grid,
                 BBuf<uint32_t> &d_ptr) {
  AlnParams &P = a.P;
  P.match = opts->match; P.mismatch = opts->mismatch; P.gap = opts->gap_p; P.hgap = opts->homo_gap_p; P.band = opts->band;
  P.homo = opts->gap_p != opts->homo_gap_p ? 1 : 0;                     // evaluate.cpp:40-46
  P.sentinel = -9999;                                                    // nwalign_endsfree.cpp:116-117
  const int maxlen = sq.maxlen, minlen = sq.minlen;
  const int lbmax = P.band < 0 ? maxlen : std::min(P.band + (maxlen - minlen), maxlen), rbmax = lbmax;
  const int Wmax = lbmax + rbmax + 1;
  const int nchunk = (((Wmax + 1) >> 1) + 31) >> 5;
  a.sq = sq;
  a.seq_bytes = (maxlen + 15) & ~15;
  a.H_words = (Wmax + 2 + 3) & ~3;
  a.ops_words = ((2 * maxlen) / 16 + 2 + 3) & ~3;
  a.mask_words = ((2 * maxlen + 31) / 32 + 2 + 3) & ~3;
  a.ptr_words = (unsigned long long)(2 * maxlen + 2) * 2 * nchunk;
  const int base_words = 2 * (a.seq_bytes / 4) + a.H_words + a.ops_words + 3 * a.mask_words;
  a.ptr_in_smem = (4 * ((size_t)base_words + a.ptr_words) * 4 <= 96 * 1024) ? 1 : 0;
  a.warp_words = base_words + (a.ptr_in_smem ? (int)a.ptr_words : 0);
  smem = (size_t)4 * a.warp_words * 4;
  if (smem > 200 * 1024) throw BErr{"dada2b: band/sequence length too large for the alignment kernel's shared memory."};
  BCK(cudaFuncSetAttribute(k_merge_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
  grid = (int)std::min<long long>((long long)num_sms * 8, std::max<long long>(1, ((long long)npairs + 3) / 4));
  if (!a.ptr_in_smem) { d_ptr.alloc((size_t)grid * 4 * a.ptr_words); a.ptr_scratch = d_ptr.p; }
  a.trim_overhang = opts->trim_overhang != 0; a.npairs = npairs; a.cons_stride = 2 * maxlen;
}

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_merge_default_opts(dada2b_merge_opts *o) {       // R/paired.R:153-155 (maxMismatch = 0), nwalign(band=-1)
  o->match = 1; o->mismatch = -64; o->gap_p = -64; o->homo_gap_p = -64; o->band = -1; o->trim_overhang = 0;
}

void dada2b_merge_free(dada2b_merge_out *o) {
  if (!o) return;
  free(o->nmatch); free(o->nmismatch); free(o->nindel); free(o->cons_concat); free(o->cons_off); free(o);
}

int dada2b_merge_pairs(int32_t nseq, const char *seq_concat, const int64_t *seq_off, int32_t npairs, const int32_t *s1_idx,
                       const int32_t *s2_idx, const int32_t *prefer, const dada2b_merge_opts *opts, int32_t device,
                       dada2b_merge_out **out, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  dada2b_merge_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!opts || !out) throw BErr{"dada2b: NULL argument."};
    *out = nullptr;
    if (npairs < 0) throw BErr{"dada2b: negative pair count."};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    int num_sms = 148;
    BCK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    BCK(cudaEventCreate(&ev0)); BCK(cudaEventCreate(&ev1));
    BCK(cudaEventRecord(ev0, s));
    long long h2d = 0, d2h = 0;
    BimSeqs sq{};
    BBuf<uint32_t> d_seq2, d_ptr; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
    upload_packed_seqs(nseq, seq_concat, seq_off, s, d_seq2, d_len, len, sq, h2d, "mergePairs alignment");
    for (int x = 0; x < npairs; x++)
      if (s1_idx[x] < 0 || s1_idx[x] >= nseq || s2_idx[x] < 0 || s2_idx[x] >= nseq) throw BErr{"dada2b: bad pair index."};
    MergeArgs a{};
    size_t smem = 0;
    int grid = 1;
    merge_setup(sq, opts, num_sms, npairs, a, smem, grid, d_ptr);
    BBuf<int32_t> d_s1, d_s2, d_pref, d_counts, d_clen; BBuf<char> d_cons; BBuf<unsigned long long> d_ctr;
    const size_t np1 = std::max(npairs, 1);
    d_s1.alloc(np1); d_s2.alloc(np1); d_pref.alloc(np1); d_counts.alloc(np1 * 3); d_clen.alloc(np1); d_cons.alloc(np1 * a.cons_stride); d_ctr.alloc(8);
    BCK(cudaMemsetAsync(d_ctr.p, 0, 64, s));
    if (npairs) {
      BCK(cudaMemcpyAsync(d_s1.p, s1_idx, (size_t)npairs * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_s2.p, s2_idx, (size_t)npairs * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_pref.p, prefer, (size_t)npairs * 4, cudaMemcpyHostToDevice, s));
      h2d += (long long)npairs * 12;
    }
    a.s1_idx = d_s1.p; a.s2_idx = d_s2.p; a.prefer = d_pref.p; a.counts = d_counts.p; a.cons = d_cons.p; a.cons_len = d_clen.p; a.ctr = d_ctr.p;
    cudaEvent_t ka = nullptr, kb = nullptr;
    BCK(cudaEventCreate(&ka)); BCK(cudaEventCreate(&kb));
    BCK(cudaEventRecord(ka, s));
    if (npairs) k_merge_pairs<<<grid, 128, smem, s>>>(a);
    BCK(cudaEventRecord(kb, s));
    std::vector<int32_t> counts((size_t)np1 * 3), clen(np1);
    std::vector<char> cons((size_t)np1 * a.cons_stride);
    unsigned long long h[8];
    if (npairs) {
      BCK(cudaMemcpyAsync(counts.data(), d_counts.p, (size_t)npairs * 12, cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(clen.data(), d_clen.p, (size_t)npairs * 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(cons.data(), d_cons.p, (size_t)npairs * a.cons_stride, cudaMemcpyDeviceToHost, s));
      d2h += (long long)npairs * (16 + a.cons_stride);
    }
    BCK(cudaMemcpyAsync(h, d_ctr.p, sizeof h, cudaMemcpyDeviceToHost, s));
    BCK(cudaEventRecord(ev1, s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    if (h[2]) throw BErr{"N-W Align out of range."};                     // nwalign_endsfree.cpp:184
    res = (dada2b_merge_out *)calloc(1, sizeof(dada2b_merge_out));
    res->npairs = npairs;
    res->nmatch = (int32_t *)malloc(np1 * 4); res->nmismatch = (int32_t *)malloc(np1 * 4); res->nindel = (int32_t *)malloc(np1 * 4);
    res->cons_off = (int64_t *)malloc(((size_t)npairs + 1) * 8);
    int64_t tot = 0;
    for (int x = 0; x < npairs; x++) { res->cons_off[x] = tot; tot += clen[x]; }
    res->cons_off[npairs] = tot;
    res->cons_concat = (char *)malloc((size_t)std::max<int64_t>(tot, 1));
    for (int x = 0; x < npairs; x++) {
      res->nmatch[x] = counts[3 * (size_t)x]; res->nmismatch[x] = counts[3 * (size_t)x + 1]; res->nindel[x] = counts[3 * (size_t)x + 2];
      memcpy(res->cons_concat + res->cons_off[x], cons.data() + (size_t)x * a.cons_stride, (size_t)clen[x]);
    }
    float ms = 0;
    BCK(cudaEventElapsedTime(&ms, ka, kb)); res->ms_k_merge = ms;
    BCK(cudaEventElapsedTime(&ms, ev0, ev1)); res->ms_device = ms;
    cudaEventDestroy(ka); cudaEventDestroy(kb);
    res->n_cells = (int64_t)h[1]; res->gpu_launches = npairs ? 1 : 0; res->h2d_bytes = h2d; res->d2h_bytes = d2h + 64;
    res->ms_total = bnow_ms() - t0;
    *out = res;
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  if (s) cudaStreamDestroy(s);
  if (rc) { if (res) dada2b_merge_free(res); if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str()); }
  return rc;
}

}  // extern "C"
