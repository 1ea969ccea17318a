// Sample pooling on the H100 (include/dada2b_pool.h).  Product code.
//
// Replaces combineDereps2 (/root/reference/R/multiSample.R:165-203), the front door of dada(pool = TRUE).
// Pipeline (byte / integer work plus one fp64 pass, HBM-bound; stream-ordered, one host synchronisation to learn the number
// of pooled uniques), over the N sample-uniques concatenated sample by sample:
//   k_dr_pack     uniques -> MSB-first 2-bit keys (dd_sort.cuh, shared with dereplication)
//   radix sort    stable LSD sort of 0..N-1 by (key words, length): equal sequences end up adjacent, in sample order, so a
//                 segment's first member is the sequence's first-seen occurrence
//   k_dr_heads    segment heads; exclusive scan -> segment ids
//   k_pl_segs     per segment: start, first-seen position, int64 abundance sum (overflow flag), prior OR, duplicate check
//   radix sort    of the segments by first-seen position, then stably by descending count: order(derepCounts, decreasing=TRUE)
//   k_pl_qual     warp per pooled unique, lanes over positions, members in segment (= sample) order:
//                 acc = acc + q * (double)a from 0.0, then acc / count -- R's and combineDereps2's operation order, bit-exact
//   k_pl_index    sample-unique -> 1-based pooled rank; k_pl_map translates the samples' maps through it
#include "../../include/dada2b_pool.h"
#include "dd_bimera.cuh"
#include "dd_hostutil.h"
#include "dd_ctx.h"
#include "dd_sort.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace dd2 {

constexpr unsigned long long PL_BAD_NT = 1, PL_DUP = 2, PL_OVERFLOW = 4, PL_BAD_MAP = 8;   // bits of the flags word

// largest s with off[s] <= x: the sample holding element x (samples with empty ranges are skipped)
__device__ __forceinline__ int pl_sample(const long long *off, int S, long long x) {
  int lo = 0, hi = S - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (off[mid] <= x) lo = mid; else hi = mid - 1; }
  return lo;
}

struct PlSeg {
  const uint32_t *head, *seg, *idx; unsigned n, npool; int S;
  const long long *uoff; const int32_t *abund; const uint8_t *prior;
  uint32_t *u_start, *u_first, *u_count, *u_ncount; uint8_t *u_prior;
  unsigned long long *flags;
};
__global__ void __launch_bounds__(256) k_pl_starts(PlSeg a) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n || !a.head[p]) return;
  const uint32_t u = a.seg[p];
  a.u_start[u] = p; a.u_first[u] = a.idx[p];
}
__global__ void __launch_bounds__(256) k_pl_segs(PlSeg a) {
  const unsigned u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= a.npool) return;
  const unsigned p0 = a.u_start[u], p1 = u + 1 < a.npool ? a.u_start[u + 1] : a.n;
  long long sum = 0;
  uint8_t pr = 0;
  int prev_s = -1;
  for (unsigned p = p0; p < p1; p++) {
    const uint32_t m = a.idx[p];
    const int s = pl_sample(a.uoff, a.S, m);
    if (s == prev_s) atomicOr(a.flags, PL_DUP);          // a sequence twice in one sample's uniques
    prev_s = s;
    sum += a.abund[m];
    if (a.prior) pr |= (a.prior[m] != 0);
  }
  if (sum > 2147483647LL) atomicOr(a.flags, PL_OVERFLOW);
  a.u_count[u] = (uint32_t)sum; a.u_ncount[u] = ~(uint32_t)sum;    // ascending sort of ~count == descending abundance
  a.u_prior[u] = pr;
}

struct PlOut {
  const uint32_t *order, *u_start, *u_first, *u_count, *idx, *head, *seg, *rank_of; const uint8_t *u_prior;
  unsigned n, npool; int S, maxlen;
  const long long *uoff, *qoff, *moff; const int32_t *mlen, *abund, *map_in; const double *quals_in;
  int32_t *abund_out, *rep, *index, *map_out; uint8_t *prior_out; double *quals_out;
  long long nmap; unsigned long long na_bits;
  unsigned long long *flags, *qmax;   // qmax: bits of the largest non-NA pooled mean (non-negative doubles order as integers)
};
__global__ void __launch_bounds__(256) k_pl_index(PlOut a) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < a.n) a.index[a.idx[p]] = (int32_t)a.rank_of[a.seg[p] + a.head[p] - 1] + 1;
  if (p < a.npool) {
    const uint32_t u = a.order[p];
    a.abund_out[p] = (int32_t)a.u_count[u]; a.rep[p] = (int32_t)a.u_first[u]; a.prior_out[p] = a.u_prior[u];
  }
}
// combineDereps2's sweep / rowsum / sweep: one warp per pooled unique, lanes over positions, members in sample order.
__global__ void __launch_bounds__(128) k_pl_qual(PlOut a) {
  const unsigned r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= a.npool) return;
  const uint32_t u = a.order[r];
  const unsigned p0 = a.u_start[u], p1 = u + 1 < a.npool ? a.u_start[u + 1] : a.n;
  const double cnt = (double)a.u_count[u];
  const double na = __longlong_as_double((long long)a.na_bits);
  for (int p0s = 0; p0s < a.maxlen; p0s += 32) {
    const int pos = p0s + lane;
    if (pos >= a.maxlen) break;
    double acc = 0.0;
    for (unsigned p = p0; p < p1; p++) {
      const uint32_t m = a.idx[p];
      const int s = pl_sample(a.uoff, a.S, m);
      const int ml = a.mlen[s];
      const double q = pos < ml ? a.quals_in[a.qoff[s] + (m - a.uoff[s]) * (long long)ml + pos] : na;   // cbind(quals, NA)
      acc = acc + q * (double)a.abund[m];
    }
    const double mean = acc / cnt;
    a.quals_out[(size_t)r * a.maxlen + pos] = mean;
    if (mean == mean && mean > 0.0) atomicMax(a.qmax, (unsigned long long)__double_as_longlong(mean));
  }
}
// map[derep$map] then match(seq, ord)[derepMap]: NA stays NA
__global__ void __launch_bounds__(256) k_pl_map(PlOut a) {
  const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (size_t)a.nmap) return;
  const int32_t v = a.map_in[j];
  if (v == INT32_MIN) { a.map_out[j] = INT32_MIN; return; }
  const int s = pl_sample(a.moff, a.S, (long long)j);
  const long long nu = a.uoff[s + 1] - a.uoff[s];
  if (v < 1 || v > nu) { atomicOr(a.flags, PL_BAD_MAP); a.map_out[j] = INT32_MIN; return; }
  a.map_out[j] = a.index[a.uoff[s] + v - 1];
}

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_ctx_free(dada2b_ctx *ctx);       // include/dada2b.h (dd_driver.cu)

void dada2b_pool_free(dada2b_pool_out *o) {
  if (!o) return;
  free(o->seq_concat); free(o->seq_off); free(o->abund); free(o->quals); free(o->map); free(o->index); free(o->prior); free(o);
}

static int pool_impl(const dada2b_pool_in *in, int32_t device, int want_quals, dada2b_pool_out **out, dada2b_ctx **ctx_out,
                     char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  dada2b_ctx *ctx = nullptr;
  cudaStream_t s = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  dada2b_pool_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!in || !out) throw BErr{"dada2b: NULL argument."};
    *out = nullptr;
    const int S = in->nsamples;
    if (S <= 0) throw BErr{"No samples to pool."};
    if (!in->nuniq || !in->maxlen || !in->nmap || !in->seq_off || !in->seq_concat || !in->abund || !in->quals)
      throw BErr{"dada2b: NULL argument."};
    // ---- host checks and per-sample offsets ----
    std::vector<long long> uoff(S + 1, 0), qoff(S + 1, 0), moff(S + 1, 0);
    int maxlen = 0;
    for (int k = 0; k < S; k++) {
      if (in->nuniq[k] <= 0) throw BErr{"Each sample must have at least one unique sequence."};
      if (in->maxlen[k] < 0 || in->nmap[k] < 0) throw BErr{"Bad quality or map dimensions."};
      uoff[k + 1] = uoff[k] + in->nuniq[k];
      qoff[k + 1] = qoff[k] + (long long)in->nuniq[k] * in->maxlen[k];
      moff[k + 1] = moff[k] + in->nmap[k];
      maxlen = std::max(maxlen, (int)in->maxlen[k]);
    }
    const long long N64 = uoff[S], M = moff[S];
    if (N64 >= INT32_MAX) throw BErr{"Too many sequences to pool."};
    const unsigned n = (unsigned)N64;
    int seqmax = 0, seqmin = INT32_MAX;
    for (int k = 0; k < S; k++)
      for (long long i = uoff[k]; i < uoff[k + 1]; i++) {
        const long long l = in->seq_off[i + 1] - in->seq_off[i];
        if (l < 0) throw BErr{"Bad sequence offsets."};
        if (l == 0) throw BErr{"Empty unique sequences cannot be pooled."};
        if (l >= 9999) throw BErr{"Input sequences exceed the maximum allowed string length."};
        if (l > in->maxlen[k]) throw BErr{"derep$quals matrices must have as many columns as the length of the derep$unique sequences."};
        seqmax = std::max(seqmax, (int)l); seqmin = std::min(seqmin, (int)l);
      }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
    const int KW = (seqmax + 15) / 16, SK = KW + 1;
    const long long o0 = in->seq_off[0], nbytes = in->seq_off[n] - o0;
    std::vector<long long> off((size_t)n + 1);
    for (unsigned r = 0; r <= n; r++) off[r] = in->seq_off[r] - o0;
    std::vector<int32_t> mlen(in->maxlen, in->maxlen + S);
    long long h2d = 0, d2h = 0;
    BBuf<char> d_seq; BBuf<long long> d_off, d_uoff, d_qoff, d_moff; BBuf<int32_t> d_abund, d_map, d_mlen; BBuf<double> d_qin;
    BBuf<uint8_t> d_prior; BBuf<uint32_t> d_keys, d_idx, d_idx2, d_head, d_seg; BBuf<unsigned long long> d_flags, d_qmax;
    d_seq.alloc(std::max<long long>(nbytes, 1)); d_off.alloc((size_t)n + 1); d_uoff.alloc(S + 1); d_qoff.alloc(S + 1); d_moff.alloc(S + 1);
    d_abund.alloc(n); d_map.alloc(std::max<long long>(M, 1)); d_mlen.alloc(S); d_qin.alloc(std::max<long long>(qoff[S], 1));
    if (in->prior) d_prior.alloc(n);
    d_keys.alloc((size_t)n * SK); d_idx.alloc(n); d_idx2.alloc(n); d_head.alloc(n); d_seg.alloc(n); d_flags.alloc(1); d_qmax.alloc(1);
    BCK(cudaEventRecord(ev[0], s));
    BCK(cudaMemcpyAsync(d_seq.p, in->seq_concat + o0, nbytes, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_off.p, off.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_uoff.p, uoff.data(), (size_t)(S + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_qoff.p, qoff.data(), (size_t)(S + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_moff.p, moff.data(), (size_t)(S + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_mlen.p, mlen.data(), (size_t)S * 4, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_abund.p, in->abund, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    if (qoff[S]) BCK(cudaMemcpyAsync(d_qin.p, in->quals, (size_t)qoff[S] * 8, cudaMemcpyHostToDevice, s));
    if (M) BCK(cudaMemcpyAsync(d_map.p, in->map, (size_t)M * 4, cudaMemcpyHostToDevice, s));
    if (in->prior) BCK(cudaMemcpyAsync(d_prior.p, in->prior, n, cudaMemcpyHostToDevice, s));
    h2d += nbytes + ((long long)n + 1) * 8 + 3 * (S + 1) * 8LL + 4LL * S + 4LL * n + 8 * qoff[S] + 4 * M + (in->prior ? n : 0);
    BCK(cudaMemsetAsync(d_flags.p, 0, 8, s));
    BCK(cudaMemsetAsync(d_qmax.p, 0, 8, s));
    BCK(cudaEventRecord(ev[1], s));
    Sorter so; so.s = s;
    DrIn di{(int)n, KW, seqmax, d_seq.p, nullptr, d_off.p, d_keys.p, d_flags.p};
    k_dr_pack<<<(unsigned)(((size_t)n * SK + 255) / 256), 256, 0, s>>>(di);
    { uint32_t *ip = d_idx.p; k_iota<<<(n + 255) / 256, 256, 0, s>>>(ip, n); }
    so.launches += 2;
    // ---- (key, length) sort: stable, so equal sequences keep sample order ----
    uint32_t *a = d_idx.p, *b = d_idx2.p;
    for (int w = KW; w >= 0; w--) {
      const int nbyte = (w == KW) ? 2 : 4;                              // lengths < 9999 fit two bytes
      for (int by = 0; by < nbyte; by++) { so.pass(RsPass{d_keys.p, SK, w, 8 * by}, a, b, n); std::swap(a, b); }
    }
    { const uint32_t *kp = d_keys.p; uint32_t *hp = d_head.p; k_dr_heads<<<(n + 255) / 256, 256, 0, s>>>(kp, SK, a, n, hp); }
    BCK(cudaMemcpyAsync(d_seg.p, d_head.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    so.scan(d_seg.p, n);
    so.launches += 1;
    uint32_t last[2];
    unsigned long long bad = 0;
    BCK(cudaMemcpyAsync(&last[0], d_seg.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&last[1], d_head.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&bad, d_flags.p, 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));                                      // the one host synchronisation: number of pooled uniques
    if (bad & PL_BAD_NT) throw BErr{"Invalid derep$uniques vector. Sequences must be made up only of A/C/G/T."};
    const unsigned npool = last[0] + last[1];
    BBuf<uint32_t> u_start, u_first, u_count, u_ncount, ord, ord2, rank_of; BBuf<uint8_t> u_prior, o_prior;
    BBuf<int32_t> o_abund, o_rep, o_index, o_map; BBuf<double> o_quals;
    u_start.alloc(npool); u_first.alloc(npool); u_count.alloc(npool); u_ncount.alloc(npool); u_prior.alloc(npool);
    ord.alloc(npool); ord2.alloc(npool); rank_of.alloc(npool);
    o_abund.alloc(npool); o_rep.alloc(npool); o_prior.alloc(npool); o_index.alloc(n); o_map.alloc(std::max<long long>(M, 1));
    o_quals.alloc(std::max<size_t>((size_t)npool * maxlen, 1));
    PlSeg sg{d_head.p, d_seg.p, a, n, npool, S, d_uoff.p, d_abund.p, in->prior ? d_prior.p : nullptr,
             u_start.p, u_first.p, u_count.p, u_ncount.p, u_prior.p, d_flags.p};
    k_pl_starts<<<(n + 255) / 256, 256, 0, s>>>(sg);
    k_pl_segs<<<(npool + 255) / 256, 256, 0, s>>>(sg);
    { uint32_t *op = ord.p; k_iota<<<(npool + 255) / 256, 256, 0, s>>>(op, npool); }
    so.launches += 3;
    // ---- order(derepCounts, decreasing = TRUE) over the first-seen order ----
    uint32_t *oa = ord.p, *ob = ord2.p;
    for (int by = 0; by < 4; by++) { so.pass(RsPass{u_first.p, 1, 0, 8 * by}, oa, ob, npool); std::swap(oa, ob); }
    for (int by = 0; by < 4; by++) { so.pass(RsPass{u_ncount.p, 1, 0, 8 * by}, oa, ob, npool); std::swap(oa, ob); }
    union { double d; unsigned long long u; } na; na.u = 0x7FF00000000007A2ULL;     // R's NA_real_
    PlOut po{oa, u_start.p, u_first.p, u_count.p, a, d_head.p, d_seg.p, rank_of.p, u_prior.p, n, npool, S, maxlen,
             d_uoff.p, d_qoff.p, d_moff.p, d_mlen.p, d_abund.p, d_map.p, d_qin.p,
             o_abund.p, o_rep.p, o_index.p, o_map.p, o_prior.p, o_quals.p, M, na.u, d_flags.p, d_qmax.p};
    {
      uint32_t *rp = rank_of.p; const uint32_t *op = oa;
      k_dr_rank<<<(npool + 255) / 256, 256, 0, s>>>(op, npool, rp);
      k_pl_index<<<(std::max(n, npool) + 255) / 256, 256, 0, s>>>(po);
      if (maxlen > 0) k_pl_qual<<<(npool + 3) / 4, 128, 0, s>>>(po);
      so.launches += 3;
      if (M) { k_pl_map<<<(unsigned)((M + 255) / 256), 256, 0, s>>>(po); so.launches += 1; }
    }
    BCK(cudaEventRecord(ev[2], s));
    res = (dada2b_pool_out *)calloc(1, sizeof(dada2b_pool_out));
    res->npool = (int32_t)npool; res->maxlen = maxlen; res->nuniq_in = n; res->nmap = M;
    res->abund = (int32_t *)malloc((size_t)npool * 4); res->prior = (uint8_t *)malloc(npool);
    res->index = (int32_t *)malloc((size_t)n * 4); res->map = (int32_t *)malloc((size_t)std::max<long long>(M, 1) * 4);
    res->quals = want_quals ? (double *)malloc(std::max<size_t>((size_t)npool * maxlen, 1) * 8) : nullptr;
    res->seq_off = (int64_t *)malloc(((size_t)npool + 1) * 8);
    std::vector<int32_t> rep(npool);
    BCK(cudaMemcpyAsync(res->abund, o_abund.p, (size_t)npool * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->prior, o_prior.p, npool, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->index, o_index.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(rep.data(), o_rep.p, (size_t)npool * 4, cudaMemcpyDeviceToHost, s));
    if (M) BCK(cudaMemcpyAsync(res->map, o_map.p, (size_t)M * 4, cudaMemcpyDeviceToHost, s));
    if (want_quals && maxlen > 0) BCK(cudaMemcpyAsync(res->quals, o_quals.p, (size_t)npool * maxlen * 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&bad, d_flags.p, 8, cudaMemcpyDeviceToHost, s));
    unsigned long long qmax_bits = 0;
    BCK(cudaMemcpyAsync(&qmax_bits, d_qmax.p, 8, cudaMemcpyDeviceToHost, s));
    d2h += 9LL * npool + 4LL * n + 4 * M + 16 + (want_quals ? 8LL * npool * maxlen : 0);
    BCK(cudaEventRecord(ev[3], s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    if (bad & PL_DUP) throw BErr{"Duplicate sequences in the uniques of one sample."};
    if (bad & PL_OVERFLOW) throw BErr{"A pooled abundance exceeds the integer range (2^31 - 1)."};
    if (bad & PL_BAD_MAP) throw BErr{"derep$map entries must index the sample's uniques (1-based) or be NA."};
    memcpy(&res->qmax, &qmax_bits, 8);
    // the pooled sequences are the bytes of their first-seen occurrence
    int64_t tot = 0;
    for (unsigned r = 0; r < npool; r++) { res->seq_off[r] = tot; tot += in->seq_off[rep[r] + 1] - in->seq_off[rep[r]]; }
    res->seq_off[npool] = tot;
    res->seq_concat = (char *)malloc((size_t)std::max<int64_t>(tot, 1));
    for (unsigned r = 0; r < npool; r++)
      memcpy(res->seq_concat + res->seq_off[r], in->seq_concat + in->seq_off[rep[r]], (size_t)(res->seq_off[r + 1] - res->seq_off[r]));
    if (ctx_out) {
      // ---- hand the pooled uniques over to dada() on the device (dd_ctx.h), priors included ----
      if (maxlen != seqmax) throw BErr{"Sequence must have associated qualities for each nucleotide position."};   // as dada2b_run
      DevIn arrays{}; cudaStream_t cs = nullptr;
      ctx = ctx_create_device(device, (int)npool, seqmax, seqmin, res->seq_concat, res->seq_off, res->abund, &arrays, &cs);
      BBuf<unsigned long long> d_maxq; d_maxq.alloc(1);
      BCK(cudaMemsetAsync(d_maxq.p, 0, 8, cs));
      DrToCtx tc{arrays, npool, maxlen, SK, d_seq.p, d_off.p, o_rep.p, o_abund.p, o_quals.p, d_keys.p, d_maxq.p, o_prior.p};
      const size_t work = (size_t)npool * ((size_t)arrays.SW + arrays.QS);
      k_dr_to_ctx<<<(unsigned)((work + 255) / 256), 256, 0, cs>>>(tc);
      unsigned long long mq = 0;
      BCK(cudaMemcpyAsync(&mq, d_maxq.p, 8, cudaMemcpyDeviceToHost, cs));
      BCK(cudaStreamSynchronize(cs));
      BCK(cudaGetLastError());
      ctx_finish_device(ctx, (int)mq);
      so.launches += 1;
    }
    float ms = 0;
    BCK(cudaEventElapsedTime(&ms, ev[0], ev[1])); res->ms_h2d = ms;
    BCK(cudaEventElapsedTime(&ms, ev[1], ev[2])); res->ms_kernels = ms;
    BCK(cudaEventElapsedTime(&ms, ev[2], ev[3])); res->ms_d2h = ms;
    res->gpu_launches = so.launches; res->h2d_bytes = h2d; res->d2h_bytes = d2h; res->ms_total = bnow_ms() - t0;
    *out = res;
    if (ctx_out) *ctx_out = ctx;
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (auto &e : ev) if (e) cudaEventDestroy(e);
  if (s) cudaStreamDestroy(s);
  if (rc) {
    if (res) dada2b_pool_free(res);
    if (ctx) dada2b_ctx_free(ctx);
    if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  }
  return rc;
}

int dada2b_pool(const dada2b_pool_in *in, int32_t device, int32_t want_quals, dada2b_pool_out **out, char errbuf[DADA2B_ERRLEN]) {
  return pool_impl(in, device, want_quals != 0, out, nullptr, errbuf);
}
int dada2b_pool_resident(const dada2b_pool_in *in, int32_t device, int32_t want_quals, dada2b_pool_out **out, dada2b_ctx **ctx,
                         char errbuf[DADA2B_ERRLEN]) {
  if (!ctx) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "dada2b: NULL context pointer."); return 1; }
  *ctx = nullptr;
  return pool_impl(in, device, want_quals != 0, out, ctx, errbuf);
}

}  // extern "C"
