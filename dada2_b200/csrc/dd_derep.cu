// Dereplication on the H100 (include/dada2b_derep.h).  Product code.
//
// Replaces what derepFastq() computes after the fastq has been parsed (/root/reference/R/sequenceIO.R):
//   qtables2: srsort / srrank / tabulate / rowsum of the quality matrix          :150-183
//   the chunk-merging loop, the mean, order(decreasing=TRUE), the final map      :56-101
// Pipeline (byte / integer work, HBM-bound, no tensor cores; everything stream-ordered, one host synchronisation to
// learn the number of uniques):
//   k_dr_pack     reads -> MSB-first 2-bit keys (16 bases per word: integer order of the words == lexical order A<C<G<T)
//   radix sort    stable LSD sort of the read indices by (key words, length): one pass per key byte -- histogram per
//                 2048-element tile, exclusive scan of the digit-major histogram, warp-ballot ranked stable scatter;
//                 passes whose digit is constant degrade to a copy
//   k_dr_heads    a read starts a new unique when its key differs from its predecessor's; exclusive scan -> unique ids
//                 (already in srsort's lexical order); segment starts give abundances and, the sort being stable, the
//                 first read of every unique (-> its FastqStreamer chunk)
//   radix sort    of the uniques by chunk, then by descending abundance (stable: ties keep chunk, then lexical order)
//   k_dr_qsum     warp per 64 sorted reads, lanes over positions: exact integer quality sums, one atomic per run of a unique;
//   k_dr_qfinal   sums / abundance in place (NA beyond a unique's length)
//   k_dr_map      read -> 1-based rank of its unique
#include "../../include/dada2b_derep.h"
#include "dd_bimera.cuh"
#include "dd_hostutil.h"
#include "dd_ctx.h"
#include "dd_sort.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace dd2 {

__global__ void __launch_bounds__(32) k_rs_hist(RsPass p, const uint32_t *src, unsigned n, uint32_t *hist, unsigned nb) {
  __shared__ uint32_t h[256];
  const int lane = threadIdx.x;
  for (int x = lane; x < 256; x += 32) h[x] = 0;
  __syncwarp();
  const unsigned t0 = blockIdx.x * RS_TILE, t1 = min(n, t0 + RS_TILE);
  for (unsigned i = t0 + lane; i < t1; i += 32) atomicAdd(&h[rs_digit(p, src[i])], 1u);
  __syncwarp();
  for (int x = lane; x < 256; x += 32) hist[(size_t)x * nb + blockIdx.x] = h[x];       // digit-major: one scan gives global offsets
}

// Stable scatter: within a tile the elements are taken 32 at a time in order; equal digits of one round are ranked by lane.
__global__ void __launch_bounds__(32) k_rs_scatter(RsPass p, const uint32_t *src, uint32_t *dst, unsigned n, const uint32_t *offs, unsigned nb,
                                                   const uint32_t *hist_total) {
  __shared__ uint32_t base[256];
  const int lane = threadIdx.x;
  const unsigned t0 = blockIdx.x * RS_TILE, t1 = min(n, t0 + RS_TILE);
  if (hist_total[0] == n) {                       // every element has the same digit: the pass is the identity
    for (unsigned i = t0 + lane; i < t1; i += 32) dst[i] = src[i];
    return;
  }
  for (int x = lane; x < 256; x += 32) base[x] = offs[(size_t)x * nb + blockIdx.x];
  __syncwarp();
  for (unsigned r0 = t0; r0 < t1; r0 += 32) {
    const unsigned i = r0 + lane;
    const bool valid = i < t1;
    const uint32_t id = valid ? src[i] : 0u;
    const unsigned d = valid ? rs_digit(p, id) : 0u;
    unsigned m = __ballot_sync(0xffffffffu, valid);
#pragma unroll
    for (int b = 0; b < 8; b++) {
      const unsigned bb = __ballot_sync(0xffffffffu, valid && ((d >> b) & 1u));
      m &= ((d >> b) & 1u) ? bb : ~bb;
    }
    const unsigned old = valid ? base[d] : 0u;
    __syncwarp();
    if (valid && (m & ((1u << lane) - 1u)) == 0u) base[d] = old + __popc(m);          // lowest lane of each digit group
    __syncwarp();
    if (valid) dst[old + __popc(m & ((1u << lane) - 1u))] = id;
  }
}

// max over digits of the per-digit totals -> total[0] (== n when the digit is constant); offs = exclusive scan input is hist itself
__global__ void k_rs_total(const uint32_t *hist, unsigned nb, uint32_t *total) {
  __shared__ uint32_t mx;
  if (threadIdx.x == 0) mx = 0;
  __syncthreads();
  uint32_t s = 0;
  for (unsigned b = 0; b < nb; b++) s += hist[(size_t)threadIdx.x * nb + b];          // 256 threads, one digit each
  atomicMax(&mx, s);
  __syncthreads();
  if (threadIdx.x == 0) total[0] = mx;
}

// ---- exclusive scan of u32 (three kernels; in place allowed) ----
__global__ void __launch_bounds__(256) k_scan1(const uint32_t *in, uint32_t *out, uint32_t *sums, size_t n) {
  __shared__ uint32_t wtot[8];
  const size_t b0 = (size_t)blockIdx.x * 1024 + threadIdx.x * 4;
  uint32_t v[4], s = 0;
#pragma unroll
  for (int x = 0; x < 4; x++) { v[x] = (b0 + x < n) ? in[b0 + x] : 0u; s += v[x]; }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) wtot[w] = inc;
  __syncthreads();
  uint32_t wbase = 0;
  for (int x = 0; x < w; x++) wbase += wtot[x];
  uint32_t run = wbase + inc - s;
#pragma unroll
  for (int x = 0; x < 4; x++) { if (b0 + x < n) out[b0 + x] = run; run += v[x]; }
  if (threadIdx.x == 255) sums[blockIdx.x] = wbase + inc;
}
__global__ void __launch_bounds__(1024) k_scan2(uint32_t *sums, size_t nblocks) {      // single block: exclusive scan of the block sums
  __shared__ uint32_t wtot[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (size_t c0 = 0; c0 < nblocks; c0 += 1024) {
    const size_t i = c0 + threadIdx.x;
    const uint32_t v = i < nblocks ? sums[i] : 0u;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) wtot[w] = inc;
    __syncthreads();
    uint32_t wbase = 0;
    for (int x = 0; x < w; x++) wbase += wtot[x];
    const uint32_t c = carry;
    if (i < nblocks) sums[i] = c + wbase + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + wbase + inc;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(256) k_scan3(uint32_t *out, const uint32_t *sums, size_t n) {
  const size_t b0 = (size_t)blockIdx.x * 1024 + threadIdx.x * 4;
  const uint32_t a = sums[blockIdx.x];
#pragma unroll
  for (int x = 0; x < 4; x++) if (b0 + x < n) out[b0 + x] += a;
}

// ---- dereplication kernels ----
__global__ void __launch_bounds__(256) k_dr_pack(DrIn a) {
  const size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int S = a.KW + 1;
  if (x >= (size_t)a.nreads * S) return;
  const int r = (int)(x / S), w = (int)(x % S);
  const long long o = a.off[r];
  const int len = (int)(a.off[r + 1] - o);
  if (w == a.KW) { a.keys[x] = (uint32_t)len; return; }
  uint32_t k = 0;
  bool bad = false;
  for (int b = 0; b < 16; b++) {
    const int p = 16 * w + b;
    unsigned code = 0;
    if (p < len) {
      switch (a.seq[o + p]) { case 'A': code = 0; break; case 'C': code = 1; break; case 'G': code = 2; break; case 'T': code = 3; break; default: bad = true; }
    }
    k |= code << (30 - 2 * b);
  }
  a.keys[x] = k;
  if (bad) atomicMax(a.flags, 1ull);
}
__global__ void __launch_bounds__(256) k_iota(uint32_t *p, unsigned n) { const unsigned i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = i; }

// head[p] = 1 when sorted read p starts a new unique (zero-length reads, sorted first, are not uniques: head 0)
__global__ void __launch_bounds__(256) k_dr_heads(const uint32_t *keys, int S, const uint32_t *idx, unsigned n, uint32_t *head) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t *a = keys + (size_t)idx[p] * S;
  uint32_t h;
  if (a[S - 1] == 0) h = 0;
  else if (p == 0) h = 1;
  else {
    const uint32_t *b = keys + (size_t)idx[p - 1] * S;
    h = 0;
    for (int w = 0; w < S; w++) h |= (a[w] != b[w]);
  }
  head[p] = h;
}
// seg[p] = exclusive scan of head; unique u = seg[p] + head[p] - 1 for p inside a unique.  Records per-unique start, first read, chunk.
__global__ void __launch_bounds__(256) k_dr_starts(const uint32_t *head, const uint32_t *seg, const uint32_t *idx, unsigned n, long long chunk_n,
                                                   uint32_t *u_start, uint32_t *u_first, uint32_t *u_chunk) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || !head[p]) return;
  const uint32_t u = seg[p];
  u_start[u] = p; u_first[u] = idx[p];
  u_chunk[u] = chunk_n > 0 ? (uint32_t)((long long)idx[p] / chunk_n) : 0u;
}
__global__ void __launch_bounds__(256) k_dr_counts(const uint32_t *u_start, unsigned nuniq, unsigned n, uint32_t *u_count, uint32_t *u_ncount) {
  const unsigned u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= nuniq) return;
  const uint32_t c = (u + 1 < nuniq ? u_start[u + 1] : n) - u_start[u];
  u_count[u] = c; u_ncount[u] = ~c;                 // ascending sort of ~count == descending abundance
}
__global__ void __launch_bounds__(256) k_dr_rank(const uint32_t *order, unsigned nuniq, uint32_t *rank_of) {
  const unsigned r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < nuniq) rank_of[order[r]] = r;
}
// Quality sums (exact integers): a warp takes 64 consecutive sorted reads, lanes over positions; runs of the same unique are
// accumulated in a register and flushed with one 64-bit atomic per (unique, position) -- balanced however skewed the
// abundances are.  k_dr_qfinal turns the sums into means in place (rowsum / abundance, sequenceIO.R:180, :95).
struct DrOut {
  const uint32_t *order, *u_count, *u_first, *idx, *keys, *head, *seg, *rank_of; int S, maxlen; unsigned nuniq, n;
  const uint8_t *qual; const long long *off;
  unsigned long long *sums;            // [nuniq][maxlen] by output rank; becomes the double matrix in place
  int32_t *abund, *rep;
  unsigned long long na_bits;
};
__global__ void __launch_bounds__(128) k_dr_qsum(DrOut a) {
  const unsigned w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const unsigned x0 = w * 64u, x1 = min(a.n, x0 + 64u);
  if (x0 >= a.n) return;
  for (int p0 = 0; p0 < a.maxlen; p0 += 32) {
    const int pos = p0 + lane;
    unsigned long long acc = 0;
    long long cur = -1;
    for (unsigned x = x0; x < x1; x++) {
      const uint32_t id = a.idx[x];
      const int len = (int)a.keys[(size_t)id * a.S + a.S - 1];
      if (len == 0) continue;
      const long long u = (long long)a.seg[x] + a.head[x] - 1;
      if (u != cur) {
        if (cur >= 0 && acc) atomicAdd(&a.sums[(size_t)a.rank_of[cur] * a.maxlen + pos], acc);
        cur = u; acc = 0;
      }
      if (pos < len) acc += a.qual[a.off[id] + pos];
    }
    if (cur >= 0 && acc) atomicAdd(&a.sums[(size_t)a.rank_of[cur] * a.maxlen + pos], acc);
  }
}
__global__ void __launch_bounds__(256) k_dr_qfinal(DrOut a) {
  const size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= (size_t)a.nuniq * a.maxlen) return;
  const unsigned r = (unsigned)(x / a.maxlen); const int pos = (int)(x % a.maxlen);
  const uint32_t u = a.order[r], cnt = a.u_count[u];
  const int len = (int)a.keys[(size_t)a.u_first[u] * a.S + a.S - 1];
  double *q = (double *)a.sums;
  q[x] = pos < len ? (double)a.sums[x] / (double)cnt : __longlong_as_double((long long)a.na_bits);
  if (pos == 0) { a.abund[r] = (int32_t)cnt; a.rep[r] = (int32_t)a.u_first[u]; }
}
__global__ void __launch_bounds__(256) k_dr_map(const uint32_t *head, const uint32_t *seg, const uint32_t *idx, const uint32_t *keys, int S, unsigned n,
                                                const uint32_t *rank_of, int32_t *map) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t id = idx[p];
  if (keys[(size_t)id * S + S - 1] == 0) { map[id] = INT32_MIN; return; }   // zero-length read: NA (sequenceIO.R:171-175)
  map[id] = (int32_t)rank_of[seg[p] + head[p] - 1] + 1;
}

// dereplication / pooling -> dada(): fill a context's packed arrays from the device-side result
__global__ void __launch_bounds__(256) k_dr_to_ctx(DrToCtx a) {
  const size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t per = (size_t)a.in.SW + a.in.QS;
  if (x >= (size_t)a.nuniq * per) return;
  const unsigned r = (unsigned)(x / per); const int w = (int)(x % per);
  const int rd = a.rep[r];
  const int len = (int)a.keys[(size_t)rd * a.S + a.S - 1];
  if (w < a.in.SW) {                                     // 2-bit packing, 16 bases per word, base b at bits 2(b%16) (DevIn::seq2)
    uint32_t v = 0;
    const long long o = a.off[rd];
    for (int b = 0; b < 16; b++) {
      const int p = 16 * w + b;
      if (p < len) { const char c = a.seq[o + p]; v |= (uint32_t)(c == 'C' ? 1 : (c == 'G' ? 2 : (c == 'T' ? 3 : 0))) << (2 * b); }
    }
    a.in.seq2[(size_t)r * a.in.SW + w] = v;
    if (w == 0) { a.in.len[r] = (uint16_t)len; a.in.reads[r] = (uint32_t)a.abund[r]; a.in.prior[r] = a.prior ? a.prior[r] : 0; }
  } else {                                               // (uint8_t) round(mean quality), containers.cpp:34 (same rounding as do_upload)
    const int p = w - a.in.SW;
    uint8_t q = 0;
    if (p < len) {
      const double xq = a.quals[(size_t)r * a.maxlen + p];
      int rv = (int)xq;                                  // mean qualities are >= 0: trunc + (fraction >= 0.5), both exact
      if (xq - (double)rv >= 0.5) rv++;
      q = (uint8_t)rv;
      atomicMax(a.maxq, (unsigned long long)q);
    }
    a.in.qual[(size_t)r * a.in.QS + p] = q;
  }
}


void Sorter::scan(uint32_t *buf, size_t n) {
  const size_t nb = (n + 1023) / 1024;
  if (sums.n < nb) sums.alloc(nb);
  uint32_t *sp = sums.p;
  k_scan1<<<(unsigned)nb, 256, 0, s>>>(buf, buf, sp, n);
  k_scan2<<<1, 1024, 0, s>>>(sp, nb);
  k_scan3<<<(unsigned)nb, 256, 0, s>>>(buf, sp, n);
  launches += 3;
}
void Sorter::pass(const RsPass &p, const uint32_t *a, uint32_t *b, unsigned n) {
  const unsigned nb = (n + RS_TILE - 1) / RS_TILE;
  if (hist.n < (size_t)256 * nb) hist.alloc((size_t)256 * nb);
  if (!total.p) total.alloc(1);
  uint32_t *hp = hist.p, *tp = total.p;
  k_rs_hist<<<nb, 32, 0, s>>>(p, a, n, hp, nb);
  k_rs_total<<<1, 256, 0, s>>>(hp, nb, tp);
  launches += 2;
  scan(hp, (size_t)256 * nb);
  k_rs_scatter<<<nb, 32, 0, s>>>(p, a, b, n, hp, nb, tp);
  launches += 1;
}

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_ctx_free(dada2b_ctx *ctx);       // include/dada2b.h (dd_driver.cu)

void dada2b_derep_free(dada2b_derep_out *o) {
  if (!o) return;
  free(o->seq_concat); free(o->seq_off); free(o->abund); free(o->quals); free(o->map); free(o);
}

static int derep_impl(const dada2b_derep_in *in, int32_t device, dada2b_derep_out **out, dada2b_ctx **ctx_out, int want_quals, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  dada2b_ctx *ctx = nullptr;
  cudaStream_t s = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  dada2b_derep_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!in || !out) throw BErr{"dada2b: NULL argument."};
    *out = nullptr;
    const unsigned n = (unsigned)in->nreads;
    if (in->nreads <= 0) throw BErr{"Only zero-length sequences detected during dereplication."};
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
    BCK(cudaEventRecord(ev[0], s));
    int maxlen = 0; long long npos = 0;
    for (unsigned r = 0; r < n; r++) {
      const long long l = in->seq_off[r + 1] - in->seq_off[r];
      if (l < 0) throw BErr{"Bad sequence offsets."};
      if (l >= 9999) throw BErr{"Input sequences exceed the maximum allowed string length."};
      maxlen = std::max(maxlen, (int)l); npos += l > 0;
    }
    if (npos == 0) throw BErr{"Only zero-length sequences detected during dereplication."};      // sequenceIO.R:153
    const long long o0 = in->seq_off[0], nbytes = in->seq_off[n] - o0;
    const int KW = (maxlen + 15) / 16, S = KW + 1;
    long long h2d = 0, d2h = 0;
    BBuf<char> d_seq; BBuf<uint8_t> d_qual; BBuf<long long> d_off; BBuf<uint32_t> d_keys, d_idx, d_idx2, d_head, d_seg;
    BBuf<unsigned long long> d_flags;
    d_seq.alloc(std::max<long long>(nbytes, 1)); d_qual.alloc(std::max<long long>(nbytes, 1)); d_off.alloc((size_t)n + 1);
    d_keys.alloc((size_t)n * S); d_idx.alloc(n); d_idx2.alloc(n); d_head.alloc(n); d_seg.alloc(n); d_flags.alloc(1);
    std::vector<long long> off((size_t)n + 1);
    for (unsigned r = 0; r <= n; r++) off[r] = in->seq_off[r] - o0;
    BCK(cudaMemcpyAsync(d_seq.p, in->seq_concat + o0, nbytes, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_qual.p, in->qual_concat + o0, nbytes, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_off.p, off.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemsetAsync(d_flags.p, 0, 8, s));
    h2d += 2 * nbytes + ((long long)n + 1) * 8;
    Sorter so; so.s = s;
    DrIn di{(int)n, KW, maxlen, d_seq.p, d_qual.p, d_off.p, d_keys.p, d_flags.p};
    k_dr_pack<<<(unsigned)(((size_t)n * S + 255) / 256), 256, 0, s>>>(di);
    { uint32_t *ip = d_idx.p; k_iota<<<(n + 255) / 256, 256, 0, s>>>(ip, n); }
    so.launches += 2;
    BCK(cudaEventRecord(ev[1], s));
    // ---- lexical sort of the reads: LSD over (length, last key word ... first key word), one byte per pass ----
    uint32_t *a = d_idx.p, *b = d_idx2.p;
    for (int w = KW; w >= 0; w--) {
      const int nbyte = (w == KW) ? 2 : 4;                              // lengths < 9999 fit two bytes
      for (int by = 0; by < nbyte; by++) { so.pass(RsPass{d_keys.p, S, w, 8 * by}, a, b, n); std::swap(a, b); }
    }
    BCK(cudaEventRecord(ev[2], s));
    // ---- uniques ----
    { const uint32_t *kp = d_keys.p; uint32_t *hp = d_head.p; k_dr_heads<<<(n + 255) / 256, 256, 0, s>>>(kp, S, a, n, hp); }
    BCK(cudaMemcpyAsync(d_seg.p, d_head.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    so.scan(d_seg.p, n);
    so.launches += 1;
    uint32_t last[2];
    BCK(cudaMemcpyAsync(&last[0], d_seg.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&last[1], d_head.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    unsigned long long bad = 0;
    BCK(cudaMemcpyAsync(&bad, d_flags.p, 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));                                      // the one host synchronisation: number of uniques
    if (bad) throw BErr{"dada2b: dereplication needs A/C/G/T reads (2-bit packed on the device)."};
    const unsigned nuniq = last[0] + last[1];
    BBuf<uint32_t> u_start, u_first, u_chunk, u_count, u_ncount, ord, ord2, rank_of;
    BBuf<double> d_quals; BBuf<int32_t> d_abund, d_rep, d_map;
    u_start.alloc(nuniq); u_first.alloc(nuniq); u_chunk.alloc(nuniq); u_count.alloc(nuniq); u_ncount.alloc(nuniq);
    ord.alloc(nuniq); ord2.alloc(nuniq); rank_of.alloc(nuniq);
    d_quals.alloc((size_t)nuniq * maxlen); d_abund.alloc(nuniq); d_rep.alloc(nuniq); d_map.alloc(n);
    {
      const uint32_t *hp = d_head.p, *sp = d_seg.p; uint32_t *us = u_start.p, *uf = u_first.p, *uc = u_chunk.p, *un = u_count.p, *unn = u_ncount.p, *op = ord.p;
      const long long cn = in->chunk_n;
      k_dr_starts<<<(n + 255) / 256, 256, 0, s>>>(hp, sp, a, n, cn, us, uf, uc);
      k_dr_counts<<<(nuniq + 255) / 256, 256, 0, s>>>(us, nuniq, n, un, unn);
      k_iota<<<(nuniq + 255) / 256, 256, 0, s>>>(op, nuniq);
      so.launches += 3;
    }
    // zero-length reads sort first and are not part of any unique: the first unique starts after them, counts follow from starts
    uint32_t *oa = ord.p, *ob = ord2.p;                                 // stable: ties keep chunk, then lexical order (sequenceIO.R:76-98)
    for (int by = 0; by < 4; by++) { so.pass(RsPass{u_chunk.p, 1, 0, 8 * by}, oa, ob, nuniq); std::swap(oa, ob); }
    for (int by = 0; by < 4; by++) { so.pass(RsPass{u_ncount.p, 1, 0, 8 * by}, oa, ob, nuniq); std::swap(oa, ob); }
    {
      uint32_t *rp = rank_of.p;
      k_dr_rank<<<(nuniq + 255) / 256, 256, 0, s>>>(oa, nuniq, rp);
      union { double d; unsigned long long u; } na; na.u = 0x7FF00000000007A2ULL;     // R's NA_real_
      BCK(cudaMemsetAsync(d_quals.p, 0, (size_t)nuniq * maxlen * 8, s));
      DrOut dq{oa, u_count.p, u_first.p, a, d_keys.p, d_head.p, d_seg.p, rp, S, maxlen, nuniq, n, d_qual.p, d_off.p,
               (unsigned long long *)d_quals.p, d_abund.p, d_rep.p, na.u};
      k_dr_qsum<<<(unsigned)(((size_t)n + 255) / 256), 128, 0, s>>>(dq);
      k_dr_qfinal<<<(unsigned)(((size_t)nuniq * maxlen + 255) / 256), 256, 0, s>>>(dq);
      so.launches += 1;
      const uint32_t *hp = d_head.p, *sp = d_seg.p, *kp = d_keys.p; int32_t *mp = d_map.p;
      k_dr_map<<<(n + 255) / 256, 256, 0, s>>>(hp, sp, a, kp, S, n, rp, mp);
      so.launches += 3;
    }
    res = (dada2b_derep_out *)calloc(1, sizeof(dada2b_derep_out));
    res->nuniq = (int32_t)nuniq; res->maxlen = maxlen; res->nreads = in->nreads;
    res->abund = (int32_t *)malloc((size_t)nuniq * 4); res->quals = want_quals ? (double *)malloc((size_t)nuniq * maxlen * 8) : nullptr;
    res->map = (int32_t *)malloc((size_t)n * 4); res->seq_off = (int64_t *)malloc(((size_t)nuniq + 1) * 8);
    std::vector<int32_t> rep(nuniq);
    BCK(cudaMemcpyAsync(res->abund, d_abund.p, (size_t)nuniq * 4, cudaMemcpyDeviceToHost, s));
    if (want_quals) BCK(cudaMemcpyAsync(res->quals, d_quals.p, (size_t)nuniq * maxlen * 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->map, d_map.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(rep.data(), d_rep.p, (size_t)nuniq * 4, cudaMemcpyDeviceToHost, s));
    d2h += (long long)nuniq * (8 + (want_quals ? (long long)maxlen * 8 : 0)) + (long long)n * 4 + 16;
    BCK(cudaEventRecord(ev[3], s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    // the unique sequences themselves are the bytes of their first read (host copy of nuniq short strings)
    int64_t tot = 0;
    for (unsigned r = 0; r < nuniq; r++) { res->seq_off[r] = tot; tot += in->seq_off[rep[r] + 1] - in->seq_off[rep[r]]; }
    res->seq_off[nuniq] = tot;
    res->seq_concat = (char *)malloc((size_t)std::max<int64_t>(tot, 1));
    for (unsigned r = 0; r < nuniq; r++)
      memcpy(res->seq_concat + res->seq_off[r], in->seq_concat + in->seq_off[rep[r]], (size_t)(res->seq_off[r + 1] - res->seq_off[r]));
    if (ctx_out) {
      // ---- hand the uniques over to dada() on the device (dd_ctx.h): no D2H of the means, no host re-pack, no H2D ----
      int minlen = maxlen;
      for (unsigned r = 0; r < nuniq; r++) minlen = std::min<int>(minlen, (int)(res->seq_off[r + 1] - res->seq_off[r]));
      DevIn arrays{}; cudaStream_t cs = nullptr;
      ctx = ctx_create_device(device, (int)nuniq, maxlen, minlen, res->seq_concat, res->seq_off, res->abund, &arrays, &cs);
      BBuf<unsigned long long> d_maxq; d_maxq.alloc(1);
      BCK(cudaMemsetAsync(d_maxq.p, 0, 8, cs));
      DrToCtx tc{arrays, nuniq, maxlen, S, d_seq.p, d_off.p, d_rep.p, d_abund.p, d_quals.p, d_keys.p, d_maxq.p};
      const size_t work = (size_t)nuniq * ((size_t)arrays.SW + arrays.QS);
      k_dr_to_ctx<<<(unsigned)((work + 255) / 256), 256, 0, cs>>>(tc);
      unsigned long long mq = 0;
      BCK(cudaMemcpyAsync(&mq, d_maxq.p, 8, cudaMemcpyDeviceToHost, cs));
      BCK(cudaStreamSynchronize(cs));
      BCK(cudaGetLastError());
      ctx_finish_device(ctx, (int)mq);
      so.launches += 1;
    }
    float ms = 0;
    BCK(cudaEventElapsedTime(&ms, ev[1], ev[2])); res->ms_sort = ms;
    BCK(cudaEventElapsedTime(&ms, ev[0], ev[3])); res->ms_device = ms;
    res->gpu_launches = so.launches; res->h2d_bytes = h2d; res->d2h_bytes = d2h; res->ms_total = bnow_ms() - t0;
    *out = res;
    if (ctx_out) *ctx_out = ctx;
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (auto &e : ev) if (e) cudaEventDestroy(e);
  if (s) cudaStreamDestroy(s);
  if (rc) {
    if (res) dada2b_derep_free(res);
    if (ctx) dada2b_ctx_free(ctx);
    if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  }
  return rc;
}

int dada2b_derep(const dada2b_derep_in *in, int32_t device, dada2b_derep_out **out, char errbuf[DADA2B_ERRLEN]) {
  return derep_impl(in, device, out, nullptr, 1, errbuf);
}
int dada2b_derep_resident(const dada2b_derep_in *in, int32_t device, int32_t want_quals, dada2b_derep_out **out, dada2b_ctx **ctx,
                          char errbuf[DADA2B_ERRLEN]) {
  if (!ctx) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "dada2b: NULL context pointer."); return 1; }
  *ctx = nullptr;
  return derep_impl(in, device, out, ctx, want_quals != 0, errbuf);
}

}  // extern "C"
