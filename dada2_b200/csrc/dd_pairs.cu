// mergePairs over whole samples on the H100 (include/dada2b_merge.h: dada2b_merge_samples).  Product code.
//
// Replaces the per-sample R of mergePairs (/root/reference/R/paired.R:111-197) around the fused alignment of dd_merge.cu.
// Per batch of whole samples (integer work, HBM-bound; one host synchronisation per batch to learn its pairing count):
//   k_pp_key      read j -> (rF, rR) = (dadaF$map[mapF[j]], dadaR$map[mapR[j]]), NA propagating; key = (batch-local forward
//                 cluster, which also encodes the sample; rR - 1); reads with an NA get a sentinel key that sorts last
//   radix sort    stable LSD sort of the read indices by the key, only as many byte digits as the batch's sizes need: each
//                 (sample, forward, reverse) becomes one segment whose head is the pairing's first read (unique()'s row order)
//   k_pp_heads    segment heads (sentinel keys start none); exclusive scan -> pairing ids
//   k_pp_segs     per pairing: start, read count, first read, sample
//   radix sort    of the pairings by first read, then stably by descending count, then stably by sample: R's
//                 order(abundance, decreasing = TRUE) over unique()'s rows, sample by sample
//   k_pp_out      per ordered pairing: sample, forward, reverse (1-based within the sample), abundance, prefer = 1 + (n0R > n0F)
// Then once over all batches: the host gives cluster sequences global ids by content and keeps one alignment per distinct
// (forward sequence, reverse sequence, prefer); k_pp_rc reverse-complements the reverse sequences in their 2-bit rows and
// k_merge_pairs (dd_merge.cu) aligns / evaluates / builds the consensus of each distinct triple once (k_pp_concat writes
// justConcatenate's F + 10 N + rc(R) instead).  The host scatters the results back to the pairings and applies the accept rule.
#include "dd_merge.cuh"
#include "dd_sort.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>

namespace dd2 {

// largest s with off[s] <= x: the sample holding element x (samples with empty ranges are skipped)
__device__ __forceinline__ int pp_sample(const long long *off, int S, long long x) {
  int lo = 0, hi = S - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (off[mid] <= x) lo = mid; else hi = mid - 1; }
  return lo;
}

struct PpBatch {
  unsigned n; int S;                           // reads and samples of the batch
  const long long *roff;                       // [S + 1] batch-local read offsets
  const int32_t *mapF, *mapR;                  // [n] derep maps of the batch's reads
  const long long *uoffF, *uoffR;              // [S] offsets of the samples' dada maps in dmapF / dmapR
  const int32_t *dmapF, *dmapR;
  const uint32_t *kbase;                       // [S] batch-local first forward cluster of each sample
  const long long *coffF, *coffR;              // [S] offsets of the samples' clusters in n0F / n0R
  const int32_t *n0F, *n0R;
  uint32_t sentinel;                           // forward clusters in the batch: the key of reads with an NA
  uint32_t *keys;                              // [n][2] (forward, reverse)
  const uint32_t *idx, *head, *seg;            // sorted read order, segment heads, exclusive scan of the heads
  unsigned npair;
  uint32_t *u_start, *u_first, *u_count, *u_ncount, *u_samp;
  const uint32_t *order;                       // pairings in output order
  int32_t *o_samp, *o_fwd, *o_rev, *o_abund, *o_pref;
  unsigned *nvalid;                            // [1] reads where both clusters are known
};

__global__ void __launch_bounds__(256) k_pp_key(PpBatch a) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  if (j < a.n) {
    const int s = pp_sample(a.roff, a.S, j);
    const int32_t mf = a.mapF[j], mr = a.mapR[j];
    const int32_t rF = mf == INT32_MIN ? INT32_MIN : a.dmapF[a.uoffF[s] + mf - 1];      // dadaF$map[mapF]: NA propagates
    const int32_t rR = mr == INT32_MIN ? INT32_MIN : a.dmapR[a.uoffR[s] + mr - 1];
    ok = rF != INT32_MIN && rR != INT32_MIN;
    uint32_t *k = a.keys + 2 * (size_t)j;
    k[0] = ok ? a.kbase[s] + (uint32_t)(rF - 1) : a.sentinel;
    k[1] = ok ? (uint32_t)(rR - 1) : 0u;
  }
  const unsigned b = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(a.nvalid, (unsigned)__popc(b));
}

__global__ void __launch_bounds__(256) k_pp_heads(PpBatch a, uint32_t *head) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n) return;
  const uint32_t *k = a.keys + 2 * (size_t)a.idx[p];
  uint32_t h;
  if (k[0] == a.sentinel) h = 0;
  else if (p == 0) h = 1;
  else { const uint32_t *q = a.keys + 2 * (size_t)a.idx[p - 1]; h = (k[0] != q[0]) | (k[1] != q[1]); }
  head[p] = h;
}

__global__ void __launch_bounds__(256) k_pp_starts(PpBatch a) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < a.n && a.head[p]) a.u_start[a.seg[p]] = p;
}

__global__ void __launch_bounds__(256) k_pp_segs(PpBatch a) {
  const unsigned u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= a.npair) return;
  const unsigned p0 = a.u_start[u], p1 = u + 1 < a.npair ? a.u_start[u + 1] : *a.nvalid;
  const uint32_t first = a.idx[p0];                              // stable sort: the segment's head is its first read
  a.u_first[u] = first; a.u_count[u] = p1 - p0; a.u_ncount[u] = a.n - (p1 - p0);
  a.u_samp[u] = (uint32_t)pp_sample(a.roff, a.S, first);
}

__global__ void __launch_bounds__(256) k_pp_out(PpBatch a) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.npair) return;
  const uint32_t u = a.order[p];
  const int s = (int)a.u_samp[u];
  const uint32_t *k = a.keys + 2 * (size_t)a.idx[a.u_start[u]];
  const int32_t f = (int32_t)(k[0] - a.kbase[s]) + 1, r = (int32_t)k[1] + 1;
  a.o_samp[p] = s; a.o_fwd[p] = f; a.o_rev[p] = r; a.o_abund[p] = (int32_t)a.u_count[u];
  a.o_pref[p] = 1 + (a.n0R[a.coffR[s] + r - 1] > a.n0F[a.coffF[s] + f - 1]);           // paired.R:165
}

// rows [nF, n) of the 2-bit pool reverse-complemented (rc(), paired.R:139); rows below nF copied.  One thread per word.
__global__ void __launch_bounds__(256) k_pp_rc(const uint32_t *in, const uint16_t *len, int n, int nF, int SW, uint32_t *out) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)n * SW) return;
  const int r = (int)(t / SW), w = (int)(t % SW);
  const uint32_t *row = in + (size_t)r * SW;
  if (r < nF) { out[t] = row[w]; return; }
  const int L = len[r];
  uint32_t acc = 0;
  for (int b = 0; b < 16; b++) {
    const int p = 16 * w + b;
    if (p >= L) break;
    const int q = L - 1 - p;
    acc |= (3u - ((row[q >> 4] >> (2 * (q & 15))) & 3u)) << (2 * b);
  }
  out[t] = acc;
}

// justConcatenate (paired.R:140-148): F + "NNNNNNNNNN" + rc(R), one warp per distinct pair, lanes over characters
__global__ void __launch_bounds__(128) k_pp_concat(BimSeqs sq, const int32_t *s1, const int32_t *s2, int npairs, char *cons, int stride,
                                                   int32_t *cons_len) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= npairs) return;
  const int a = s1[gw], b = s2[gw], la = sq.len[a], lb = sq.len[b], n = la + 10 + lb;
  char *o = cons + (size_t)gw * stride;
  for (int c = lane; c < n; c += 32) {
    int r = -1, p = 0;
    if (c < la) { r = a; p = c; } else if (c >= la + 10) { r = b; p = c - la - 10; }
    o[c] = r < 0 ? 'N' : "ACGT"[(sq.seq2[(size_t)r * sq.SW + (p >> 4)] >> (2 * (p & 15))) & 3u];
  }
  if (lane == 0) cons_len[gw] = n;
}

static int nbytes_for(unsigned long long maxval) {     // byte digits an LSD pass needs for keys in [0, maxval]
  int b = 1;
  while (b < 4 && (maxval >> (8 * b))) b++;
  return b;
}

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_merge_samples_free(dada2b_pairs_out *o) {
  if (!o) return;
  free(o->pair_off); free(o->forward); free(o->reverse); free(o->abundance); free(o->nmatch); free(o->nmismatch); free(o->nindel);
  free(o->prefer); free(o->accept); free(o->cons_concat); free(o->cons_off); free(o);
}

int dada2b_merge_samples(const dada2b_pairs_in *in, const dada2b_pairs_opts *opts, int32_t device, dada2b_pairs_out **out,
                         char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ka = nullptr, kb = nullptr;
  dada2b_pairs_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!in || !opts || !out) throw BErr{"dada2b: NULL argument."};
    *out = nullptr;
    const int S = in->nsamples;
    if (S <= 0) throw BErr{"dada2b: no samples to merge."};
    if (!in->nreadsF || !in->nreadsR || !in->nuniqF || !in->nuniqR || !in->nclustF || !in->nclustR || !in->seqF_off || !in->seqR_off)
      throw BErr{"dada2b: NULL argument."};
    if (opts->align.band != -1) throw BErr{"dada2b: mergePairs aligns unbanded (band = -1)."};
    // ---- host checks, before any launch: paired.R:116-119, and the maps' ranges ----
    std::vector<long long> roffF(S + 1, 0), roffR(S + 1, 0), uoffF(S + 1, 0), uoffR(S + 1, 0), coffF(S + 1, 0), coffR(S + 1, 0);
    for (int k = 0; k < S; k++) {
      if (in->nreadsF[k] < 0 || in->nreadsR[k] < 0 || in->nuniqF[k] < 0 || in->nuniqR[k] < 0 || in->nclustF[k] < 0 || in->nclustR[k] < 0)
        throw BErr{"dada2b: negative sample size."};
      roffF[k + 1] = roffF[k] + in->nreadsF[k]; roffR[k + 1] = roffR[k] + in->nreadsR[k];
      uoffF[k + 1] = uoffF[k] + in->nuniqF[k]; uoffR[k + 1] = uoffR[k] + in->nuniqR[k];
      coffF[k + 1] = coffF[k] + in->nclustF[k]; coffR[k + 1] = coffR[k] + in->nclustR[k];
    }
    auto map_max = [](const int32_t *m, long long b, long long e) {      // max(map, na.rm = TRUE); -1 stands for -Inf
      long long mx = -1;
      for (long long i = b; i < e; i++) {
        if (m[i] == INT32_MIN) continue;
        if (m[i] < 1) throw BErr{"derep$map entries must be 1-based indices or NA."};
        mx = std::max<long long>(mx, m[i]);
      }
      return mx;
    };
    for (int k = 0; k < S; k++) {
      if (in->nreadsF[k] != in->nreadsR[k] || map_max(in->mapF, roffF[k], roffF[k + 1]) != in->nuniqF[k] ||
          map_max(in->mapR, roffR[k], roffR[k + 1]) != in->nuniqR[k])
        throw BErr{"Non-corresponding derep-class and dada-class objects."};
      for (long long i = uoffF[k]; i < uoffF[k + 1]; i++)
        if (in->dmapF[i] != INT32_MIN && (in->dmapF[i] < 1 || in->dmapF[i] > in->nclustF[k])) throw BErr{"dada$map entries must index the sample's clusters (1-based) or be NA."};
      for (long long i = uoffR[k]; i < uoffR[k + 1]; i++)
        if (in->dmapR[i] != INT32_MIN && (in->dmapR[i] < 1 || in->dmapR[i] > in->nclustR[k])) throw BErr{"dada$map entries must index the sample's clusters (1-based) or be NA."};
    }
    const long long NR = roffF[S], NCF = coffF[S], NCR = coffR[S];
    if (NCF >= (1LL << 30) || NCR >= (1LL << 30)) throw BErr{"dada2b: too many clusters."};
    // cluster sequences: A/C/G/T (nwalign, R/misc.R:186-188), global ids by content
    std::unordered_map<std::string, int32_t> idF, idR;
    std::vector<int32_t> gidF(NCF), gidR(NCR);
    std::vector<std::string> useqF, useqR;
    auto ids = [](const char *cat, const int64_t *off, long long n, std::unordered_map<std::string, int32_t> &id, std::vector<int32_t> &gid,
                  std::vector<std::string> &useq) {
      for (long long c = 0; c < n; c++) {
        const long long l = off[c + 1] - off[c];
        if (l <= 0 || l >= 9999) throw BErr{"dada2b: cluster sequences must have 1 to 9998 bases."};
        std::string q(cat + off[c], (size_t)l);
        for (char ch : q) if (ch != 'A' && ch != 'C' && ch != 'G' && ch != 'T') throw BErr{"Sequences must contain only A/C/G/T characters."};
        auto it = id.emplace(q, (int32_t)useq.size());
        if (it.second) useq.push_back(std::move(q));
        gid[c] = it.first->second;
      }
    };
    ids(in->seqF, in->seqF_off, NCF, idF, gidF, useqF);
    ids(in->seqR, in->seqR_off, NCR, idR, gidR, useqR);

    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
    BCK(cudaSetDevice(device));
    int num_sms = 148;
    BCK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    BCK(cudaEventCreate(&ka)); BCK(cudaEventCreate(&kb));
    long long h2d = 0, d2h = 0, nbatch = 0;
    double ms_tab = 0;
    Sorter so; so.s = s;
    // dada maps and n0 of all samples stay on the device for every batch
    BBuf<int32_t> d_dmapF, d_dmapR, d_n0F, d_n0R;
    d_dmapF.alloc(std::max<long long>(uoffF[S], 1)); d_dmapR.alloc(std::max<long long>(uoffR[S], 1));
    d_n0F.alloc(std::max<long long>(NCF, 1)); d_n0R.alloc(std::max<long long>(NCR, 1));
    if (uoffF[S]) BCK(cudaMemcpyAsync(d_dmapF.p, in->dmapF, uoffF[S] * 4, cudaMemcpyHostToDevice, s));
    if (uoffR[S]) BCK(cudaMemcpyAsync(d_dmapR.p, in->dmapR, uoffR[S] * 4, cudaMemcpyHostToDevice, s));
    if (NCF) BCK(cudaMemcpyAsync(d_n0F.p, in->n0F, NCF * 4, cudaMemcpyHostToDevice, s));
    if (NCR) BCK(cudaMemcpyAsync(d_n0R.p, in->n0R, NCR * 4, cudaMemcpyHostToDevice, s));
    h2d += 4 * (uoffF[S] + uoffR[S] + NCF + NCR);
    // ---- batches of whole samples ----
    long long cap = 1LL << 25;
    if (const char *e = getenv("DADA2B_PAIRS_BATCH")) cap = std::max(1LL, atoll(e));      // test hook: several batches on small inputs
    long long maxb = 0;
    std::vector<std::pair<int, int>> batches;
    for (int k0 = 0; k0 < S;) {
      int k1 = k0 + 1;
      while (k1 < S && roffF[k1 + 1] - roffF[k0] <= cap) k1++;
      batches.push_back({k0, k1});
      maxb = std::max(maxb, roffF[k1] - roffF[k0]);
      k0 = k1;
    }
    if (maxb >= (long long)UINT32_MAX - 1) throw BErr{"dada2b: a sample has too many reads."};
    const size_t mb = (size_t)std::max(maxb, 1LL);
    BBuf<int32_t> d_mapF, d_mapR; BBuf<uint32_t> d_keys, d_idx, d_idx2, d_head, d_seg, d_kbase; BBuf<unsigned> d_nvalid;
    BBuf<long long> d_roff, d_uoffF, d_uoffR, d_coffF, d_coffR;
    d_mapF.alloc(mb); d_mapR.alloc(mb); d_keys.alloc(2 * mb); d_idx.alloc(mb); d_idx2.alloc(mb); d_head.alloc(mb); d_seg.alloc(mb);
    d_kbase.alloc(S); d_nvalid.alloc(1); d_roff.alloc(S + 1); d_uoffF.alloc(S); d_uoffR.alloc(S); d_coffF.alloc(S); d_coffR.alloc(S);
    std::vector<int32_t> p_samp, p_fwd, p_rev, p_abund, p_pref;           // all pairings, sample by sample
    std::vector<int64_t> pair_off(S + 1, 0);
    for (auto &bt : batches) {
      const int b0 = bt.first, b1 = bt.second, SB = b1 - b0;
      const long long nb = roffF[b1] - roffF[b0];
      if (nb == 0) continue;
      const unsigned n = (unsigned)nb;
      std::vector<long long> roff(SB + 1), uf(SB), ur(SB), cf(SB), cr(SB);
      std::vector<uint32_t> kbase(SB);
      uint32_t kf = 0, maxkr = 0;
      for (int k = 0; k < SB; k++) {
        roff[k] = roffF[b0 + k] - roffF[b0]; uf[k] = uoffF[b0 + k]; ur[k] = uoffR[b0 + k]; cf[k] = coffF[b0 + k]; cr[k] = coffR[b0 + k];
        kbase[k] = kf; kf += (uint32_t)in->nclustF[b0 + k]; maxkr = std::max(maxkr, (uint32_t)in->nclustR[b0 + k]);
      }
      roff[SB] = nb;
      BCK(cudaMemcpyAsync(d_mapF.p, in->mapF + roffF[b0], nb * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_mapR.p, in->mapR + roffR[b0], nb * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_roff.p, roff.data(), (SB + 1) * 8, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_uoffF.p, uf.data(), SB * 8, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_uoffR.p, ur.data(), SB * 8, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_coffF.p, cf.data(), SB * 8, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_coffR.p, cr.data(), SB * 8, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_kbase.p, kbase.data(), SB * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemsetAsync(d_nvalid.p, 0, 4, s));
      h2d += 8 * nb + 8LL * (SB + 1) + 32LL * SB + 4LL * SB;
      PpBatch a{};
      a.n = n; a.S = SB; a.roff = d_roff.p; a.mapF = d_mapF.p; a.mapR = d_mapR.p; a.uoffF = d_uoffF.p; a.uoffR = d_uoffR.p;
      a.dmapF = d_dmapF.p; a.dmapR = d_dmapR.p; a.kbase = d_kbase.p; a.coffF = d_coffF.p; a.coffR = d_coffR.p; a.n0F = d_n0F.p; a.n0R = d_n0R.p;
      a.sentinel = kf; a.keys = d_keys.p; a.nvalid = d_nvalid.p;
      BCK(cudaEventRecord(ka, s));
      k_pp_key<<<(n + 255) / 256, 256, 0, s>>>(a);
      { uint32_t *ip = d_idx.p; k_iota<<<(n + 255) / 256, 256, 0, s>>>(ip, n); }
      so.launches += 2;
      // ---- (forward, reverse) sort: stable, so each segment's head is the pairing's first read ----
      uint32_t *x = d_idx.p, *y = d_idx2.p;
      const int nlo = nbytes_for(maxkr ? maxkr - 1 : 0), nhi = nbytes_for(kf);
      for (int by = 0; by < nlo; by++) { so.pass(RsPass{d_keys.p, 2, 1, 8 * by}, x, y, n); std::swap(x, y); }
      for (int by = 0; by < nhi; by++) { so.pass(RsPass{d_keys.p, 2, 0, 8 * by}, x, y, n); std::swap(x, y); }
      a.idx = x;
      { uint32_t *hp = d_head.p; k_pp_heads<<<(n + 255) / 256, 256, 0, s>>>(a, hp); }
      BCK(cudaMemcpyAsync(d_seg.p, d_head.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
      so.scan(d_seg.p, n);
      so.launches += 1;
      uint32_t last[2];
      BCK(cudaMemcpyAsync(&last[0], d_seg.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(&last[1], d_head.p + (n - 1), 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaEventRecord(kb, s));
      BCK(cudaStreamSynchronize(s));                                    // the batch's one host synchronisation: its pairing count
      float ms = 0;
      BCK(cudaEventElapsedTime(&ms, ka, kb)); ms_tab += ms;
      d2h += 8;
      nbatch++;
      const unsigned npair = last[0] + last[1];
      if (npair == 0) continue;
      BBuf<uint32_t> u_start, u_first, u_count, u_ncount, u_samp, ord, ord2; BBuf<int32_t> o_all;
      u_start.alloc(npair); u_first.alloc(npair); u_count.alloc(npair); u_ncount.alloc(npair); u_samp.alloc(npair);
      ord.alloc(npair); ord2.alloc(npair); o_all.alloc((size_t)5 * npair);
      a.head = d_head.p; a.seg = d_seg.p; a.npair = npair;
      a.u_start = u_start.p; a.u_first = u_first.p; a.u_count = u_count.p; a.u_ncount = u_ncount.p; a.u_samp = u_samp.p;
      BCK(cudaEventRecord(ka, s));
      k_pp_starts<<<(n + 255) / 256, 256, 0, s>>>(a);
      k_pp_segs<<<(npair + 255) / 256, 256, 0, s>>>(a);
      { uint32_t *op = ord.p; k_iota<<<(npair + 255) / 256, 256, 0, s>>>(op, npair); }
      so.launches += 3;
      // ---- order(abundance, decreasing = TRUE) over unique()'s rows, within each sample ----
      uint32_t *oa = ord.p, *ob = ord2.p;
      const int nr = nbytes_for(n), ns = nbytes_for((unsigned)(SB - 1));
      for (int by = 0; by < nr; by++) { so.pass(RsPass{u_first.p, 1, 0, 8 * by}, oa, ob, npair); std::swap(oa, ob); }
      for (int by = 0; by < nr; by++) { so.pass(RsPass{u_ncount.p, 1, 0, 8 * by}, oa, ob, npair); std::swap(oa, ob); }
      if (SB > 1) for (int by = 0; by < ns; by++) { so.pass(RsPass{u_samp.p, 1, 0, 8 * by}, oa, ob, npair); std::swap(oa, ob); }
      a.order = oa;
      a.o_samp = o_all.p; a.o_fwd = o_all.p + npair; a.o_rev = o_all.p + 2 * (size_t)npair; a.o_abund = o_all.p + 3 * (size_t)npair;
      a.o_pref = o_all.p + 4 * (size_t)npair;
      k_pp_out<<<(npair + 255) / 256, 256, 0, s>>>(a);
      so.launches += 1;
      BCK(cudaEventRecord(kb, s));
      std::vector<int32_t> h((size_t)5 * npair);
      BCK(cudaMemcpyAsync(h.data(), o_all.p, (size_t)5 * npair * 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      BCK(cudaEventElapsedTime(&ms, ka, kb)); ms_tab += ms;
      d2h += 20LL * npair;
      for (unsigned p = 0; p < npair; p++) {
        const int sg = b0 + h[p];
        pair_off[sg + 1]++;
        p_samp.push_back(sg); p_fwd.push_back(h[npair + p]); p_rev.push_back(h[2 * (size_t)npair + p]);
        p_abund.push_back(h[3 * (size_t)npair + p]); p_pref.push_back(h[4 * (size_t)npair + p]);
      }
    }
    for (int k = 0; k < S; k++) pair_off[k + 1] += pair_off[k];
    const size_t NP = p_samp.size();
    // ---- one alignment per distinct (forward sequence, reverse sequence, prefer) across all samples ----
    const bool just = opts->just_concatenate != 0;
    std::unordered_map<uint64_t, int32_t> distinct;
    std::vector<int32_t> dof(NP), d_f, d_r, d_p;
    for (size_t p = 0; p < NP; p++) {
      const int k = p_samp[p];
      const int32_t f = gidF[coffF[k] + p_fwd[p] - 1], r = gidR[coffR[k] + p_rev[p] - 1], pr = just ? 0 : p_pref[p];
      const uint64_t key = ((uint64_t)f << 32) | ((uint64_t)r << 2) | (uint64_t)pr;
      auto it = distinct.emplace(key, (int32_t)d_f.size());
      if (it.second) { d_f.push_back(f); d_r.push_back(r); d_p.push_back(pr); }
      dof[p] = it.first->second;
    }
    const int ND = (int)d_f.size();
    std::vector<int32_t> counts((size_t)3 * std::max(ND, 1), 0), clen(std::max(ND, 1), 0);
    std::vector<char> cons;
    int cons_stride = 0;
    long long cells = 0, merge_launches = 0;
    float ms_merge = 0;
    if (ND) {
      const int nF = (int)useqF.size(), nRs = (int)useqR.size(), npool = nF + nRs;
      std::vector<int64_t> poff(npool + 1, 0);
      std::string pool;
      for (int i = 0; i < npool; i++) { pool += i < nF ? useqF[i] : useqR[i - nF]; poff[i + 1] = (int64_t)pool.size(); }
      BimSeqs sq{};
      BBuf<uint32_t> d_seq2, d_rc, d_ptr; BBuf<uint16_t> d_len; std::vector<uint16_t> len;
      upload_packed_seqs(npool, pool.data(), poff.data(), s, d_seq2, d_len, len, sq, h2d, "mergePairs alignment");
      d_rc.alloc((size_t)npool * sq.SW);
      {
        const size_t words = (size_t)npool * sq.SW;
        const uint32_t *ip = d_seq2.p; const uint16_t *lp = d_len.p; uint32_t *rp = d_rc.p; const int SW = sq.SW;
        k_pp_rc<<<(unsigned)((words + 255) / 256), 256, 0, s>>>(ip, lp, npool, nF, SW, rp);
        merge_launches++;
      }
      sq.seq2 = d_rc.p;
      for (auto &r : d_r) r += nF;
      BBuf<int32_t> d_s1, d_s2, d_pref, d_counts, d_clen; BBuf<char> d_cons; BBuf<unsigned long long> d_ctr;
      d_s1.alloc(ND); d_s2.alloc(ND); d_pref.alloc(ND); d_counts.alloc((size_t)3 * ND); d_clen.alloc(ND); d_ctr.alloc(8);
      BCK(cudaMemcpyAsync(d_s1.p, d_f.data(), (size_t)ND * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_s2.p, d_r.data(), (size_t)ND * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemcpyAsync(d_pref.p, d_p.data(), (size_t)ND * 4, cudaMemcpyHostToDevice, s));
      BCK(cudaMemsetAsync(d_ctr.p, 0, 64, s));
      BCK(cudaMemsetAsync(d_counts.p, 0, (size_t)3 * ND * 4, s));
      h2d += 12LL * ND;
      BCK(cudaEventRecord(ka, s));
      if (just) {
        cons_stride = 2 * sq.maxlen + 10;
        d_cons.alloc((size_t)ND * cons_stride);
        const int32_t *s1p = d_s1.p, *s2p = d_s2.p; char *cp = d_cons.p; int32_t *lp = d_clen.p;
        k_pp_concat<<<(unsigned)(((size_t)ND * 32 + 127) / 128), 128, 0, s>>>(sq, s1p, s2p, ND, cp, cons_stride, lp);
      } else {
        MergeArgs ma{};
        size_t smem = 0;
        int grid = 1;
        merge_setup(sq, &opts->align, num_sms, ND, ma, smem, grid, d_ptr);
        d_cons.alloc((size_t)ND * ma.cons_stride);
        cons_stride = ma.cons_stride;
        ma.s1_idx = d_s1.p; ma.s2_idx = d_s2.p; ma.prefer = d_pref.p; ma.counts = d_counts.p; ma.cons = d_cons.p; ma.cons_len = d_clen.p;
        ma.ctr = d_ctr.p;
        k_merge_pairs<<<grid, 128, smem, s>>>(ma);
      }
      merge_launches++;
      BCK(cudaEventRecord(kb, s));
      cons.resize((size_t)ND * cons_stride);
      unsigned long long hc[8];
      BCK(cudaMemcpyAsync(counts.data(), d_counts.p, (size_t)ND * 12, cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(clen.data(), d_clen.p, (size_t)ND * 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(cons.data(), d_cons.p, (size_t)ND * cons_stride, cudaMemcpyDeviceToHost, s));
      BCK(cudaMemcpyAsync(hc, d_ctr.p, sizeof hc, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      BCK(cudaGetLastError());
      d2h += (long long)ND * (16 + cons_stride) + 64;
      if (hc[2]) throw BErr{"N-W Align out of range."};                  // nwalign_endsfree.cpp:184
      cells = (long long)hc[1];
      BCK(cudaEventElapsedTime(&ms_merge, ka, kb));
    }
    // ---- scatter back to the pairings: accept rule (paired.R:166), rejected sequences blanked (:177) ----
    res = (dada2b_pairs_out *)calloc(1, sizeof(dada2b_pairs_out));
    res->nsamples = S;
    const size_t np1 = std::max<size_t>(NP, 1);
    res->pair_off = (int64_t *)malloc((size_t)(S + 1) * 8);
    memcpy(res->pair_off, pair_off.data(), (size_t)(S + 1) * 8);
    res->forward = (int32_t *)malloc(np1 * 4); res->reverse = (int32_t *)malloc(np1 * 4); res->abundance = (int32_t *)malloc(np1 * 4);
    res->nmatch = (int32_t *)malloc(np1 * 4); res->nmismatch = (int32_t *)malloc(np1 * 4); res->nindel = (int32_t *)malloc(np1 * 4);
    res->prefer = (int32_t *)malloc(np1 * 4); res->accept = (uint8_t *)malloc(np1); res->cons_off = (int64_t *)malloc((np1 + 1) * 8);
    int64_t tot = 0;
    for (size_t p = 0; p < NP; p++) {
      const int d = dof[p];
      const int32_t m = counts[3 * (size_t)d], mm = counts[3 * (size_t)d + 1], id = counts[3 * (size_t)d + 2];
      const bool acc = just || (m >= opts->min_overlap && (long long)mm + id <= opts->max_mismatch);
      res->forward[p] = p_fwd[p]; res->reverse[p] = p_rev[p]; res->abundance[p] = p_abund[p];
      res->nmatch[p] = m; res->nmismatch[p] = mm; res->nindel[p] = id; res->prefer[p] = just ? 0 : p_pref[p]; res->accept[p] = acc;
      res->cons_off[p] = tot;
      if (acc) tot += clen[d];
    }
    res->cons_off[NP] = tot;
    res->cons_concat = (char *)malloc((size_t)std::max<int64_t>(tot, 1));
    for (size_t p = 0; p < NP; p++)
      if (res->cons_off[p + 1] > res->cons_off[p])
        memcpy(res->cons_concat + res->cons_off[p], cons.data() + (size_t)dof[p] * cons_stride, (size_t)(res->cons_off[p + 1] - res->cons_off[p]));
    res->n_reads = NR; res->n_pairings = (int64_t)NP; res->n_aligned = just ? 0 : ND; res->n_batches = nbatch; res->n_cells = cells;
    res->gpu_launches = so.launches + merge_launches; res->h2d_bytes = h2d; res->d2h_bytes = d2h;
    res->ms_k_tab = ms_tab; res->ms_k_merge = ms_merge; res->ms_total = bnow_ms() - t0;
    *out = res;
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  if (ka) cudaEventDestroy(ka);
  if (kb) cudaEventDestroy(kb);
  if (s) cudaStreamDestroy(s);
  if (rc) { if (res) dada2b_merge_samples_free(res); if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str()); }
  return rc;
}

}  // extern "C"
