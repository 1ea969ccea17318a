// Taxonomic classification on the H100 (include/dada2b_taxonomy.h).  Product code.
//
// Replaces C_assign_taxonomy2 (src/taxonomy.cpp:206-338).  The contract is DESIGN.md 21; every sum is a sequential fp32
// sum in the reference's order, and ties are broken by a hash of (seed, query, replicate, genus), so a result does not
// depend on the launch geometry or on how the genera are split into chunks.
// Table build (once per database, or per chunk and call when chunked):
//   k_tax_presence  one block per reference: its 8-mer presence bitmap (8 KB) in shared memory, then one atomic count
//                   per present k-mer into the k-mer-major table [65536][cpad] (and into count_k at the first build)
//   k_tax_prior     one thread per k-mer: prior_k in fp64, rounded once
//   k_tax_log       one thread per entry, in place: count -> (float)log((double)(((float)cnt + prior) / (M_g + 1)))
// Classification, per batch of queries of at least 50 nt:
//   k_tax_qkmers    one block per query: its valid 8-mers, bitonic-sorted in shared memory; the reverse complement's
//                   array from the forward k-mers (same multiset), sorted again
//   k_tax_main      one block per (query, 128 genera), a thread per genus: the forward and reverse-complement main sums,
//                   rows read straight from the table (one 512-B row segment per k-mer); block arg-max by the tie rule
//   k_tax_pick      one thread per query: arg-max over genus groups and chunks, the orientation
//   k_tax_draws     one block per query: distinct k-mers of the chosen array and the bootstrap draws as row indices
//   k_tax_boot      one block per (query, 128 genera), two threads per genus (50 bootstraps each): the rows of the
//                   query's distinct k-mers staged in shared memory (read from the table when they do not fit), the
//                   100 bootstrap sums, block arg-max per bootstrap
//   k_tax_bootpick  one thread per (query, bootstrap): arg-max over groups and chunks
//   k_tax_count     one thread per query: boot counts per level
#include "../../include/dada2b_taxonomy.h"
#include "dd_flt.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace dd2 {

constexpr int TAX_NK = 65536;                   // 4^8 k-mers
constexpr int TAX_NBOOT = DADA2B_TAX_NBOOT;
constexpr int TAX_GRP = 128;                    // genera per block of the sum kernels (tables are padded to a multiple)
constexpr int TAX_STAGE_ROWS = 416;             // distinct k-mers whose 128-genus rows (512 B each) k_tax_boot stages
constexpr unsigned TAX_NONE = 0xffffffffu;

__host__ __device__ __forceinline__ unsigned long long tax_mix(unsigned long long z) {      // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ unsigned long long tax_hash(unsigned long long jb, int r, int g) {
  return tax_mix(jb + (((unsigned long long)(unsigned)r << 32) | (unsigned)g));
}
__device__ __forceinline__ int tax_code(char c) {
  return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}
__device__ __forceinline__ unsigned tax_kmer_at(const char *s) {         // TAX_NONE unless 8 A/C/G/T letters
  unsigned km = 0;
  for (int t = 0; t < 8; t++) {
    const int c = tax_code(s[t]);
    if (c < 0) return TAX_NONE;
    km = km * 4u + (unsigned)c;
  }
  return km;
}
__device__ __forceinline__ unsigned tax_rc(unsigned km) {                 // 8-mer of the reverse complement
  unsigned c = ~km & 0xffffu, r = 0;
  for (int t = 0; t < 8; t++) { r = (r << 2) | (c & 3u); c >>= 2; }
  return r;
}

struct TaxCand { float lp; int g; };            // g < 0: no candidate

// The tie rule as a total order: larger logp, then smaller hash, then smaller genus.
__device__ __forceinline__ bool tax_better(float la, unsigned long long ha, int ga, float lb, unsigned long long hb, int gb) {
  if (ga < 0) return false;
  if (gb < 0) return true;
  if (la != lb) return la > lb;
  if (ha != hb) return ha < hb;
  return ga < gb;
}

// Warp arg-max; the winner ends in lane 0.
__device__ __forceinline__ void tax_warp_best(float &lp, unsigned long long &h, int &g) {
  for (int o = 16; o > 0; o >>= 1) {
    const float ol = __shfl_down_sync(FULL, lp, o);
    const unsigned long long oh = __shfl_down_sync(FULL, h, o);
    const int og = __shfl_down_sync(FULL, g, o);
    if (tax_better(ol, oh, og, lp, h, g)) { lp = ol; h = oh; g = og; }
  }
}

// ---- table build ----
__global__ void __launch_bounds__(256) k_tax_presence(const char *seq, const long long *off, const int *rg, int r0, int g0, int cpad,
                                                     unsigned *cnt, unsigned *ck) {
  __shared__ unsigned bm[TAX_NK / 32];
  const int r = r0 + blockIdx.x;
  for (int i = threadIdx.x; i < TAX_NK / 32; i += blockDim.x) bm[i] = 0u;
  __syncthreads();
  const long long b = off[r];
  const int L = (int)(off[r + 1] - b);
  for (int p = threadIdx.x; p + 8 <= L; p += blockDim.x) {
    const unsigned km = tax_kmer_at(seq + b + p);
    if (km != TAX_NONE) atomicOr(&bm[km >> 5], 1u << (km & 31));
  }
  __syncthreads();
  const int g = rg[r] - g0;
  for (int w = threadIdx.x; w < TAX_NK / 32; w += blockDim.x) {
    unsigned m = bm[w];
    while (m) {
      const unsigned km = (unsigned)w * 32u + (unsigned)(__ffs((int)m) - 1);
      m &= m - 1u;
      if (cnt) atomicAdd(&cnt[(size_t)km * cpad + g], 1u);
      if (ck) atomicAdd(&ck[km], 1u);
    }
  }
}

__global__ void k_tax_prior(const unsigned *ck, double nref, float *prior) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < TAX_NK) prior[k] = (float)(((double)ck[k] + 0.5) / (1.0 + nref));     // taxonomy.cpp:261
}

__global__ void k_tax_log(float *tab, const float *prior, const float *gnp1, int cn, int cpad) {
  const size_t n = (size_t)TAX_NK * cpad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % (size_t)cpad);
    const int k = (int)(i / (size_t)cpad);
    const unsigned c = ((const unsigned *)tab)[i];
    float v = 0.f;
    if (g < cn) {
      const float x = ((float)c + prior[k]) / gnp1[g];                       // taxonomy.cpp:268, float add then divide
      v = (float)log((double)x);
    }
    tab[i] = v;
  }
}

// ---- classification ----
struct TaxQ {                                   // one batch of queries
  int nq, MK;                                   // queries; stride of the per-query k-mer arrays (>= every arraylen)
  const char *seq; const long long *off;        // the batch's sequences
  const int *alen;                              // [nq] valid 8-mers
  const int *j;                                 // [nq] 0-based query index of the call (hash and draws)
  unsigned *kf, *kr, *kd;                       // [nq][MK] sorted forward / reverse-complement k-mers, distinct chosen
  int *nd;                                      // [nq] distinct k-mers of the chosen array
  unsigned short *dr;                           // [nq][DS] bootstrap draws: distinct index (staged) or k-mer
  long long DS;
};

__device__ void tax_bitonic(unsigned *a, int P) {
  for (int k = 2; k <= P; k <<= 1)
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ix = i ^ jj;
        if (ix > i) {
          const unsigned x = a[i], y = a[ix];
          if ((x > y) == ((i & k) == 0)) { a[i] = y; a[ix] = x; }
        }
      }
      __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_tax_qkmers(TaxQ q, int P, int want_rc) {
  extern __shared__ unsigned tsm[];
  const int qb = blockIdx.x;
  const long long b = q.off[qb];
  const int L = (int)(q.off[qb + 1] - b);
  const int W = L >= 8 ? L - 7 : 0;
  for (int i = threadIdx.x; i < P; i += blockDim.x) tsm[i] = i < W ? tax_kmer_at(q.seq + b + i) : TAX_NONE;
  __syncthreads();
  tax_bitonic(tsm, P);
  const int n = q.alen[qb];
  unsigned *kf = q.kf + (size_t)qb * q.MK;
  for (int i = threadIdx.x; i < n; i += blockDim.x) kf[i] = tsm[i];
  if (!want_rc) return;
  for (int i = threadIdx.x; i < P; i += blockDim.x) tsm[i] = i < n ? tax_rc(tsm[i]) : TAX_NONE;
  __syncthreads();
  tax_bitonic(tsm, P);
  unsigned *kr = q.kr + (size_t)qb * q.MK;
  for (int i = threadIdx.x; i < n; i += blockDim.x) kr[i] = tsm[i];
}

struct TaxChunk {                               // the resident table of one chunk of genera
  const float *tab; int cpad, cn, g0, grp0;     // padded width, genera, first genus, first global 128-genus group
};

__global__ void __launch_bounds__(TAX_GRP) k_tax_main(TaxQ q, TaxChunk c, int ngrp, int try_rc, unsigned long long seed, TaxCand *cand,
                                                      float *dump, int ngenus) {
  __shared__ TaxCand rb[2][TAX_GRP / 32];
  __shared__ unsigned long long rh[2][TAX_GRP / 32];
  const int qb = blockIdx.y, grp = blockIdx.x;
  const int gc = grp * TAX_GRP + threadIdx.x;
  const bool live = gc < c.cn;
  const float *col = c.tab + gc;
  const int n = q.alen[qb];
  const int no = try_rc ? 2 : 1;
  const unsigned long long jb = tax_mix(tax_mix(seed) + (unsigned long long)q.j[qb]);
  const int g = c.g0 + gc;
  for (int o = 0; o < no; o++) {
    const unsigned *a = (o ? q.kr : q.kf) + (size_t)qb * q.MK;
    float s = 0.f;
#pragma unroll 8
    for (int p = 0; p < n; p++) s += col[(size_t)a[p] * c.cpad];
    if (dump && live) dump[((size_t)qb * 2 + o) * ngenus + g] = s;
    float lp = live ? s : -INFINITY;
    int gg = live ? g : -1;
    unsigned long long h = live ? tax_hash(jb, TAX_NBOOT + o, g) : 0ull;
    tax_warp_best(lp, h, gg);
    if ((threadIdx.x & 31) == 0) { rb[o][threadIdx.x >> 5] = TaxCand{lp, gg}; rh[o][threadIdx.x >> 5] = h; }
  }
  __syncthreads();
  if (threadIdx.x < no) {
    const int o = threadIdx.x;
    TaxCand best = rb[o][0];
    unsigned long long bh = rh[o][0];
    for (int w = 1; w < TAX_GRP / 32; w++)
      if (tax_better(rb[o][w].lp, rh[o][w], rb[o][w].g, best.lp, bh, best.g)) { best = rb[o][w]; bh = rh[o][w]; }
    cand[((size_t)qb * ngrp + c.grp0 + grp) * 2 + o] = best;
  }
}

__global__ void k_tax_pick(TaxQ q, int ngrp, int try_rc, unsigned long long seed, const TaxCand *cand, int *best_g, float *best_lp,
                           unsigned char *used) {
  const int qb = blockIdx.x * blockDim.x + threadIdx.x;
  if (qb >= q.nq) return;
  const unsigned long long jb = tax_mix(tax_mix(seed) + (unsigned long long)q.j[qb]);
  TaxCand b[2] = {{0.f, -1}, {0.f, -1}};
  unsigned long long bh[2] = {0ull, 0ull};
  for (int o = 0; o < (try_rc ? 2 : 1); o++)
    for (int grp = 0; grp < ngrp; grp++) {
      const TaxCand x = cand[((size_t)qb * ngrp + grp) * 2 + o];
      if (x.g < 0) continue;
      const unsigned long long h = tax_hash(jb, TAX_NBOOT + o, x.g);
      if (tax_better(x.lp, h, x.g, b[o].lp, bh[o], b[o].g)) { b[o] = x; bh[o] = h; }
    }
  const int u = try_rc && b[1].lp > b[0].lp ? 1 : 0;                   // taxonomy.cpp:173, strictly better
  best_g[qb] = b[u].g; best_lp[qb] = b[u].lp; used[qb] = (unsigned char)u;
}

__global__ void __launch_bounds__(256) k_tax_draws(TaxQ q, const unsigned char *used, const double *unifs, long long mal,
                                                   unsigned long long seed) {
  extern __shared__ unsigned dix[];             // [MK] distinct index of each position
  __shared__ unsigned part[256];
  const int qb = blockIdx.x, t = threadIdx.x;
  const unsigned *a = (used[qb] ? q.kr : q.kf) + (size_t)qb * q.MK;
  const int n = q.alen[qb];
  const int chunk = (n + 255) / 256;
  const int p0 = min(n, t * chunk), p1 = min(n, p0 + chunk);
  unsigned c = 0;
  for (int p = p0; p < p1; p++) c += (p == 0 || a[p] != a[p - 1]) ? 1u : 0u;
  part[t] = c;
  __syncthreads();
  for (int o = 1; o < 256; o <<= 1) {           // inclusive Hillis-Steele scan
    const unsigned v = t >= o ? part[t - o] : 0u;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  unsigned d = part[t] - c;
  unsigned *kd = q.kd + (size_t)qb * q.MK;
  for (int p = p0; p < p1; p++) {
    if (p == 0 || a[p] != a[p - 1]) { kd[d] = a[p]; d++; }
    dix[p] = d - 1u;
  }
  const int nd = (int)part[255];
  if (t == 0) q.nd[qb] = nd;
  __syncthreads();
  const bool staged = nd <= TAX_STAGE_ROWS;
  const int n8 = n / 8;
  const long long base = (long long)q.j[qb] * mal;
  const unsigned long long sb = tax_mix(seed ^ 0x9E3779B97F4A7C15ull);
  unsigned short *dr = q.dr + (size_t)qb * q.DS;
  for (int idx = t; idx < TAX_NBOOT * n8; idx += blockDim.x) {
    const double u = unifs ? unifs[base + idx] : (double)(tax_mix(sb + (unsigned long long)(base + idx)) >> 11) * 0x1.0p-53;
    int pos = (int)((double)n * u);             // taxonomy.cpp:185, the product in double, truncated
    pos = min(max(pos, 0), n - 1);
    dr[idx] = (unsigned short)(staged ? dix[pos] : a[pos]);
  }
}

__global__ void __launch_bounds__(256) k_tax_boot(TaxQ q, TaxChunk c, int ngrp, unsigned long long seed, TaxCand *cand) {
  extern __shared__ float rows[];               // [nd][128] when staged
  __shared__ TaxCand rb[TAX_NBOOT][TAX_GRP / 32];
  __shared__ unsigned long long rh[TAX_NBOOT][TAX_GRP / 32];
  const int qb = blockIdx.y, grp = blockIdx.x;
  const int gl = threadIdx.x & (TAX_GRP - 1), half = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3;
  const int gc = grp * TAX_GRP + gl;
  const bool live = gc < c.cn;
  const int n8 = q.alen[qb] / 8, nd = q.nd[qb];
  const bool staged = nd <= TAX_STAGE_ROWS;
  if (staged) {
    const unsigned *kd = q.kd + (size_t)qb * q.MK;
    const float *tg = c.tab + grp * TAX_GRP;
    for (int i = threadIdx.x; i < nd * TAX_GRP; i += blockDim.x)
      rows[i] = tg[(size_t)kd[i >> 7] * c.cpad + (i & (TAX_GRP - 1))];
  }
  __syncthreads();
  const float *base = staged ? rows + gl : c.tab + gc;
  const size_t stride = staged ? (size_t)TAX_GRP : (size_t)c.cpad;
  const unsigned short *dq = q.dr + (size_t)qb * q.DS;
  const unsigned long long jb = tax_mix(tax_mix(seed) + (unsigned long long)q.j[qb]);
  const int g = c.g0 + gc;
  for (int bt = half * (TAX_NBOOT / 2); bt < (half + 1) * (TAX_NBOOT / 2); bt++) {
    const unsigned short *d = dq + (size_t)bt * n8;
    float s = 0.f;
#pragma unroll 8
    for (int i = 0; i < n8; i++) s += base[(size_t)d[i] * stride];
    float lp = live ? s : -INFINITY;
    int gg = live ? g : -1;
    unsigned long long h = live ? tax_hash(jb, bt, g) : 0ull;
    tax_warp_best(lp, h, gg);
    if ((threadIdx.x & 31) == 0) { rb[bt][w] = TaxCand{lp, gg}; rh[bt][w] = h; }
  }
  __syncthreads();
  if (threadIdx.x < TAX_NBOOT) {
    const int bt = threadIdx.x;
    TaxCand best = rb[bt][0];
    unsigned long long bh = rh[bt][0];
    for (int v = 1; v < TAX_GRP / 32; v++)
      if (tax_better(rb[bt][v].lp, rh[bt][v], rb[bt][v].g, best.lp, bh, best.g)) { best = rb[bt][v]; bh = rh[bt][v]; }
    cand[((size_t)qb * ngrp + c.grp0 + grp) * TAX_NBOOT + bt] = best;
  }
}

__global__ void k_tax_bootpick(TaxQ q, int ngrp, unsigned long long seed, const TaxCand *cand, int *boot_g) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)q.nq * TAX_NBOOT) return;
  const int qb = (int)(i / TAX_NBOOT), bt = (int)(i % TAX_NBOOT);
  const unsigned long long jb = tax_mix(tax_mix(seed) + (unsigned long long)q.j[qb]);
  TaxCand b{0.f, -1};
  unsigned long long bh = 0ull;
  for (int grp = 0; grp < ngrp; grp++) {
    const TaxCand x = cand[((size_t)qb * ngrp + grp) * TAX_NBOOT + bt];
    if (x.g < 0) continue;
    const unsigned long long h = tax_hash(jb, bt, x.g);
    if (tax_better(x.lp, h, x.g, b.lp, bh, b.g)) { b = x; bh = h; }
  }
  boot_g[i] = b.g;
}

__global__ void k_tax_count(int nq, int nlevel, const int *gm, const int *best_g, const int *boot_g, int *boot) {
  const int qb = blockIdx.x * blockDim.x + threadIdx.x;
  if (qb >= nq) return;
  const int mg = best_g[qb];
  int *bo = boot + (size_t)qb * nlevel;
  for (int l = 0; l < nlevel; l++) bo[l] = 0;
  for (int bt = 0; bt < TAX_NBOOT; bt++) {                        // taxonomy.cpp:189-195
    const int bg = boot_g[(size_t)qb * TAX_NBOOT + bt];
    for (int l = 0; l < nlevel; l++) {
      if (gm[(size_t)bg * nlevel + l] != gm[(size_t)mg * nlevel + l]) break;
      bo[l]++;
    }
  }
}

__global__ void k_tax_gather(const float *tab, int cpad, int g0, int cn, int nk, const int *kmers, int ng, const int *genera, float *out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)nk * ng) return;
  const int g = genera[i % ng] - g0;
  if (g >= 0 && g < cn) out[i] = tab[(size_t)kmers[i / ng] * cpad + g];
}

}  // namespace dd2

using namespace dd2;

struct dada2b_tax_db {
  int device = 0, nref = 0, ngenus = 0, nlevel = 0, nchunk = 0, cg = 0, cpad = 0, ngrp = 0;
  std::vector<int> cg0, cr0, cgrp0;             // per chunk (+1 sentinel): first genus, first (genus-sorted) reference, first group
  int resident = -1;                            // chunk whose table is in tab
  BBuf<float> tab, prior, gnp1;
  BBuf<int> gm, rg;
  BBuf<char> rseq;
  BBuf<long long> roff;
  dada2b_tax_db_info info{};
};

namespace {

long long g_launches = 0, g_kbytes = 0;         // counters of the call in progress (calls are not concurrent on one db)

void tax_fail(char *errbuf, const std::string &m) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", m.c_str()); }

int valid_kmers(const char *s, long long L) {   // A/C/G/T runs of length r contribute r - 7
  long long run = 0, n = 0;
  for (long long i = 0; i < L; i++) {
    const char c = s[i];
    if (c == 'A' || c == 'C' || c == 'G' || c == 'T') { if (++run >= 8) n++; }
    else run = 0;
  }
  return n > INT32_MAX ? INT32_MAX : (int)n;
}

// Builds chunk c's table into db->tab (db->resident = c).
void build_chunk(dada2b_tax_db *db, int c, cudaStream_t s, bool first) {
  if (db->resident == c) return;
  const int g0 = db->cg0[c], cn = db->cg0[c + 1] - g0, r0 = db->cr0[c], nr = db->cr0[c + 1] - r0;
  const size_t n = (size_t)TAX_NK * db->cpad;
  BCK(cudaMemsetAsync(db->tab.p, 0, n * 4, s));
  BBuf<unsigned> ck;
  if (first) { ck.alloc(TAX_NK); BCK(cudaMemsetAsync(ck.p, 0, TAX_NK * 4, s)); }
  if (nr > 0) {
    const char *sp = db->rseq.p; const long long *op = db->roff.p; const int *rp = db->rg.p;
    unsigned *cp = (unsigned *)db->tab.p, *kp = ck.p;
    const int cpad = db->cpad;
    k_tax_presence<<<nr, 256, 0, s>>>(sp, op, rp, r0, g0, cpad, cp, kp);
    g_launches++;
  }
  if (first) {
    const unsigned *kp = ck.p; float *pp = db->prior.p; const double nref = (double)db->nref;
    k_tax_prior<<<TAX_NK / 256, 256, 0, s>>>(kp, nref, pp);
    g_launches++; g_kbytes += TAX_NK * 8;
  }
  {
    float *tp = db->tab.p; const float *pp = db->prior.p; const float *gp = db->gnp1.p + g0; const int cpad = db->cpad;
    const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, 132 * 64);
    k_tax_log<<<grid, 256, 0, s>>>(tp, pp, gp, cn, cpad);
    g_launches++; g_kbytes += (long long)n * 8 + TAX_NK * 4;
  }
  BCK(cudaStreamSynchronize(s));
  if (first) ck.release();
  db->resident = c;
}

void put_stats(long long launches, long long h2d, long long d2h, long long kb, cudaEvent_t *ev, int64_t &L, int64_t &H, int64_t &D, int64_t &K,
               double &mh, double &mk, double &md, double &mdev) {
  float ms = 0;
  BCK(cudaEventElapsedTime(&ms, ev[0], ev[1])); mh = ms;
  BCK(cudaEventElapsedTime(&ms, ev[1], ev[2])); mk = ms;
  BCK(cudaEventElapsedTime(&ms, ev[2], ev[3])); md = ms;
  BCK(cudaEventElapsedTime(&ms, ev[0], ev[3])); mdev = ms;
  L = launches; H = h2d; D = d2h; K = kb;
}

struct Events {
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaStream_t s = nullptr;
  Events() {
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
  }
  ~Events() {
    for (auto &e : ev) if (e) cudaEventDestroy(e);
    if (s) cudaStreamDestroy(s);
  }
};

dada2b_tax_db *db_build(const dada2b_tax_seqs *refs, const int32_t *ref_to_genus, const int32_t *genusmat, int32_t ngenus, int32_t nlevel,
                        const dada2b_tax_opts *opts, int32_t device) {
  const double t0 = bnow_ms();
  if (!refs) throw BErr{"dada2b: NULL argument."};
  if (refs->n < 0) throw BErr{"dada2b: negative reference count."};
  if ((long long)refs->n >= (1LL << 24))
    throw BErr{"dada2b: 2^24 or more references: per-genus and per-k-mer counts would not be exact in float."};
  if (ngenus < 1) throw BErr{"dada2b: no genera."};
  if (nlevel < 1) throw BErr{"dada2b: the genus matrix needs at least one level."};
  if ((refs->n > 0 && (!ref_to_genus || !refs->seq_off || !refs->seq_concat)) || !genusmat) throw BErr{"dada2b: NULL argument."};
  const int nref = refs->n;
  for (int i = 0; i < nref; i++)
    if (ref_to_genus[i] < 1 || ref_to_genus[i] > ngenus) throw BErr{"Invalid map from references to genus."};   // taxonomy.cpp:222
  dada2b_tax_opts o;
  dada2b_tax_default_opts(&o);
  if (opts) o = *opts;
  long long cg = ngenus;
  if (o.max_table_bytes > 0) {
    cg = o.max_table_bytes / ((long long)TAX_NK * 4 * TAX_GRP) * TAX_GRP;
    if (cg < TAX_GRP) throw BErr{"dada2b: max_table_bytes is below one 128-genus table (32 MiB)."};
  }
  if (o.chunk_genera > 0) cg = o.chunk_genera;
  if (const char *e = getenv("DADA2B_TAX_CHUNK_GENERA")) { const long long v = atoll(e); if (v > 0) cg = v; }
  cg = std::min<long long>(cg, ngenus);
  need_device(device);
  std::unique_ptr<dada2b_tax_db> db(new dada2b_tax_db());
  db->device = device; db->nref = nref; db->ngenus = ngenus; db->nlevel = nlevel;
  db->cg = (int)cg;
  db->nchunk = (int)((ngenus + cg - 1) / cg);
  db->cpad = (int)((cg + TAX_GRP - 1) / TAX_GRP * TAX_GRP);
  // references ordered by genus (stable), so that a chunk's references are one range
  std::vector<int> order(nref);
  for (int i = 0; i < nref; i++) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ref_to_genus[a] < ref_to_genus[b]; });
  std::vector<float> gnp1(ngenus, 0.f);
  for (int i = 0; i < nref; i++) gnp1[ref_to_genus[i] - 1]++;                     // taxonomy.cpp:229-234
  for (auto &v : gnp1) v++;
  for (int c = 0; c <= db->nchunk; c++) {
    const int g0 = (int)std::min<long long>((long long)c * cg, ngenus);
    db->cg0.push_back(g0);
    db->cgrp0.push_back(c * (db->cpad / TAX_GRP));
    db->cr0.push_back((int)(std::lower_bound(order.begin(), order.end(), g0 + 1,
                                             [&](int r, int v) { return ref_to_genus[r] < v; }) - order.begin()));
  }
  db->ngrp = db->nchunk * (db->cpad / TAX_GRP);
  long long nb = 0;
  for (int i = 0; i < nref; i++) {
    const long long l = refs->seq_off[i + 1] - refs->seq_off[i];
    if (l < 0) throw BErr{"Bad sequence offsets."};
    nb += l;
  }
  std::vector<char> rs((size_t)std::max<long long>(nb, 1));
  std::vector<long long> ro((size_t)nref + 1, 0);
  std::vector<int> rg((size_t)std::max(nref, 1), 0);
  for (int i = 0; i < nref; i++) {
    const int r = order[i];
    const long long l = refs->seq_off[r + 1] - refs->seq_off[r];
    memcpy(rs.data() + ro[i], refs->seq_concat + refs->seq_off[r], (size_t)l);
    ro[i + 1] = ro[i] + l;
    rg[i] = ref_to_genus[r] - 1;
  }
  Events E;
  cudaStream_t s = E.s;
  long long h2d = 0, d2h = 0;
  g_launches = 0; g_kbytes = 0;
  BCK(cudaEventRecord(E.ev[0], s));
  db->rseq.alloc(rs.size()); db->roff.alloc(ro.size()); db->rg.alloc(rg.size());
  db->gm.alloc((size_t)ngenus * nlevel); db->gnp1.alloc(ngenus); db->prior.alloc(TAX_NK);
  BCK(cudaMemcpyAsync(db->rseq.p, rs.data(), rs.size(), cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->roff.p, ro.data(), ro.size() * 8, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->rg.p, rg.data(), rg.size() * 4, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->gm.p, genusmat, (size_t)ngenus * nlevel * 4, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->gnp1.p, gnp1.data(), (size_t)ngenus * 4, cudaMemcpyHostToDevice, s));
  h2d += (long long)rs.size() + (long long)ro.size() * 8 + (long long)rg.size() * 4 + (long long)ngenus * nlevel * 4 + (long long)ngenus * 4;
  BCK(cudaEventRecord(E.ev[1], s));
  db->tab.alloc((size_t)TAX_NK * db->cpad);
  // the first build also counts count_k over every reference: one pass over all of them without table counts when chunked
  if (db->nchunk == 1) {
    build_chunk(db.get(), 0, s, true);
  } else {
    BBuf<unsigned> ck; ck.alloc(TAX_NK);
    BCK(cudaMemsetAsync(ck.p, 0, TAX_NK * 4, s));
    if (nref) {
      const char *sp = db->rseq.p; const long long *op = db->roff.p; const int *rp = db->rg.p; unsigned *kp = ck.p;
      unsigned *np = nullptr;
      k_tax_presence<<<nref, 256, 0, s>>>(sp, op, rp, 0, 0, 0, np, kp);
      g_launches++;
    }
    const unsigned *kp = ck.p; float *pp = db->prior.p; const double dn = (double)nref;
    k_tax_prior<<<TAX_NK / 256, 256, 0, s>>>(kp, dn, pp);
    g_launches++;
    BCK(cudaStreamSynchronize(s));
  }
  g_kbytes += nb;
  BCK(cudaEventRecord(E.ev[2], s));
  BCK(cudaEventRecord(E.ev[3], s));
  BCK(cudaStreamSynchronize(s));
  BCK(cudaGetLastError());
  if (db->nchunk == 1) { db->rseq.release(); db->roff.release(); db->rg.release(); }    // the resident table is all that is needed
  dada2b_tax_db_info &I = db->info;
  I.nref = nref; I.ngenus = ngenus; I.nlevel = nlevel; I.nchunk = db->nchunk; I.chunk_genera = db->cg;
  I.table_bytes = (long long)TAX_NK * db->cpad * 4;
  put_stats(g_launches, h2d, d2h, g_kbytes, E.ev, I.gpu_launches, I.h2d_bytes, I.d2h_bytes, I.kernel_bytes, I.ms_h2d, I.ms_kernels,
            I.ms_d2h, I.ms_device);
  I.ms_total = bnow_ms() - t0;
  return db.release();
}

// The one launch sequence of dada2b_tax_classify and the logp hook (dump != NULL: every query, main sums only).
dada2b_tax_out *classify(dada2b_tax_db *db, const dada2b_tax_seqs *sq, int try_rc, const double *unifs, long long nunifs,
                         unsigned long long seed, float *dump) {
  const double t0 = bnow_ms();
  if (!db || !sq) throw BErr{"dada2b: NULL argument."};
  const int nseq = sq->n;
  if (nseq <= 0) throw BErr{"No seqs provided to classify."};                      // taxonomy.cpp:212
  if (!sq->seq_off || !sq->seq_concat) throw BErr{"dada2b: NULL argument."};
  std::vector<int> alen(nseq), act;
  long long mal = 0;
  for (int i = 0; i < nseq; i++) {
    const long long L = sq->seq_off[i + 1] - sq->seq_off[i];
    if (L < 0) throw BErr{"Bad sequence offsets."};
    if (L >= 7) mal = std::max(mal, L - 7);                                          // taxonomy.cpp:279 (shorter: left out)
    alen[i] = valid_kmers(sq->seq_concat + sq->seq_off[i], L);
    if (alen[i] > DADA2B_TAX_MAXKMERS)
      throw BErr{"dada2b: query " + std::to_string(i + 1) + " has " + std::to_string(alen[i]) + " valid 8-mers; at most " +
                 std::to_string(DADA2B_TAX_MAXKMERS) + " are supported (the reference's limit)."};
    if (dump || L >= DADA2B_TAX_MINLEN) act.push_back(i);
  }
  const long long need = (long long)nseq * TAX_NBOOT * (mal / 8);
  if (unifs && nunifs != need)
    throw BErr{"dada2b: unifs must hold nseq * 100 * (max_arraylen / 8) = " + std::to_string(need) + " values (got " +
               std::to_string(nunifs) + ")."};
  BCK(cudaSetDevice(db->device));
  std::unique_ptr<dada2b_tax_out, void (*)(dada2b_tax_out *)> res((dada2b_tax_out *)calloc(1, sizeof(dada2b_tax_out)), dada2b_tax_free);
  dada2b_tax_out *R = res.get();
  const int nl = db->nlevel;
  R->nseq = nseq; R->nlevel = nl;
  R->tax = (int32_t *)malloc((size_t)nseq * 4);
  R->boot = (int32_t *)calloc((size_t)nseq * nl, 4);
  R->boot_tax = (int32_t *)malloc((size_t)nseq * TAX_NBOOT * 4);
  R->logp = (float *)malloc((size_t)nseq * 4);
  R->used_rc = (uint8_t *)calloc((size_t)nseq, 1);
  for (int i = 0; i < nseq; i++) { R->tax[i] = DADA2B_TAX_NA; R->logp[i] = NAN; }
  for (long long i = 0; i < (long long)nseq * TAX_NBOOT; i++) R->boot_tax[i] = DADA2B_TAX_NA;
  Events E;
  cudaStream_t s = E.s;
  long long h2d = 0, d2h = 0;
  g_launches = 0; g_kbytes = 0;
  double ms_h = 0, ms_k = 0, ms_d = 0;
  BBuf<double> d_u;
  if (unifs && need > 0) {
    d_u.alloc((size_t)need);
    BCK(cudaMemcpyAsync(d_u.p, unifs, (size_t)need * 8, cudaMemcpyHostToDevice, s));
    h2d += need * 8;
  }
  const double *up = unifs ? d_u.p : nullptr;
  const int want_rc = (try_rc || dump) ? 1 : 0;
  const int MKall = std::max(8, act.empty() ? 8 : *std::max_element(alen.begin(), alen.end()));
  const long long per_q = (long long)db->ngrp * (TAX_NBOOT + 2) * 8 + (long long)MKall * (12 + 26) + 64;
  const int B = (int)std::max<long long>(1, std::min<long long>(16384, (512LL << 20) / per_q));
  BCK(cudaEventRecord(E.ev[0], s));
  BCK(cudaEventRecord(E.ev[1], s));
  for (size_t a0 = 0; a0 < act.size(); a0 += B) {
    const int nq = (int)std::min<size_t>(B, act.size() - a0);
    std::vector<long long> off((size_t)nq + 1, 0);
    std::vector<int> al(nq), jj(nq);
    int MK = 8, maxW = 1;
    for (int i = 0; i < nq; i++) {
      const int j = act[a0 + i];
      const long long L = sq->seq_off[j + 1] - sq->seq_off[j];
      off[i + 1] = off[i] + L; al[i] = alen[j]; jj[i] = j;
      MK = std::max(MK, al[i]);
      maxW = std::max<long long>(maxW, L >= 8 ? L - 7 : 0);
    }
    std::vector<char> cat((size_t)std::max<long long>(off[nq], 1));
    for (int i = 0; i < nq; i++) memcpy(cat.data() + off[i], sq->seq_concat + sq->seq_off[jj[i]], (size_t)(off[i + 1] - off[i]));
    BBuf<char> d_seq; BBuf<long long> d_off; BBuf<int> d_al, d_j, d_nd, d_bg, d_btg, d_boot; BBuf<unsigned> d_kf, d_kr, d_kd;
    BBuf<unsigned short> d_dr; BBuf<TaxCand> d_cm, d_cb; BBuf<float> d_lp, d_dump; BBuf<unsigned char> d_used;
    d_seq.alloc(cat.size()); d_off.alloc(off.size()); d_al.alloc(nq); d_j.alloc(nq);
    const double th = bnow_ms();
    BCK(cudaMemcpyAsync(d_seq.p, cat.data(), cat.size(), cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_al.p, al.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_j.p, jj.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
    BCK(cudaStreamSynchronize(s));
    ms_h += bnow_ms() - th;
    h2d += (long long)cat.size() + (long long)off.size() * 8 + 8LL * nq;
    const double tk = bnow_ms();
    TaxQ q{};
    q.nq = nq; q.MK = MK; q.seq = d_seq.p; q.off = d_off.p; q.alen = d_al.p; q.j = d_j.p;
    d_kf.alloc((size_t)nq * MK); q.kf = d_kf.p;
    if (want_rc) { d_kr.alloc((size_t)nq * MK); q.kr = d_kr.p; }
    int P = 2;
    while (P < maxW) P <<= 1;
    const int qsm = P * 4;
    BCK(cudaFuncSetAttribute(k_tax_qkmers, cudaFuncAttributeMaxDynamicSharedMemorySize, qsm));
    k_tax_qkmers<<<nq, 256, qsm, s>>>(q, P, want_rc);
    g_launches++; g_kbytes += off[nq] + (long long)nq * MK * 4 * (want_rc ? 2 : 1);
    const int ngrp = db->ngrp;
    d_cm.alloc((size_t)nq * ngrp * 2);
    if (dump) d_dump.alloc((size_t)nq * 2 * db->ngenus);
    float *dp = dump ? d_dump.p : nullptr;
    const int ng = db->ngenus;
    for (int c = 0; c < db->nchunk; c++) {
      build_chunk(db, c, s, false);
      TaxChunk ch{db->tab.p, db->cpad, db->cg0[c + 1] - db->cg0[c], db->cg0[c], db->cgrp0[c]};
      TaxCand *cp = d_cm.p;
      const int trc = want_rc;
      k_tax_main<<<dim3((unsigned)(db->cpad / TAX_GRP), (unsigned)nq), TAX_GRP, 0, s>>>(q, ch, ngrp, trc, seed, cp, dp, ng);
      g_launches++;
      long long sumk = 0;
      for (int i = 0; i < nq; i++) sumk += al[i];
      g_kbytes += sumk * (want_rc ? 2 : 1) * ((long long)db->cpad * 4 + 4);
    }
    if (dump) {
      BCK(cudaStreamSynchronize(s));
      for (int i = 0; i < nq; i++)
        BCK(cudaMemcpyAsync(dump + (size_t)jj[i] * 2 * ng, d_dump.p + (size_t)i * 2 * ng, (size_t)2 * ng * 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      d2h += (long long)nq * 2 * ng * 4;
      continue;
    }
    d_bg.alloc(nq); d_lp.alloc(nq); d_used.alloc(nq);
    {
      const TaxCand *cp = d_cm.p; int *bp = d_bg.p; float *lp = d_lp.p; unsigned char *usp = d_used.p;
      const int trc = try_rc ? 1 : 0;
      k_tax_pick<<<(nq + 127) / 128, 128, 0, s>>>(q, ngrp, trc, seed, cp, bp, lp, usp);
      g_launches++; g_kbytes += (long long)nq * ngrp * 16 + 9LL * nq;
    }
    d_kd.alloc((size_t)nq * MK); d_nd.alloc(nq); q.kd = d_kd.p; q.nd = d_nd.p;
    q.DS = (long long)TAX_NBOOT * (MK / 8);
    d_dr.alloc((size_t)std::max<long long>(1, (long long)nq * q.DS)); q.dr = d_dr.p;
    {
      const int dsm = MK * 4;
      BCK(cudaFuncSetAttribute(k_tax_draws, cudaFuncAttributeMaxDynamicSharedMemorySize, dsm));
      const unsigned char *usp = d_used.p;
      k_tax_draws<<<nq, 256, dsm, s>>>(q, usp, up, mal, seed);
      g_launches++; g_kbytes += (long long)nq * MK * 8 + (long long)nq * q.DS * 2;
    }
    d_cb.alloc((size_t)nq * ngrp * TAX_NBOOT);
    const int bsm = std::min(MK, TAX_STAGE_ROWS) * TAX_GRP * 4;
    BCK(cudaFuncSetAttribute(k_tax_boot, cudaFuncAttributeMaxDynamicSharedMemorySize, bsm));
    for (int c = 0; c < db->nchunk; c++) {
      build_chunk(db, c, s, false);
      TaxChunk ch{db->tab.p, db->cpad, db->cg0[c + 1] - db->cg0[c], db->cg0[c], db->cgrp0[c]};
      TaxCand *cp = d_cb.p;
      k_tax_boot<<<dim3((unsigned)(db->cpad / TAX_GRP), (unsigned)nq), 256, bsm, s>>>(q, ch, ngrp, seed, cp);
      g_launches++;
      long long sumb = 0;
      for (int i = 0; i < nq; i++) sumb += al[i] / 8;
      g_kbytes += sumb * TAX_NBOOT * ((long long)db->cpad * 4 + 2) + (long long)nq * ngrp * TAX_NBOOT * 8;
    }
    d_btg.alloc((size_t)nq * TAX_NBOOT); d_boot.alloc((size_t)nq * nl);
    {
      const TaxCand *cp = d_cb.p; int *tp = d_btg.p;
      const long long nb = (long long)nq * TAX_NBOOT;
      k_tax_bootpick<<<(unsigned)((nb + 255) / 256), 256, 0, s>>>(q, ngrp, seed, cp, tp);
      const int *gp = db->gm.p, *bp = d_bg.p, *btp = d_btg.p; int *op = d_boot.p;
      k_tax_count<<<(nq + 127) / 128, 128, 0, s>>>(nq, nl, gp, bp, btp, op);
      g_launches += 2; g_kbytes += nb * ngrp * 8 + nb * 4 * 2 + (long long)nq * nl * 4;
    }
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    ms_k += bnow_ms() - tk;
    const double td = bnow_ms();
    std::vector<int> bg(nq), btg((size_t)nq * TAX_NBOOT), bo((size_t)nq * nl);
    std::vector<float> lp(nq);
    std::vector<unsigned char> us(nq);
    BCK(cudaMemcpyAsync(bg.data(), d_bg.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(lp.data(), d_lp.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(us.data(), d_used.p, (size_t)nq, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(btg.data(), d_btg.p, (size_t)nq * TAX_NBOOT * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(bo.data(), d_boot.p, (size_t)nq * nl * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    ms_d += bnow_ms() - td;
    d2h += (long long)nq * (4 + 4 + 1 + TAX_NBOOT * 4 + nl * 4);
    for (int i = 0; i < nq; i++) {
      const int j = jj[i];
      R->tax[j] = bg[i] + 1; R->logp[j] = lp[i]; R->used_rc[j] = us[i];
      for (int b = 0; b < TAX_NBOOT; b++) R->boot_tax[(size_t)j * TAX_NBOOT + b] = btg[(size_t)i * TAX_NBOOT + b] + 1;
      for (int l = 0; l < nl; l++) R->boot[(size_t)j * nl + l] = bo[(size_t)i * nl + l];
    }
  }
  BCK(cudaEventRecord(E.ev[2], s));
  BCK(cudaEventRecord(E.ev[3], s));
  BCK(cudaStreamSynchronize(s));
  BCK(cudaGetLastError());
  float ms = 0;
  BCK(cudaEventElapsedTime(&ms, E.ev[0], E.ev[3]));
  R->ms_device = ms;                                   // the batches' phases are host-timed around synchronised steps
  R->ms_h2d = ms_h; R->ms_kernels = ms_k; R->ms_d2h = ms_d;
  R->gpu_launches = g_launches; R->h2d_bytes = h2d; R->d2h_bytes = d2h; R->kernel_bytes = g_kbytes;
  R->ms_total = bnow_ms() - t0;
  return res.release();
}

template <class F> int guarded(char *errbuf, F f) {
  try { f(); return 0; }
  catch (BErr &e) { tax_fail(errbuf, e.msg); }
  catch (std::exception &e) { tax_fail(errbuf, e.what()); }
  return 1;
}

}  // namespace

extern "C" {

void dada2b_tax_default_opts(dada2b_tax_opts *o) {
  if (o) memset(o, 0, sizeof(*o));
}

int dada2b_tax_db_build(const dada2b_tax_seqs *refs, const int32_t *ref_to_genus, const int32_t *genusmat, int32_t ngenus, int32_t nlevel,
                        const dada2b_tax_opts *opts, int32_t device, dada2b_tax_db **db, char errbuf[DADA2B_ERRLEN]) {
  if (!db) { tax_fail(errbuf, "dada2b: NULL argument."); return 1; }
  *db = nullptr;
  return guarded(errbuf, [&] { *db = db_build(refs, ref_to_genus, genusmat, ngenus, nlevel, opts, device); });
}

int dada2b_tax_db_info_get(const dada2b_tax_db *db, dada2b_tax_db_info *info) {
  if (!db || !info) return 1;
  *info = db->info;
  return 0;
}

void dada2b_tax_db_free(dada2b_tax_db *db) {
  if (!db) return;
  cudaSetDevice(db->device);
  delete db;
}

int dada2b_tax_classify(dada2b_tax_db *db, const dada2b_tax_seqs *seqs, int32_t try_rc, const double *unifs, int64_t nunifs, uint64_t seed,
                        dada2b_tax_out **out, char errbuf[DADA2B_ERRLEN]) {
  if (!out) { tax_fail(errbuf, "dada2b: NULL argument."); return 1; }
  *out = nullptr;
  return guarded(errbuf, [&] { *out = classify(db, seqs, try_rc, unifs, nunifs, seed, nullptr); });
}

void dada2b_tax_free(dada2b_tax_out *o) {
  if (!o) return;
  free(o->tax); free(o->boot); free(o->boot_tax); free(o->logp); free(o->used_rc);
  free(o);
}

int dada2b_assign_taxonomy(const dada2b_tax_seqs *seqs, const dada2b_tax_seqs *refs, const int32_t *ref_to_genus, const int32_t *genusmat,
                           int32_t ngenus, int32_t nlevel, int32_t try_rc, const double *unifs, int64_t nunifs, uint64_t seed, int32_t device,
                           dada2b_tax_out **out, char errbuf[DADA2B_ERRLEN]) {
  if (!out) { tax_fail(errbuf, "dada2b: NULL argument."); return 1; }
  *out = nullptr;
  if (!seqs || seqs->n <= 0) { tax_fail(errbuf, "No seqs provided to classify."); return 1; }
  dada2b_tax_db *db = nullptr;
  if (dada2b_tax_db_build(refs, ref_to_genus, genusmat, ngenus, nlevel, nullptr, device, &db, errbuf)) return 1;
  const int rc = dada2b_tax_classify(db, seqs, try_rc, unifs, nunifs, seed, out, errbuf);
  dada2b_tax_db_free(db);
  return rc;
}

int dada2b_test_tax_table(dada2b_tax_db *db, int32_t nk, const int32_t *kmers, int32_t ng, const int32_t *genera, float *out,
                          char errbuf[DADA2B_ERRLEN]) {
  return guarded(errbuf, [&] {
    if (!db || (nk > 0 && (!kmers || !out)) || (ng > 0 && !genera)) throw BErr{"dada2b: NULL argument."};
    if (nk <= 0 || ng <= 0) return;
    for (int i = 0; i < nk; i++) if (kmers[i] < 0 || kmers[i] >= TAX_NK) throw BErr{"dada2b: k-mer out of range."};
    for (int i = 0; i < ng; i++) if (genera[i] < 0 || genera[i] >= db->ngenus) throw BErr{"dada2b: genus out of range."};
    BCK(cudaSetDevice(db->device));
    Events E;
    BBuf<int> dk, dg; BBuf<float> dout;
    dk.alloc(nk); dg.alloc(ng); dout.alloc((size_t)nk * ng);
    BCK(cudaMemcpyAsync(dk.p, kmers, (size_t)nk * 4, cudaMemcpyHostToDevice, E.s));
    BCK(cudaMemcpyAsync(dg.p, genera, (size_t)ng * 4, cudaMemcpyHostToDevice, E.s));
    const long long n = (long long)nk * ng;
    for (int c = 0; c < db->nchunk; c++) {
      build_chunk(db, c, E.s, false);
      const float *tp = db->tab.p; const int cpad = db->cpad, g0 = db->cg0[c], cn = db->cg0[c + 1] - g0;
      const int *kp = dk.p, *gp = dg.p; float *op = dout.p;
      k_tax_gather<<<(unsigned)((n + 255) / 256), 256, 0, E.s>>>(tp, cpad, g0, cn, nk, kp, ng, gp, op);
    }
    BCK(cudaMemcpyAsync(out, dout.p, (size_t)n * 4, cudaMemcpyDeviceToHost, E.s));
    BCK(cudaStreamSynchronize(E.s));
    BCK(cudaGetLastError());
  });
}

int dada2b_test_tax_logp(dada2b_tax_db *db, const dada2b_tax_seqs *seqs, float *out, char errbuf[DADA2B_ERRLEN]) {
  return guarded(errbuf, [&] {
    if (!out) throw BErr{"dada2b: NULL argument."};
    dada2b_tax_out *r = classify(db, seqs, 1, nullptr, 0, 0, out);
    dada2b_tax_free(r);
  });
}

}  // extern "C"
