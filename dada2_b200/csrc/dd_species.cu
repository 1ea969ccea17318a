// Species assignment by exact matching on the H100 (include/dada2b_species.h).  Product code.
//
// Replaces the PDict / vcountPDict loop of assignSpecies (R/taxonomy.R:264-280).  The contract is DESIGN.md 22: a hit is
// an exact substring occurrence of a query (or, with try_rc, of its reverse complement) in a reference; a reference
// position that is not A/C/G/T matches nothing; hits are reduced to distinct (query, reference) pairs and then to the
// distinct genus and species label ids of each query on the device.
//
// Layout.  The references are laid end to end, each followed by one separator position, and 2-bit packed (16 bases per
// word, base j of a word in bits 2j..2j+1) with a 1-bit mask of positions that are not A/C/G/T (32 per word); the
// separators and the tail padding are masked.  So any window that crosses a reference end or a non-ACGT position fails
// its mask test, and the scan never needs to know which reference a position belongs to until a hit is confirmed.
//
// Patterns are the queries and, with try_rc, their reverse complements.  A pattern of L >= 32 nt is anchored by one
// 32-mer at an offset chosen on the host so that few patterns share an anchor (ASVs of one clade share long prefixes); a
// shorter pattern is its own anchor.  The anchors are grouped by (length, code) into an open-addressing table with a
// presence filter, built on the host (their number is that of the queries) and uploaded.
//   k_sp_pack     one thread per 32 positions: the references' packed words and mask word (database build)
//   k_sp_scan     grid-stride over every position: the 32 bases and mask bits starting there; for each anchor length
//                 present, the filter bit (shared memory), then the table; every pattern of a matching group is verified
//                 word by word (32 bases at a time) against the packed bases and mask at start p - offset; a confirmed
//                 occurrence appends (reference, query) to the hit buffer (the count runs on past the capacity, so an
//                 overflow is seen, the buffer grown and the scan repeated)
//   k_sp_heads / k_sp_compact / k_sp_count / k_sp_emit  the hit records sorted by (query, reference) with the shared LSD
//                 radix sort (dd_sort.cuh), deduplicated; then the same for (query, genus) and (query, species): per-query
//                 counts and the ascending label lists of the queries whose count is within keep
#include "../../include/dada2b_species.h"
#include "dd_flt.cuh"
#include "dd_sort.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace dd2 {

constexpr int SP_ANCHOR = DADA2B_SPECIES_ANCHOR;
constexpr int SP_NCAND = 8;                     // candidate anchor offsets per pattern
constexpr int SP_THREADS = 512;
constexpr int SP_MAX_FBITS = 19;                // presence filter of at most 2^19 bits (64 KB of shared memory)

__host__ __device__ __forceinline__ unsigned long long sp_hash(unsigned long long code, int k) {   // splitmix64 finaliser
  unsigned long long z = code + (unsigned long long)k * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ int sp_code(char c) {
  return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
}
// The 32 bases starting at position g (base j in bits 2j..2j+1); pk holds at least g / 16 + 3 words.
__device__ __forceinline__ unsigned long long sp_bases32(const uint32_t *pk, long long g) {
  const long long w = g >> 4;
  const int sh = (int)(g & 15) * 2;
  const unsigned long long lo = (unsigned long long)pk[w] | ((unsigned long long)pk[w + 1] << 32);
  return sh ? (lo >> sh) | ((unsigned long long)pk[w + 2] << (64 - sh)) : lo;
}
// The 32 mask bits starting at position g; mk holds at least g / 32 + 2 words.
__device__ __forceinline__ uint32_t sp_mask32(const uint32_t *mk, long long g) {
  const long long w = g >> 5;
  const int sh = (int)(g & 31);
  return sh ? (mk[w] >> sh) | (mk[w + 1] << (32 - sh)) : mk[w];
}

__global__ void __launch_bounds__(256) k_sp_pack(const char *raw, long long N, long long nmw, uint32_t *pk, uint32_t *mk) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nmw) return;
  uint32_t m = 0, b0 = 0, b1 = 0;
  for (int j = 0; j < 32; j++) {
    const long long g = w * 32 + j;
    const int c = g < N ? sp_code(raw[g]) : -1;
    if (c < 0) m |= 1u << j;
    else if (j < 16) b0 |= (uint32_t)c << (2 * j);
    else b1 |= (uint32_t)c << (2 * (j - 16));
  }
  mk[w] = m; pk[2 * w] = b0; pk[2 * w + 1] = b1;
}

struct SpScan {
  const uint32_t *pk, *mk; long long N;         // packed bases and mask of the references (with separators)
  const long long *rstart; int nref;            // [nref + 1] first position of each reference
  const uint32_t *filt; int fbits;              // presence filter (2^fbits bits, bit = hash >> (64 - fbits))
  const unsigned long long *tcode; const int *tk, *tbeg;   // table [tmask + 1]: anchor code, length (0: empty), group start
  unsigned tmask;
  const int *gpat;                              // patterns of each group: gpat[tbeg[s] .. tbeg[s] + tcnt[s])
  const int *tcnt;
  const uint32_t *pw; const long long *pwoff;   // pattern words (16 bases each, an even number per pattern, padded)
  const int *plen, *poff, *pq;                  // pattern length, anchor offset, query
  int nk; int ks[SP_ANCHOR];                    // anchor lengths present
  unsigned long long *nhit; uint32_t *hit;      // hit records [cap][2] = (reference, query); nhit counts past cap
  unsigned long long cap;
};

__device__ __forceinline__ void sp_verify(const SpScan &a, int p, long long g) {
  const long long s = g - a.poff[p];
  const int L = a.plen[p];
  if (s < 0 || s + L > a.N) return;
  const uint32_t *w = a.pw + a.pwoff[p];
  for (int i = 0; i < L; i += 32) {
    const int nb = min(32, L - i);
    const uint32_t mm = nb == 32 ? 0xffffffffu : (1u << nb) - 1u;
    if (sp_mask32(a.mk, s + i) & mm) return;
    const unsigned long long pb = (unsigned long long)w[i >> 4] | ((unsigned long long)w[(i >> 4) + 1] << 32);
    const unsigned long long bm = nb == 32 ? ~0ull : (1ull << (2 * nb)) - 1ull;
    if ((sp_bases32(a.pk, s + i) ^ pb) & bm) return;
  }
  int lo = 0, hi = a.nref - 1;                  // the reference holding s: last r with rstart[r] <= s
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.rstart[mid] <= s) lo = mid; else hi = mid - 1;
  }
  const unsigned long long slot = atomicAdd(a.nhit, 1ull);
  if (slot < a.cap) { a.hit[2 * slot] = (uint32_t)lo; a.hit[2 * slot + 1] = (uint32_t)a.pq[p]; }
}

__global__ void __launch_bounds__(SP_THREADS) k_sp_scan(SpScan a) {
  extern __shared__ uint32_t sfilt[];
  const int fw = 1 << (a.fbits - 5);
  for (int i = threadIdx.x; i < fw; i += blockDim.x) sfilt[i] = a.filt[i];
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < a.N; g += stride) {
    const uint32_t m = sp_mask32(a.mk, g);
    if (m & 1u) continue;                       // no anchor starts on a separator or a non-ACGT position
    const unsigned long long c = sp_bases32(a.pk, g);
    for (int t = 0; t < a.nk; t++) {
      const int k = a.ks[t];
      if (m & (k == 32 ? 0xffffffffu : (1u << k) - 1u)) continue;
      const unsigned long long code = k == 32 ? c : c & ((1ull << (2 * k)) - 1ull);
      const unsigned long long h = sp_hash(code, k);
      const unsigned fi = (unsigned)(h >> (64 - a.fbits));
      if (!((sfilt[fi >> 5] >> (fi & 31)) & 1u)) continue;
      for (unsigned s = (unsigned)h & a.tmask;; s = (s + 1u) & a.tmask) {
        const int tk = a.tk[s];
        if (tk == 0) break;
        if (tk == k && a.tcode[s] == code) {
          const int b = a.tbeg[s], e = b + a.tcnt[s];
          for (int i = b; i < e; i++) sp_verify(a, a.gpat[i], g);
          break;
        }
      }
    }
  }
}

// head[i] = 1 where sorted pair i differs from pair i - 1 (keys [n][2], order idx)
__global__ void __launch_bounds__(256) k_sp_heads(const uint32_t *keys, const uint32_t *idx, unsigned n, uint32_t *head) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t a = idx[i];
  if (i == 0) { head[i] = 1u; return; }
  const uint32_t b = idx[i - 1];
  head[i] = (keys[2 * a] != keys[2 * b] || keys[2 * a + 1] != keys[2 * b + 1]) ? 1u : 0u;
}

// out[pos[i]] = pair idx[i] where head[i]
__global__ void __launch_bounds__(256) k_sp_compact(const uint32_t *keys, const uint32_t *idx, const uint32_t *head, const uint32_t *pos,
                                                    unsigned n, uint32_t *out) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !head[i]) return;
  const uint32_t a = idx[i];
  out[2 * pos[i]] = keys[2 * a]; out[2 * pos[i] + 1] = keys[2 * a + 1];
}

// (reference, query) -> (label of the reference, query)
__global__ void __launch_bounds__(256) k_sp_relabel(const uint32_t *pairs, unsigned n, const int *lab, uint32_t *out) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[2 * i] = (uint32_t)lab[pairs[2 * i]]; out[2 * i + 1] = pairs[2 * i + 1];
}

__global__ void __launch_bounds__(256) k_sp_count(const uint32_t *pairs, unsigned n, uint32_t *cnt) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&cnt[pairs[2 * i + 1]], 1u);
}

// emit[q] = cnt[q] when the list is returned (keep <= 0 or cnt <= keep), else 0
__global__ void __launch_bounds__(256) k_sp_keep(const uint32_t *cnt, int nq, int keep, uint32_t *emit) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < nq) emit[q] = (keep <= 0 || cnt[q] <= (uint32_t)keep) ? cnt[q] : 0u;
}

// pairs sorted by (query, label): the labels of returned lists to out[off[q] + (i - first[q])]
__global__ void __launch_bounds__(256) k_sp_emit(const uint32_t *pairs, unsigned n, const uint32_t *first, const uint32_t *emit,
                                                 const uint32_t *off, int32_t *out) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t q = pairs[2 * i + 1];
  if (emit[q]) out[off[q] + (i - first[q])] = (int32_t)pairs[2 * i];
}

}  // namespace dd2

using namespace dd2;

struct dada2b_species_db {
  int device = 0, nref = 0, maxg = 0, maxs = 0;
  long long N = 0;                              // positions, separators included
  BBuf<uint32_t> pk, mk;
  BBuf<long long> rstart;
  BBuf<int> rg, rs;
  dada2b_species_db_info info{};
};

namespace {

void sp_fail(char *errbuf, const std::string &m) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", m.c_str()); }

struct Events {
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaStream_t s = nullptr;
  Events() {
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
  }
  ~Events() {
    for (auto &e : ev) if (e) cudaEventDestroy(e);
    if (s) cudaStreamDestroy(s);
  }
  double ms(int a, int b) { float m = 0; BCK(cudaEventElapsedTime(&m, ev[a], ev[b])); return m; }
};

int nbytes_of(long long maxv) { int b = 1; while (b < 4 && maxv >= (1LL << (8 * b))) b++; return b; }
unsigned nblk(long long n) { return (unsigned)((n + 255) / 256); }

dada2b_species_db *db_build(const dada2b_species_seqs *refs, const int32_t *rg, const int32_t *rs, int32_t device) {
  const double t0 = bnow_ms();
  if (!refs || (refs->n > 0 && (!refs->seq_off || !refs->seq_concat || !rg || !rs))) throw BErr{"dada2b: NULL argument."};
  if (refs->n <= 0) throw BErr{"dada2b: no reference sequences."};
  const int nref = refs->n;
  int maxg = 0, maxs = 0;
  long long nb = 0;
  for (int i = 0; i < nref; i++) {
    const long long l = refs->seq_off[i + 1] - refs->seq_off[i];
    if (l < 0) throw BErr{"Bad sequence offsets."};
    if (rg[i] < 0 || rs[i] < 0) throw BErr{"dada2b: label ids must be >= 0 (0 is NA)."};
    maxg = std::max(maxg, (int)rg[i]); maxs = std::max(maxs, (int)rs[i]);
    nb += l;
  }
  const long long N = nb + nref;                // one separator after each reference
  need_device(device);
  std::unique_ptr<dada2b_species_db> db(new dada2b_species_db());
  db->device = device; db->nref = nref; db->N = N; db->maxg = maxg; db->maxs = maxs;
  std::vector<char> raw((size_t)N);
  std::vector<long long> rst((size_t)nref + 1);
  long long g = 0;
  for (int i = 0; i < nref; i++) {
    const long long l = refs->seq_off[i + 1] - refs->seq_off[i];
    rst[i] = g;
    memcpy(raw.data() + g, refs->seq_concat + refs->seq_off[i], (size_t)l);
    raw[(size_t)(g + l)] = '\n';
    g += l + 1;
  }
  rst[nref] = g;
  const long long nmw = N / 32 + 4;             // mask words; two packed words each, so every window read stays inside
  Events E;
  cudaStream_t s = E.s;
  BCK(cudaEventRecord(E.ev[0], s));
  BBuf<char> d_raw;
  d_raw.alloc((size_t)N);
  db->pk.alloc((size_t)nmw * 2); db->mk.alloc((size_t)nmw); db->rstart.alloc((size_t)nref + 1);
  db->rg.alloc((size_t)nref); db->rs.alloc((size_t)nref);
  BCK(cudaMemcpyAsync(d_raw.p, raw.data(), (size_t)N, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->rstart.p, rst.data(), rst.size() * 8, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->rg.p, rg, (size_t)nref * 4, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(db->rs.p, rs, (size_t)nref * 4, cudaMemcpyHostToDevice, s));
  BCK(cudaEventRecord(E.ev[1], s));
  {
    const char *rp = d_raw.p; uint32_t *pp = db->pk.p, *mp = db->mk.p;
    k_sp_pack<<<nblk(nmw), 256, 0, s>>>(rp, N, nmw, pp, mp);
  }
  BCK(cudaEventRecord(E.ev[2], s));
  BCK(cudaEventRecord(E.ev[3], s));
  BCK(cudaStreamSynchronize(s));
  BCK(cudaGetLastError());
  dada2b_species_db_info &I = db->info;
  I.nref = nref; I.nbases = nb;
  I.device_bytes = nmw * 12 + ((long long)nref + 1) * 8 + (long long)nref * 8;
  I.gpu_launches = 1;
  I.h2d_bytes = N + ((long long)nref + 1) * 8 + (long long)nref * 8;
  I.kernel_bytes = N + nmw * 12;
  I.ms_h2d = E.ms(0, 1); I.ms_kernels = E.ms(1, 2); I.ms_d2h = 0; I.ms_device = E.ms(0, 3);
  I.ms_total = bnow_ms() - t0;
  return db.release();
}

// Open addressing on (anchor code, anchor length) with the device table's probe sequence: slot sp_hash & mask, then
// linear.  It counts the patterns per chosen anchor on the host and its arrays become the device's anchor table.
struct AnchorMap {
  std::vector<unsigned long long> code;
  std::vector<int> k, v;                        // k = 0: empty slot
  unsigned mask = 0;
  explicit AnchorMap(size_t n) {
    unsigned c = 16;
    while (c < 2 * n) c <<= 1;
    code.assign(c, 0ull); k.assign(c, 0); v.assign(c, 0); mask = c - 1;
  }
  unsigned slot(unsigned long long c, int kk) const {
    unsigned s = (unsigned)sp_hash(c, kk) & mask;
    while (k[s] && (k[s] != kk || code[s] != c)) s = (s + 1u) & mask;
    return s;
  }
  unsigned add(unsigned long long c, int kk) {  // the slot of (c, kk), inserted with v = 0 when absent
    const unsigned s = slot(c, kk);
    if (!k[s]) { k[s] = kk; code[s] = c; }
    return s;
  }
};

// Patterns, anchors and the anchor table of one call (host side; their size is that of the queries).
struct Patterns {
  std::vector<uint32_t> pw;
  std::vector<long long> pwoff;
  std::vector<int> plen, poff, pq, gpat, tbeg, ks;
  AnchorMap table{0};                           // v: patterns of the slot's group
  std::vector<uint32_t> filt;
  int fbits = 12, max_group = 0;
};

void make_patterns(const dada2b_species_seqs *sq, bool try_rc, bool anchor0, Patterns &P) {
  const int nq = sq->n;
  const int np = try_rc ? 2 * nq : nq;
  P.plen.resize(np); P.poff.resize(np); P.pq.resize(np); P.pwoff.resize(np);
  long long nw = 0;
  for (int p = 0; p < np; p++) {
    const int L = (int)(sq->seq_off[p % nq + 1] - sq->seq_off[p % nq]);
    P.plen[p] = L; P.pq[p] = p % nq; P.pwoff[p] = nw;
    nw += 2LL * ((L + 31) / 32) + 2;            // two words of padding: any 32-base window reads three words
  }
  // pattern p: query p, or for p >= nq the reverse complement of query p - nq (the complement of code c is 3 - c)
  P.pw.assign((size_t)nw, 0u);
  for (int p = 0; p < np; p++) {
    const char *s = sq->seq_concat + sq->seq_off[p % nq];
    const int L = P.plen[p];
    uint32_t *w = P.pw.data() + P.pwoff[p];
    if (p < nq) for (int j = 0; j < L; j++) w[j >> 4] |= (uint32_t)sp_code(s[j]) << (2 * (j & 15));
    else for (int j = 0; j < L; j++) w[j >> 4] |= (uint32_t)(3 - sp_code(s[L - 1 - j])) << (2 * (j & 15));
  }
  auto code_at = [&](int p, int o, int k) {
    const uint32_t *w = P.pw.data() + P.pwoff[p] + (o >> 4);
    const int sh = (o & 15) * 2;
    unsigned long long c = (unsigned long long)w[0] | ((unsigned long long)w[1] << 32);
    if (sh) c = (c >> sh) | ((unsigned long long)w[2] << (64 - sh));
    return k == 32 ? c : c & ((1ull << (2 * k)) - 1ull);
  };
  std::vector<unsigned> aslot(np);
  AnchorMap uses((size_t)np);                   // v: patterns anchored on each anchor so far
  for (int p = 0; p < np; p++) {
    const int L = P.plen[p];
    int o = 0;
    if (L > SP_ANCHOR && !anchor0) {            // the least shared of up to SP_NCAND evenly spaced offsets, first on ties
      const int span = L - SP_ANCHOR, nc = std::min(SP_NCAND, span + 1);
      int best = -1;
      for (int i = 0; i < nc; i++) {
        const int oi = (int)((long long)span * i / (nc - 1));
        const int u = uses.v[uses.slot(code_at(p, oi, SP_ANCHOR), SP_ANCHOR)];
        if (best < 0 || u < best) { best = u; o = oi; }
      }
    }
    const int k = std::min(L, SP_ANCHOR);
    P.poff[p] = o;
    aslot[p] = uses.add(code_at(p, o, k), k);
    uses.v[aslot[p]]++;
  }
  // the groups of patterns sharing an anchor, in pattern order: uses is the table
  P.table = std::move(uses);
  AnchorMap &T = P.table;
  const size_t cap = T.k.size();
  P.tbeg.assign(cap, 0);
  long long ng = 0;
  for (size_t s = 0, run = 0; s < cap; s++) {
    P.tbeg[s] = (int)run;
    run += (size_t)T.v[s];
    if (T.k[s]) { ng++; P.max_group = std::max(P.max_group, T.v[s]); }
  }
  P.gpat.assign((size_t)std::max(np, 1), 0);
  std::vector<int> fill(P.tbeg);
  for (int p = 0; p < np; p++) P.gpat[(size_t)fill[aslot[p]]++] = p;
  P.fbits = 12;
  while (P.fbits < SP_MAX_FBITS && (1LL << P.fbits) < 16LL * ng) P.fbits++;
  P.filt.assign((size_t)1 << (P.fbits - 5), 0u);
  bool seen[SP_ANCHOR + 1] = {false};
  for (size_t s = 0; s < cap; s++) {
    if (!T.k[s]) continue;
    const unsigned fi = (unsigned)(sp_hash(T.code[s], T.k[s]) >> (64 - P.fbits));
    P.filt[fi >> 5] |= 1u << (fi & 31);
    if (!seen[T.k[s]]) { seen[T.k[s]] = true; P.ks.push_back(T.k[s]); }
  }
  std::sort(P.ks.begin(), P.ks.end());
}

template <class T> void up(BBuf<T> &d, const std::vector<T> &h, cudaStream_t s, long long &h2d) {
  d.alloc(std::max<size_t>(h.size(), 1));
  if (!h.empty()) BCK(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, s));
  h2d += (long long)(h.size() * sizeof(T));
}

struct Reducer {                                // sorted unique (word 1, word 0) pairs on one stream
  cudaStream_t s;
  Sorter so;
  BBuf<uint32_t> idx, idx2, head, pos;
  long long launches = 0, d2h = 0;
  // pairs [n][2] -> out [nu][2] sorted by (word 1, word 0), duplicates removed; returns nu
  unsigned operator()(const uint32_t *pairs, unsigned n, int bytes0, int bytes1, BBuf<uint32_t> &out) {
    so.s = s;
    idx.alloc(n); idx2.alloc(n); head.alloc(n); pos.alloc(n);
    uint32_t *a = idx.p, *b = idx2.p;
    k_iota<<<nblk(n), 256, 0, s>>>(a, n);
    launches++;
    for (int by = 0; by < bytes0; by++) { so.pass(RsPass{pairs, 2, 0, 8 * by}, a, b, n); std::swap(a, b); }
    for (int by = 0; by < bytes1; by++) { so.pass(RsPass{pairs, 2, 1, 8 * by}, a, b, n); std::swap(a, b); }
    uint32_t *hp = head.p, *pp = pos.p;
    k_sp_heads<<<nblk(n), 256, 0, s>>>(pairs, a, n, hp);
    BCK(cudaMemcpyAsync(pp, hp, (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    so.scan(pp, n);
    uint32_t last[2];
    BCK(cudaMemcpyAsync(&last[0], pp + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&last[1], hp + (n - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    d2h += 8;
    const unsigned nu = last[0] + last[1];
    out.alloc((size_t)nu * 2);
    uint32_t *op = out.p;
    k_sp_compact<<<nblk(n), 256, 0, s>>>(pairs, a, hp, pp, n, op);
    launches += 2;
    return nu;
  }
};

// One label level: distinct (query, label) pairs, per-query counts, the returned lists.  Returns the list entries.
void labels(Reducer &R, const uint32_t *uhits, unsigned nu, const int *lab, int maxlab, int nq, int keep, int bytesq, cudaStream_t s,
            std::vector<uint32_t> &cnt, std::vector<int32_t> &ids, long long &d2h) {
  cnt.assign((size_t)nq, 0u);
  ids.clear();
  if (nu == 0) return;
  BBuf<uint32_t> rel, ul, d_cnt, d_first, d_emit, d_off;
  BBuf<int32_t> d_ids;
  rel.alloc((size_t)nu * 2);
  uint32_t *rp = rel.p;
  k_sp_relabel<<<nblk(nu), 256, 0, s>>>(uhits, nu, lab, rp);
  R.launches++;
  const unsigned nl = R(rel.p, nu, nbytes_of(maxlab), bytesq, ul);
  d_cnt.alloc(nq); d_first.alloc(nq); d_emit.alloc(nq); d_off.alloc(nq);
  uint32_t *cp = d_cnt.p, *fp = d_first.p, *ep = d_emit.p, *op = d_off.p;
  const uint32_t *up = ul.p;
  BCK(cudaMemsetAsync(cp, 0, (size_t)nq * 4, s));
  k_sp_count<<<nblk(nl), 256, 0, s>>>(up, nl, cp);
  k_sp_keep<<<nblk(nq), 256, 0, s>>>(cp, nq, keep, ep);
  BCK(cudaMemcpyAsync(fp, cp, (size_t)nq * 4, cudaMemcpyDeviceToDevice, s));
  BCK(cudaMemcpyAsync(op, ep, (size_t)nq * 4, cudaMemcpyDeviceToDevice, s));
  R.so.scan(fp, nq);
  R.so.scan(op, nq);
  R.launches += 2;
  uint32_t last[2];
  BCK(cudaMemcpyAsync(&last[0], op + (nq - 1), 4, cudaMemcpyDeviceToHost, s));
  BCK(cudaMemcpyAsync(&last[1], ep + (nq - 1), 4, cudaMemcpyDeviceToHost, s));
  BCK(cudaStreamSynchronize(s));
  const unsigned total = last[0] + last[1];
  d_ids.alloc(std::max(total, 1u));
  int32_t *ip = d_ids.p;
  k_sp_emit<<<nblk(nl), 256, 0, s>>>(up, nl, fp, ep, op, ip);
  R.launches++;
  ids.resize(total);
  BCK(cudaMemcpyAsync(cnt.data(), cp, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
  if (total) BCK(cudaMemcpyAsync(ids.data(), ip, (size_t)total * 4, cudaMemcpyDeviceToHost, s));
  BCK(cudaStreamSynchronize(s));
  d2h += 8 + (long long)nq * 4 + (long long)total * 4;
}

void csr(const std::vector<uint32_t> &cnt, int keep, std::vector<int32_t> &ids, int32_t *&n_out, int64_t *&off_out, int32_t *&ids_out) {
  const size_t nq = cnt.size();
  n_out = (int32_t *)malloc(std::max<size_t>(nq, 1) * 4);
  off_out = (int64_t *)malloc((nq + 1) * 8);
  ids_out = (int32_t *)malloc(std::max<size_t>(ids.size(), 1) * 4);
  off_out[0] = 0;
  for (size_t q = 0; q < nq; q++) {
    n_out[q] = (int32_t)cnt[q];
    off_out[q + 1] = off_out[q] + ((keep <= 0 || cnt[q] <= (uint32_t)keep) ? cnt[q] : 0);
  }
  if (!ids.empty()) memcpy(ids_out, ids.data(), ids.size() * 4);
}

dada2b_species_out *assign(dada2b_species_db *db, const dada2b_species_seqs *sq, int try_rc, int keep_g, int keep_s, bool want_hits) {
  const double t0 = bnow_ms();
  if (!db || !sq) throw BErr{"dada2b: NULL argument."};
  const int nq = sq->n;
  if (nq < 0) throw BErr{"dada2b: negative query count."};
  if (nq > 0 && (!sq->seq_off || !sq->seq_concat)) throw BErr{"dada2b: NULL argument."};
  for (int q = 0; q < nq; q++) {
    const long long L = sq->seq_off[q + 1] - sq->seq_off[q];
    if (L < 0) throw BErr{"Bad sequence offsets."};
    if (L == 0) throw BErr{"dada2b: query " + std::to_string(q + 1) + " is empty; assignSpecies needs non-empty queries."};
    if (L > INT32_MAX / 2) throw BErr{"dada2b: query too long."};
    const char *s = sq->seq_concat + sq->seq_off[q];
    for (long long j = 0; j < L; j++)
      if (sp_code(s[j]) < 0) throw BErr{"Non-ACGT characters present in the query sequences."};
  }
  BCK(cudaSetDevice(db->device));
  std::unique_ptr<dada2b_species_out, void (*)(dada2b_species_out *)> res((dada2b_species_out *)calloc(1, sizeof(dada2b_species_out)),
                                                                           dada2b_species_free);
  dada2b_species_out *O = res.get();
  O->nseq = nq;
  if (nq == 0) {
    std::vector<uint32_t> z;
    std::vector<int32_t> e;
    O->nhits = (int32_t *)malloc(4);
    csr(z, 0, e, O->genus_n, O->genus_off, O->genus_ids);
    csr(z, 0, e, O->species_n, O->species_off, O->species_ids);
    if (want_hits) { O->hit_off = (int64_t *)calloc(1, 8); O->hit_refs = (int32_t *)malloc(4); }
    O->ms_total = bnow_ms() - t0;
    return res.release();
  }
  const char *ea = getenv("DADA2B_SPECIES_ANCHOR0");
  Patterns P;
  make_patterns(sq, try_rc != 0, ea && atoi(ea) != 0, P);
  const int np = (int)P.plen.size();
  Events E;
  cudaStream_t s = E.s;
  long long h2d = 0, d2h = 0, launches = 0, kbytes = 0;
  BCK(cudaEventRecord(E.ev[0], s));
  BBuf<uint32_t> d_pw, d_filt; BBuf<long long> d_pwoff; BBuf<int> d_plen, d_poff, d_pq, d_gpat, d_tk, d_tbeg, d_tcnt;
  BBuf<unsigned long long> d_tcode, d_nhit;
  up(d_pw, P.pw, s, h2d); up(d_filt, P.filt, s, h2d); up(d_pwoff, P.pwoff, s, h2d); up(d_plen, P.plen, s, h2d);
  up(d_poff, P.poff, s, h2d); up(d_pq, P.pq, s, h2d); up(d_gpat, P.gpat, s, h2d); up(d_tk, P.table.k, s, h2d);
  up(d_tbeg, P.tbeg, s, h2d); up(d_tcnt, P.table.v, s, h2d); up(d_tcode, P.table.code, s, h2d);
  d_nhit.alloc(1);
  BCK(cudaEventRecord(E.ev[1], s));
  SpScan a{};
  a.pk = db->pk.p; a.mk = db->mk.p; a.N = db->N; a.rstart = db->rstart.p; a.nref = db->nref;
  a.filt = d_filt.p; a.fbits = P.fbits; a.tcode = d_tcode.p; a.tk = d_tk.p; a.tbeg = d_tbeg.p; a.tmask = P.table.mask;
  a.gpat = d_gpat.p; a.tcnt = d_tcnt.p; a.pw = d_pw.p; a.pwoff = d_pwoff.p; a.plen = d_plen.p; a.poff = d_poff.p; a.pq = d_pq.p;
  a.nk = (int)P.ks.size();
  for (int t = 0; t < a.nk; t++) a.ks[t] = P.ks[t];
  unsigned long long cap = std::max<unsigned long long>(1ull << 20, 8ull * (unsigned long long)np);
  if (const char *e = getenv("DADA2B_SPECIES_HITCAP")) { const long long v = atoll(e); if (v > 0) cap = (unsigned long long)v; }
  int sms = 0;
  BCK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, db->device));
  const int smem = (1 << P.fbits) / 8;
  const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>((db->N + SP_THREADS - 1) / SP_THREADS, 3LL * sms));
  BCK(cudaFuncSetAttribute(k_sp_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  BBuf<uint32_t> d_hit;
  unsigned long long nrec = 0;
  int scans = 0;
  for (;;) {
    d_hit.alloc((size_t)cap * 2);
    a.hit = d_hit.p; a.cap = cap; a.nhit = d_nhit.p;
    BCK(cudaMemsetAsync(d_nhit.p, 0, 8, s));
    k_sp_scan<<<grid, SP_THREADS, smem, s>>>(a);
    launches++; scans++;
    kbytes += db->N * 3 / 8;
    BCK(cudaMemcpyAsync(&nrec, d_nhit.p, 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    d2h += 8;
    if (nrec <= cap) break;
    if (nrec >= (1ull << 31)) throw BErr{"dada2b: " + std::to_string(nrec) + " hit occurrences; at most 2^31 - 1 are supported."};
    cap = nrec;                                 // the scan is deterministic in its count: one more pass records them all
  }
  BCK(cudaGetLastError());
  BCK(cudaEventRecord(E.ev[2], s));
  Reducer R; R.s = s;
  BBuf<uint32_t> uh;
  const int bytesq = nbytes_of(nq - 1);
  const unsigned nu = nrec ? R((const uint32_t *)d_hit.p, (unsigned)nrec, nbytes_of(db->nref - 1), bytesq, uh) : 0u;
  d_hit.release();
  std::vector<uint32_t> hcnt((size_t)nq, 0u), gcnt, scnt;
  std::vector<int32_t> hids, gids, sids;
  if (nu) {
    BBuf<uint32_t> d_c;
    d_c.alloc(nq);
    uint32_t *cp = d_c.p; const uint32_t *up_ = uh.p;
    BCK(cudaMemsetAsync(cp, 0, (size_t)nq * 4, s));
    k_sp_count<<<nblk(nu), 256, 0, s>>>(up_, nu, cp);
    R.launches++;
    BCK(cudaMemcpyAsync(hcnt.data(), cp, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    d2h += (long long)nq * 4;
  }
  labels(R, uh.p, nu, db->rg.p, db->maxg, nq, keep_g, bytesq, s, gcnt, gids, d2h);
  labels(R, uh.p, nu, db->rs.p, db->maxs, nq, keep_s, bytesq, s, scnt, sids, d2h);
  BCK(cudaEventRecord(E.ev[3], s));
  std::vector<uint32_t> hpairs;
  if (want_hits && nu) {
    hpairs.resize((size_t)nu * 2);
    BCK(cudaMemcpyAsync(hpairs.data(), uh.p, (size_t)nu * 8, cudaMemcpyDeviceToHost, s));
    d2h += (long long)nu * 8;
  }
  BCK(cudaEventRecord(E.ev[4], s));
  BCK(cudaStreamSynchronize(s));
  BCK(cudaGetLastError());
  O->nhits = (int32_t *)malloc((size_t)nq * 4);
  for (int q = 0; q < nq; q++) O->nhits[q] = (int32_t)hcnt[q];
  csr(gcnt, keep_g, gids, O->genus_n, O->genus_off, O->genus_ids);
  csr(scnt, keep_s, sids, O->species_n, O->species_off, O->species_ids);
  if (want_hits) {
    O->hit_off = (int64_t *)malloc(((size_t)nq + 1) * 8);
    O->hit_refs = (int32_t *)malloc(std::max<size_t>(nu, 1) * 4);
    O->hit_off[0] = 0;
    for (int q = 0; q < nq; q++) O->hit_off[q + 1] = O->hit_off[q] + hcnt[q];
    for (unsigned i = 0; i < nu; i++) O->hit_refs[i] = (int32_t)hpairs[2 * (size_t)i];     // sorted by (query, reference)
  }
  O->npatterns = np; O->hit_records = (int64_t)nrec; O->hit_capacity = (int64_t)cap; O->distinct_hits = nu;
  O->scans = scans; O->max_group = P.max_group;
  O->gpu_launches = launches + R.launches + R.so.launches; O->h2d_bytes = h2d; O->d2h_bytes = d2h + R.d2h;
  O->kernel_bytes = kbytes + (long long)nrec * 8 * 12;
  O->ms_h2d = E.ms(0, 1); O->ms_scan = E.ms(1, 2); O->ms_reduce = E.ms(2, 3); O->ms_d2h = E.ms(3, 4); O->ms_device = E.ms(0, 4);
  O->ms_total = bnow_ms() - t0;
  return res.release();
}

template <class F> int guarded(char *errbuf, F f) {
  try { f(); return 0; }
  catch (BErr &e) { sp_fail(errbuf, e.msg); }
  catch (std::exception &e) { sp_fail(errbuf, e.what()); }
  return 1;
}

}  // namespace

extern "C" {

int dada2b_species_db_build(const dada2b_species_seqs *refs, const int32_t *ref_to_genus, const int32_t *ref_to_species, int32_t device,
                            dada2b_species_db **db, char errbuf[DADA2B_ERRLEN]) {
  if (!db) { sp_fail(errbuf, "dada2b: NULL argument."); return 1; }
  *db = nullptr;
  return guarded(errbuf, [&] { *db = db_build(refs, ref_to_genus, ref_to_species, device); });
}

int dada2b_species_db_info_get(const dada2b_species_db *db, dada2b_species_db_info *info) {
  if (!db || !info) return 1;
  *info = db->info;
  return 0;
}

void dada2b_species_db_free(dada2b_species_db *db) {
  if (!db) return;
  cudaSetDevice(db->device);
  delete db;
}

int dada2b_species_assign(dada2b_species_db *db, const dada2b_species_seqs *seqs, int32_t try_rc, int32_t keep_genus, int32_t keep_species,
                          dada2b_species_out **out, char errbuf[DADA2B_ERRLEN]) {
  if (!out) { sp_fail(errbuf, "dada2b: NULL argument."); return 1; }
  *out = nullptr;
  return guarded(errbuf, [&] { *out = assign(db, seqs, try_rc, keep_genus, keep_species, false); });
}

void dada2b_species_free(dada2b_species_out *o) {
  if (!o) return;
  free(o->nhits); free(o->genus_n); free(o->genus_off); free(o->genus_ids); free(o->species_n); free(o->species_off);
  free(o->species_ids); free(o->hit_off); free(o->hit_refs);
  free(o);
}

int dada2b_test_species_hits(dada2b_species_db *db, const dada2b_species_seqs *seqs, int32_t try_rc, dada2b_species_out **out,
                             char errbuf[DADA2B_ERRLEN]) {
  if (!out) { sp_fail(errbuf, "dada2b: NULL argument."); return 1; }
  *out = nullptr;
  return guarded(errbuf, [&] { *out = assign(db, seqs, try_rc, 0, 0, true); });
}

}  // extern "C"
