// Host driver of libdada2b.so: the C-ABI of include/dada2b.h.  Product code.
//
// Restates the control flow of dada_uniques()/run_dada() (/root/reference/src/Rmain.cpp:30-336)
// around device kernels (dd_kernels.cu).  The only state kept on the host is what the
// reference's tie-breaks depend on and what is O(moves), not O(nraw): the per-cluster member
// arrays with their slot order (Bi::raw; swap-with-last pops, containers.cpp:183-197) and the
// per-cluster birth records.  Every O(nraw) / O(pairs) computation runs on the GPU.
// There is NO CPU fallback: without a CUDA device every entry point returns an error.
#include "../../include/dada2b.h"
#include "../../include/dada2b_test.h"
#include <memory>
#include <stdexcept>
#include <dlfcn.h>
#include <nccl.h>
#include "dd_common.h"
#include "dd_kernels.h"
#include "dd_ctx.h"

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#if defined(__SSE2__)
#include <emmintrin.h>
#endif
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>

using namespace dd2;

namespace {

struct Err { std::string msg; };
double now_ms();
// DADA2B_STALLWATCH=<ms> (diagnostics): report every CUDA runtime call of the driver that takes longer
// than <ms>, and every stretch of host code between two calls that does
struct StallWatch {
  double thr = 0, last_end = 0;
  StallWatch() { if (const char *e = getenv("DADA2B_STALLWATCH")) thr = atof(e); }
  double begin(const char *what) {
    const double t = now_ms();
    if (last_end != 0 && t - last_end > thr) fprintf(stderr, "[dada2b] stall: %.1f ms of host time before %s\n", t - last_end, what);
    return t;
  }
  void end(const char *what, double t0) {
    const double t = now_ms();
    if (t - t0 > thr) fprintf(stderr, "[dada2b] stall: %.1f ms inside %s\n", t - t0, what);
    last_end = t;
  }
};
static StallWatch g_watch;
#define CK(x) do { const double w0_ = g_watch.thr > 0 ? g_watch.begin(#x) : 0.0; cudaError_t e_ = (x); if (g_watch.thr > 0) g_watch.end(#x, w0_); \
                   if (e_ != cudaSuccess) throw Err{std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " #x}; } while (0)

#define TDBG(msg) do { if (getenv("DADA2B_VERBOSE")) fprintf(stderr, "[dada2b] t=%.3f ms %s\n", now_ms() - g_t0, msg); } while (0)
#define DBG(...) do { if (getenv("DADA2B_SYNCDEBUG")) { fprintf(stderr, "[dada2b] " __VA_ARGS__); fprintf(stderr, "\n"); } } while (0)
double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static double g_t0 = 0;
double na_real() { union { double d; uint64_t u; } v; v.u = 0x7FF00000000007A2ULL; return v.d; }

template <typename T> struct DBuf {   // device buffer (grow-only: reused across runs of a context)
  T *p = nullptr; size_t n = 0, cap = 0;
  void alloc(size_t count) {
    if (count <= cap && p) { n = count; return; }
    free(); n = cap = count;
    if (count) CK(cudaMalloc(&p, count * sizeof(T)));
  }
  void free() { if (p) cudaFree(p); p = nullptr; n = cap = 0; }
  void zero(cudaStream_t s) { if (n) CK(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
  void swap(DBuf &o) { std::swap(p, o.p); std::swap(n, o.n); std::swap(cap, o.cap); }
  ~DBuf() { free(); }
};
template <typename T> struct PBuf {   // pinned host buffer (grow-only)
  T *p = nullptr; size_t n = 0, cap = 0;
  void alloc(size_t count) {
    if (count <= cap && p) { n = count; return; }
    free(); n = cap = count;
    if (count) CK(cudaMallocHost(&p, count * sizeof(T)));
  }
  void free() { if (p) cudaFreeHost(p); p = nullptr; n = cap = 0; }
  ~PBuf() { free(); }
};

// (uint8_t) round(x) of a row of qualities (containers.cpp:34), returns the row's largest value.  For x >= 0: t = trunc(x) and
// x - t are both exact in fp64, and round() (half away from zero) is t + (x - t >= 0.5) -- unlike (int)(x + 0.5), whose sum rounds
// up to 1.0 for the double just below 0.5.  Negative / NaN / out-of-int-range values go through round() and the cast themselves.
// 2 GB of doubles per 1e6 uniques pass through here on every upload: eight at a time with SSE2 (baseline x86-64; cvttpd2dq has
// cvttsd2si's semantics per lane, so the out-of-range cases agree with the scalar cast as well).
inline uint8_t round_qual(double x) {
  int rv = (int)x;
  if (x - (double)rv >= 0.5) rv++;
  if (!(x >= 0 && x < 2147483648.0)) rv = (int)round(x);           // negative, NaN, beyond int: whatever the plain cast gives
  return (uint8_t)rv;
}
inline int round_quals_row(const double *src, uint8_t *q, int L) {
  int mq = 0, p = 0;
#if defined(__SSE2__)
  const __m128d half = _mm_set1_pd(0.5), zero = _mm_setzero_pd(), big = _mm_set1_pd(2147483648.0);
  __m128i vmax = _mm_setzero_si128();
  for (; p + 8 <= L; p += 8) {
    __m128i r[4];
    int ok = 3;
    for (int k = 0; k < 4; k++) {
      const __m128d x = _mm_loadu_pd(src + p + 2 * k);
      ok &= _mm_movemask_pd(_mm_and_pd(_mm_cmpge_pd(x, zero), _mm_cmplt_pd(x, big)));   // false for negative, NaN and huge lanes
      const __m128i rv = _mm_cvttpd_epi32(x);                           // two int32 in the low half
      const __m128d f = _mm_sub_pd(x, _mm_cvtepi32_pd(rv));
      const __m128i up = _mm_castpd_si128(_mm_cmpge_pd(f, half));       // all-ones 64-bit lanes where the fraction is >= 0.5
      r[k] = _mm_sub_epi32(rv, _mm_shuffle_epi32(up, _MM_SHUFFLE(3, 3, 2, 0)));     // - (-1) in the matching 32-bit lanes 0 and 1
    }
    if (ok != 3) { for (int u = 0; u < 8; u++) { const uint8_t v = round_qual(src[p + u]); q[p + u] = v; if (v > mq) mq = v; } continue; }
    const __m128i lo = _mm_unpacklo_epi64(r[0], r[1]), hi = _mm_unpacklo_epi64(r[2], r[3]);
    const __m128i m = _mm_set1_epi32(0xFF);                              // (uint8_t) truncation
    const __m128i w = _mm_packs_epi32(_mm_and_si128(lo, m), _mm_and_si128(hi, m));
    const __m128i b = _mm_packus_epi16(w, w);
    _mm_storel_epi64((__m128i *)(q + p), b);
    vmax = _mm_max_epu8(vmax, b);
  }
  uint8_t tmp[16];
  _mm_storeu_si128((__m128i *)tmp, vmax);
  for (int u = 0; u < 8; u++) if (tmp[u] > mq) mq = tmp[u];
#endif
  for (; p < L; p++) { const uint8_t v = round_qual(src[p]); q[p] = v; if (v > mq) mq = v; }
  return mq;
}

// 2-bit packing of one read (DevIn::seq2: base b at bits 2(b%16) of word b/16; A,C,G,T = 0..3), returns 1 when a character
// other than ACGT was seen (it packs as A; the caller turns the flag into the reference's error, misc.cpp:6-24).
// 250 MB of bases per 1e6 uniques: sixteen at a time with SSE2 -- (c >> 1) & 3 maps A,C,G,T to 0,1,3,2 and t ^ (t >> 1) to
// 0,1,2,3; the sixteen 2-bit fields are then folded together by shift-or steps.  A per-character switch costs a mispredicted
// branch on most bases.
inline int pack_bases_row(const char *s, uint32_t *row, int L, int SW) {
  int p = 0, w = 0, bad = 0;
#if defined(__SSE2__)
  const __m128i cA = _mm_set1_epi8('A'), cC = _mm_set1_epi8('C'), cG = _mm_set1_epi8('G'), cT = _mm_set1_epi8('T');
  const __m128i m3 = _mm_set1_epi8(3), m1 = _mm_set1_epi8(1), mF = _mm_set1_epi16(0x000F);
  for (; p + 16 <= L; p += 16, w++) {
    const __m128i v = _mm_loadu_si128((const __m128i *)(s + p));
    const __m128i okv = _mm_or_si128(_mm_or_si128(_mm_cmpeq_epi8(v, cA), _mm_cmpeq_epi8(v, cC)), _mm_or_si128(_mm_cmpeq_epi8(v, cG), _mm_cmpeq_epi8(v, cT)));
    if (_mm_movemask_epi8(okv) != 0xFFFF) break;                         // finish this read character by character
    const __m128i t = _mm_and_si128(_mm_srli_epi16(v, 1), m3);
    const __m128i c = _mm_xor_si128(t, _mm_and_si128(_mm_srli_epi16(t, 1), m1));          // one 2-bit code per byte
    const __m128i n = _mm_and_si128(_mm_or_si128(c, _mm_srli_epi16(c, 6)), mF);           // two codes per 16-bit lane
    const __m128i b = _mm_packus_epi16(n, n);                                             // eight bytes, a nibble each
    uint64_t q = (uint64_t)_mm_cvtsi128_si64(b);
    q = (q | (q >> 4)) & 0x00FF00FF00FF00FFull;
    q = (q | (q >> 8)) & 0x0000FFFF0000FFFFull;
    q = (q | (q >> 16));
    row[w] = (uint32_t)q;
  }
#endif
  for (int x = w; x < SW; x++) row[x] = 0;
  for (; p < L; p++) {
    unsigned code;
    switch (s[p]) { case 'A': code = 0; break; case 'C': code = 1; break; case 'G': code = 2; break;
                    case 'T': code = 3; break; default: code = 0; bad = 1; }
    row[p >> 4] |= code << (2 * (p & 15));
  }
  return bad;
}

template <typename F> void parallel_for(size_t n, F f) {
  unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
  if (n < 4096 || nt == 1) { f(0, n); return; }
  std::vector<std::thread> th;
  size_t chunk = (n + nt - 1) / nt;
  for (unsigned t = 0; t < nt; t++) {
    size_t b = t * chunk, e = std::min(n, b + chunk);
    if (b >= e) break;
    th.emplace_back([=]() { f(b, e); });
  }
  for (auto &t : th) t.join();
}

}  // namespace

namespace {
struct Run; void delete_run(Run *);
// NCCL is resolved at run time from the process (torch's bundled libnccl.so.2 when present): single-GPU use has no
// NCCL dependency at all.
struct NcclApi {
  void *h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool load(std::string &why) {
    if (h) return true;
    for (const char *name : {"libnccl.so.2", "libnccl.so"}) { h = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
    if (!h) { why = "dada2b: cannot load libnccl.so.2"; return false; }
    GetUniqueId = (decltype(GetUniqueId))dlsym(h, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(h, "ncclCommInitRank");
    AllGather = (decltype(AllGather))dlsym(h, "ncclAllGather");
    AllReduce = (decltype(AllReduce))dlsym(h, "ncclAllReduce");
    CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
    GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllGather || !AllReduce || !CommDestroy) { why = "dada2b: libnccl lacks required symbols"; return false; }
    return true;
  }
};
NcclApi g_nccl;
}  // namespace
#define NC(x) do { ncclResult_t r_ = (x); if (r_ != ncclSuccess) throw Err{std::string("NCCL error: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "?") + " at " #x}; } while (0)
struct dada2b_ctx {
  ncclComm_t comm = nullptr;      // sharded runs
  int rank = 0, world = 1;
  Run *run = nullptr;             // per-run device state, kept across runs (grow-only buffers)
  int device = 0;
  cudaStream_t stream = nullptr;
  DevIn in{};
  int maxq = 0;            // largest rounded quality present
  bool has_quals = false;
  bool bad_nt = false;
  bool qual_sharded = false;      // dada2b_reupload on a sharded context: quality rows of this rank's raws only are on the device
  DBuf<uint8_t> d_qual_own, d_seq_own, d_seq_all;
  DBuf<int> d_flags;
  unsigned total_reads = 0;
  int reads_argmax = -1;          // first raw with the largest abundance (bi_assign_center of the initial cluster), -1 if all are 0
  std::vector<uint16_t> len;
  std::vector<uint32_t> reads;
  std::vector<uint8_t> prior;
  DBuf<uint32_t> d_seq2, d_reads;
  DBuf<uint8_t> d_qual, d_prior;
  DBuf<uint16_t> d_len;
  PBuf<uint32_t> st_seq;          // pinned staging for the packed upload
  PBuf<uint8_t> st_qual;
  PBuf<uint8_t> st_meta;          // len (u16) | reads (u32) | prior (u8), pinned
  int num_sms = 148;
  long long upload_h2d = 0;
  unsigned long long upload_gen = 0;   // bumped by every (re)upload: per-sequence tables derived on the device are rebuilt when it changes
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_next = 0;
  cudaEvent_t get_event() {
    if (ev_next == ev_pool.size()) { cudaEvent_t e; cudaEventCreate(&e); ev_pool.push_back(e); }
    return ev_pool[ev_next++];
  }
};

// SMs the dada() path sizes its grids from: the device's count, or fewer under DADA2B_SMS=<n> (test hook: with a small cap,
// golden-sized inputs give every CTA of the grid-stride kernels several tiles / jobs, as 1e6-unique runs do on all SMs).
// Every grid is min(work, k * SMs) with a floor of one CTA, so any cap >= 1 is valid.
static int dada_sms(int device) {
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  if (const char *e = getenv("DADA2B_SMS")) {
    const int cap = atoi(e);
    if (cap < 1) throw Err{"dada2b: DADA2B_SMS must be a positive integer"};
    sms = std::min(sms, cap);
  }
  return sms;
}

// ------------------------------------------------------------------------------------
// upload: validation of Rmain.cpp:52-78, raw_new (containers.cpp:19-43) and packing
// ------------------------------------------------------------------------------------
static dada2b_ctx *do_upload(const dada2b_in *in, int device, dada2b_ctx *reuse = nullptr) {
  const unsigned nraw = in->nraw;
  const double tu0 = now_ms();
  DBG("upload: nraw=%u", nraw);
  if (in->nraw <= 0) throw Err{"Zero input sequences."};
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    throw Err{"dada2b: no CUDA device available (this library has no CPU path)."};
  CK(cudaSetDevice(device));
  std::unique_ptr<dada2b_ctx> fresh;
  dada2b_ctx *cx = reuse;
  if (!cx) {
    fresh.reset(new dada2b_ctx());
    cx = fresh.get();
    cx->device = device;
    cx->num_sms = dada_sms(device);
    CK(cudaStreamCreateWithFlags(&cx->stream, cudaStreamNonBlocking));
  }
  DBG("upload: device ready, %d SMs", cx->num_sms);
  // validate everything into locals first: a failed dada2b_reupload() must leave the live context untouched
  unsigned maxlen = 0, minlen = 9999;
  std::vector<uint16_t> len_new(nraw);
  for (unsigned i = 0; i < nraw; i++) {
    int64_t l = in->seq_off[i + 1] - in->seq_off[i];
    if (l < 0) throw Err{"Bad sequence offsets."};
    if (l >= 9999) throw Err{"Input sequences exceed the maximum allowed string length."};
    len_new[i] = (uint16_t)l;
    maxlen = std::max<unsigned>(maxlen, (unsigned)l); minlen = std::min<unsigned>(minlen, (unsigned)l);
  }
  if (maxlen >= 9999) throw Err{"Input sequences exceed the maximum allowed string length."};
  if (minlen <= (unsigned)KMER) throw Err{"Input sequences must all be longer than the kmer-size (5)."};
  if (!(in->maxlen > 0 && in->quals != nullptr))
    throw Err{"A quality matrix is required (the reference dereferences raw->qual unconditionally, error.cpp:160)."};
  if ((unsigned)in->maxlen != maxlen) throw Err{"Sequence must have associated qualities for each nucleotide position."};
  cx->len.swap(len_new);
  cx->maxq = 0; cx->bad_nt = false; cx->has_quals = true;
  DevIn &d = cx->in;
  d.nraw = nraw; d.maxlen = maxlen; d.minlen = minlen;
  d.SW = (((int)maxlen + 15) / 16 + 3) & ~3;
  d.QS = ((int)maxlen + 15) & ~15;
  cx->reads.resize(nraw); cx->prior.resize(nraw);             // filled below, by the calling thread while the workers pack
  // pack on the host into pinned staging, then one H2D per array
  const double tu1 = now_ms();
  PBuf<uint32_t> &h_seq = cx->st_seq;
  // a context that already shards a sample (dada2b_reupload after dada2b_comm_init) needs the quality rows of ITS raws only:
  // they are packed densely (row it <-> raw it * world + rank) and scattered into place on the device
  const bool qshard = reuse && cx->comm && cx->world > 1;
  const unsigned qworld = qshard ? (unsigned)cx->world : 1u, qrank = qshard ? (unsigned)cx->rank : 0u;
  const size_t nqown = ((size_t)nraw + qworld - 1 - qrank) / qworld;
  const size_t nqmax = ((size_t)nraw + qworld - 1) / qworld;          // rows of the largest shard (all-gather chunks are equally long)
  PBuf<uint8_t> &h_qual = cx->st_qual; h_qual.alloc(std::max<size_t>(nqown, 1) * d.QS);
  h_seq.alloc(qshard ? nqmax * d.SW : (size_t)nraw * d.SW);          // sharded: this rank packs its own reads only, the rest arrives over NVLink
  std::vector<int> tmaxq(64, 0), tbad(64, 0);
  const char *sc = in->seq_concat;                                    // read in place: no host copy of the strings is kept (finish() decodes the packed rows)
  const int64_t *soff = in->seq_off;
  const double *qd = in->quals;
  const int SW = d.SW, QS = d.QS, ML = in->maxlen;
  cx->d_seq2.alloc((size_t)nraw * d.SW); cx->d_qual.alloc((size_t)nraw * d.QS);
  cx->d_len.alloc(nraw); cx->d_reads.alloc(nraw); cx->d_prior.alloc(nraw);
  cx->st_meta.alloc((size_t)nraw * 8);                                // reads (u32) | len (u16) | prior (u8), pinned
  const size_t seq_chunk = nqmax * d.SW * 4;                          // sharded: bytes of one rank's all-gather chunk
  uint8_t *seq_dst = (uint8_t *)cx->d_seq2.p, *qual_dst = cx->d_qual.p;
  if (qshard) {
    cx->d_seq_own.alloc(seq_chunk); cx->d_seq_all.alloc(seq_chunk * qworld); cx->d_qual_own.alloc(nqown * d.QS);
    CK(cudaMemsetAsync(cx->d_seq_own.p, 0, seq_chunk, cx->stream));
    seq_dst = cx->d_seq_own.p; qual_dst = cx->d_qual_own.p;
  }
  // Packing and the H2D copies are pipelined: worker threads take blocks of PACK_BLK raws from a counter, the calling thread
  // sends every group of PACK_GRP finished blocks on its way while the later ones are still being packed (pinned staging, one
  // stream: the copies arrive in order).  own(x) = how many of the raws below x are packed by this rank = their staging row.
  auto own = [&](size_t x) { return (x + qworld - 1 - qrank) / qworld; };
  size_t PACK_BLK = 4096; const size_t PACK_GRP = 16;
  if (const char *e = getenv("DADA2B_PACK_BLK")) PACK_BLK = (size_t)std::max(1, atoi(e));      // test hook: many blocks / groups on small inputs
  const size_t nblk = ((size_t)nraw + PACK_BLK - 1) / PACK_BLK;
  std::unique_ptr<std::atomic<int>[]> blk_done(new std::atomic<int>[nblk]);
  for (size_t k = 0; k < nblk; k++) blk_done[k].store(0, std::memory_order_relaxed);
  std::atomic<size_t> blk_next{0};
  {
    unsigned nt = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    if (nraw < 20000) nt = std::min(nt, 4u);
    nt = (unsigned)std::min<size_t>(nt, nblk);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; t++) {
      th.emplace_back([&, t]() {
        int mq = 0, bad = 0;
        for (;;) {
          const size_t k = blk_next.fetch_add(1, std::memory_order_relaxed);
          if (k >= nblk) break;
          const size_t b = k * PACK_BLK, e = std::min<size_t>(nraw, b + PACK_BLK);
          for (size_t r = b; r < e; r++) {
            if (r % qworld != qrank) continue;                     // not this rank's read (sharded re-upload)
            const char *s = sc + soff[r];
            const int L = cx->len[r];
            bad |= pack_bases_row(s, h_seq.p + (r / qworld) * SW, L, SW);
            uint8_t *q = h_qual.p + (r / qworld) * QS;
            mq = std::max(mq, round_quals_row(qd + (size_t)ML * r, q, L));      // (uint8_t) round(qual[i]), containers.cpp:34
            for (int p = L; p < QS; p++) q[p] = 0;
          }
          blk_done[k].store(1, std::memory_order_release);
        }
        tmaxq[t] = mq; tbad[t] = bad;
      });
    }
    cudaError_t copy_err = cudaSuccess;
    {  // meanwhile: abundances / priors / lengths (7 bytes per raw) from the calling thread
      unsigned tot = 0, mx = 0;
      int amax = -1;
      uint8_t *m = cx->st_meta.p;
      uint32_t *m_reads = (uint32_t *)m; uint8_t *m_prior = m + (size_t)nraw * 6;
      for (unsigned i = 0; i < nraw; i++) {
        const uint32_t rd = (uint32_t)in->abund[i];
        const uint8_t pr = in->prior ? (in->prior[i] != 0) : 0;
        cx->reads[i] = rd; cx->prior[i] = pr; m_reads[i] = rd; m_prior[i] = pr;
        tot += rd;                                              // unsigned int accumulation, containers.cpp:100
        if (rd > mx) { mx = rd; amax = (int)i; }
      }
      cx->total_reads = tot; cx->reads_argmax = amax;
      memcpy(m + (size_t)nraw * 4, cx->len.data(), (size_t)nraw * 2);
      copy_err = cudaMemcpyAsync(cx->d_reads.p, m, (size_t)nraw * 4, cudaMemcpyHostToDevice, cx->stream);
      if (copy_err == cudaSuccess) copy_err = cudaMemcpyAsync(cx->d_len.p, m + (size_t)nraw * 4, (size_t)nraw * 2, cudaMemcpyHostToDevice, cx->stream);
      if (copy_err == cudaSuccess) copy_err = cudaMemcpyAsync(cx->d_prior.p, m + (size_t)nraw * 6, nraw, cudaMemcpyHostToDevice, cx->stream);
    }
    for (size_t g = 0; g < nblk; g += PACK_GRP) {
      const size_t ge = std::min(nblk, g + PACK_GRP);
      for (size_t k = g; k < ge; k++)
        while (!blk_done[k].load(std::memory_order_acquire)) std::this_thread::sleep_for(std::chrono::microseconds(50));
      const size_t r0 = own(g * PACK_BLK), r1 = own(std::min<size_t>(nraw, ge * PACK_BLK));
      if (r1 == r0 || copy_err != cudaSuccess) continue;             // (after an error: only wait for the workers)
      copy_err = cudaMemcpyAsync(seq_dst + r0 * SW * 4, h_seq.p + r0 * SW, (r1 - r0) * SW * 4, cudaMemcpyHostToDevice, cx->stream);
      if (copy_err == cudaSuccess)
        copy_err = cudaMemcpyAsync(qual_dst + r0 * QS, h_qual.p + r0 * QS, (r1 - r0) * QS, cudaMemcpyHostToDevice, cx->stream);
    }
    for (auto &x : th) x.join();
    CK(copy_err);
  }
  const double tu2 = now_ms();
  DBG("upload: packed on host");
  for (int v : tmaxq) cx->maxq = std::max(cx->maxq, v);
  for (int v : tbad) cx->bad_nt |= (v != 0);
  if (qshard) {   // own packed reads are up: everybody's over NVLink (one all-gather), rows scattered into raw order
    NC(g_nccl.AllGather(cx->d_seq_own.p, cx->d_seq_all.p, seq_chunk, ncclChar, cx->comm, cx->stream));
    for (unsigned q = 0; q < qworld; q++) {
      const size_t nq = ((size_t)nraw + qworld - 1 - q) / qworld;
      launch_qrows_scatter((uint8_t *)cx->d_seq2.p, d.SW * 4, nullptr, (int)nq, (int)q, (int)qworld, cx->d_seq_all.p + seq_chunk * q, cx->stream);
    }
    launch_qrows_scatter(cx->d_qual.p, d.QS, nullptr, (int)nqown, (int)qrank, (int)qworld, cx->d_qual_own.p, cx->stream);
    // the largest quality present decides an error of the whole call (Rmain.cpp / pval.cpp:169-171): every rank must see the same value
    DBuf<int> &dq = cx->d_flags; dq.alloc(2);                    // member: no cudaMalloc / cudaFree per re-upload
    int hq[2] = {cx->maxq, cx->bad_nt ? 1 : 0};                  // ... and so does an unexpected nucleotide in anybody's reads
    CK(cudaMemcpyAsync(dq.p, hq, 8, cudaMemcpyHostToDevice, cx->stream));
    NC(g_nccl.AllReduce(dq.p, dq.p, 2, ncclInt32, ncclMax, cx->comm, cx->stream));
    CK(cudaMemcpyAsync(hq, dq.p, 8, cudaMemcpyDeviceToHost, cx->stream));
    CK(cudaStreamSynchronize(cx->stream));
    cx->maxq = hq[0]; cx->bad_nt = hq[1] != 0;
  }
  cx->qual_sharded = qshard;
  CK(cudaStreamSynchronize(cx->stream));
  if (getenv("DADA2B_VERBOSE")) fprintf(stderr, "[dada2b] upload: validate+copy %.2f ms, pack %.2f ms, alloc+H2D %.2f ms\n", tu1 - tu0, tu2 - tu1, now_ms() - tu2);
  DBG("upload: H2D done");
  cx->upload_h2d = (long long)(qshard ? nqown : nraw) * (d.SW * 4 + d.QS) + (long long)nraw * 7;
  cx->upload_gen++;
  d.seq2 = cx->d_seq2.p; d.qual = cx->d_qual.p; d.len = cx->d_len.p; d.reads = cx->d_reads.p; d.prior = cx->d_prior.p;
  if (fresh) fresh.release();
  return cx;
}

// Device-resident constructor (dd_ctx.h): the uniques come from kernels of another driver (dereplication), not from the host.
namespace dd2 {
dada2b_ctx *ctx_create_device(int device, int nraw, int maxlen, int minlen, const char *seq_concat, const int64_t *seq_off,
                              const int32_t *abund, DevIn *arrays, cudaStream_t *stream) {
  try {
    if (nraw <= 0) throw Err{"Zero input sequences."};
    if (maxlen >= 9999) throw Err{"Input sequences exceed the maximum allowed string length."};
    if (minlen <= KMER) throw Err{"Input sequences must all be longer than the kmer-size (5)."};
    CK(cudaSetDevice(device));
    std::unique_ptr<dada2b_ctx> cx(new dada2b_ctx());
    cx->device = device;
    cx->num_sms = dada_sms(device);
    CK(cudaStreamCreateWithFlags(&cx->stream, cudaStreamNonBlocking));
    cx->has_quals = true; cx->bad_nt = false; cx->maxq = 0;
    cx->len.resize(nraw); cx->reads.resize(nraw); cx->prior.assign(nraw, 0);
    unsigned tot = 0, mx = 0;
    for (int i = 0; i < nraw; i++) {
      cx->len[i] = (uint16_t)(seq_off[i + 1] - seq_off[i]);
      cx->reads[i] = (uint32_t)abund[i]; tot += cx->reads[i];
      if (cx->reads[i] > mx) { mx = cx->reads[i]; cx->reads_argmax = i; }
    }
    cx->total_reads = tot;
    DevIn &d = cx->in;
    d.nraw = nraw; d.maxlen = maxlen; d.minlen = minlen;
    d.SW = ((maxlen + 15) / 16 + 3) & ~3;
    d.QS = (maxlen + 15) & ~15;
    cx->d_seq2.alloc((size_t)nraw * d.SW); cx->d_qual.alloc((size_t)nraw * d.QS);
    cx->d_len.alloc(nraw); cx->d_reads.alloc(nraw); cx->d_prior.alloc(nraw);
    d.seq2 = cx->d_seq2.p; d.qual = cx->d_qual.p; d.len = cx->d_len.p; d.reads = cx->d_reads.p; d.prior = cx->d_prior.p;
    cx->upload_h2d = 0;
    *arrays = d; *stream = cx->stream;
    return cx.release();
  } catch (Err &e) { throw std::runtime_error(e.msg); }
}
void ctx_finish_device(dada2b_ctx *ctx, int maxq) { ctx->maxq = maxq; }
}  // namespace dd2

// ------------------------------------------------------------------------------------
namespace {

struct Birth {                     // Bi birth_* fields, dada.h:99-104
  char type = 'I';
  uint32_t from = 0;
  double pval = 0, fold = 1, e = 0;
  uint32_t comp_i = 0, comp_index = 0, comp_ham = 0;
  double comp_lambda = 0;
};

struct Run {
  dada2b_ctx *cx;
  const dada2b_opts *o;
  cudaStream_t s;
  DevIn in;
  AlnParams P{};
  DevState st{};
  int nraw, ncol;
  // device state buffers
  DBuf<uint8_t> lock, is_center, slot0, correct, cl_update_e, cl_check_locks, b_nt0, b_nt1, b_q1, b_ops, kind_out;
  DBuf<double> E_minmax, p, comp_lambda, cs_lambda, err, b_lambda, trip_v, pa_E, pa_out;
  DBuf<uint32_t> comp_ham, cluster_of, cs_index, cs_i, cs_ham, cl_reads, cl_center, nw_list, gl_list,
      nsubs_final, ptr_scratch, pair_centre, pair_raw, b_nsubs, b_nops, trip_ij;
  DBuf<uint16_t> b_pos;
  DBuf<unsigned long long> ctr, cq_sum, cq_cnt;
  DBuf<int> trans, center_cluster, pa_reads, pa_prior;
  PBuf<unsigned long long> h_ctr;
  DBuf<uint32_t> pinfo;
  // Report and move list share ONE device buffer [RoundReport | moves], so that the round's copy back (sharded: its all-gather)
  // carries the report together with the first `eager` moves of every rank: the move lists need a copy (collective) of their own
  // only in the few rounds that move more (one call + one host synchronisation less per round).
  DBuf<uint8_t> d_repmv, d_gather_all;
  PBuf<uint8_t> h_gather_all;
  static constexpr size_t RR_PAD = (sizeof(RoundReport) + 15) & ~(size_t)15;
  unsigned eager = 0;
  std::vector<const RoundReport *> rep_all;   // every rank's report of the round (pinned host copy)
  PBuf<RoundReport> h_report_buf;
  PBuf<uint32_t> h_moves_buf;
  RoundReport *h_report = nullptr;       // the ranks' reports merged, refreshed once per round
  uint32_t *h_moves = nullptr;
  int NP = 3;                            // shuffle passes launched speculatively per round
  unsigned move_cap = 0;
  DBuf<uint32_t> fb_list, surv_list, uneq_list;
  DBuf<unsigned long long> uneq_ctr;
  DBuf<double> raw_S, raw_rho;           // two-phase loop NW: per-raw bound factors (dd_round.cu:k_raw_bounds)
  DBuf<uint32_t> row_mv;                 // thread-per-pair exact NW (dd_nwrow.cu): per-thread scratch columns for the moves ...
  DBuf<uint16_t> row_sub;                // ... and the substitutions found by the traceback
  int row_grid_cap = 0;
  DBuf<uint32_t> lane_mv;                // lane-group fused NW for small rounds (dd_nwlane.cu): scratch for LANE_MAX pairs in flight
  DBuf<uint16_t> lane_sub;
  unsigned long long lane_max = 0;
  // streaming tier of the k-mer screen (dd_prescreen.cu): 5-mer presence bitmaps of this rank's raws, candidates per round
  DBuf<uint32_t> kbits, kmeta, cand_list, old_list;
  DBuf<uint16_t> krep, cand_ms;
  // scratch of the rare paths and of finish(): members, so that a steady-state pass makes no cudaMalloc / cudaFree (those go through the
  // kernel driver and wait behind whatever else holds its lock, e.g. a monitoring agent polling the GPU)
  DBuf<uint32_t> tie_d1, tie_d2, tie_g1, tie_g2, fin_nwl, fin_gll, fin_sij, fin_gij;
  DBuf<unsigned long long> win_buf, fin_dcount, fin_dall, fin_keep;
  DBuf<uint32_t> fin_tl;                // per-cluster tallies of finish(): abundance, n0, n1, nunq, largest member reads (dd_final.cu)
  DBuf<int32_t> fin_map;
  DBuf<uint8_t> fin_cq, fin_rep_d;
  DBuf<uint32_t> fin_rep_rows;
  DBuf<uint32_t> ft_off, ft_chk, ft_cur, ft_ord, ft_sums;   // k_final_tally's per-cluster offsets and cluster-ordered raws (dd_final.cu)
  PBuf<uint8_t> fin_rep_h;          // representative sequences of the clusters: row list up, packed rows back
  DBuf<double> fin_sv, fin_gv;
  bool prescreen = false;
  unsigned long long kbits_gen = ~0ull;
  unsigned n_ovf = 0;                     // this rank's raws whose repeated-5-mer list overflowed (they alone need the warp-per-pair screen)
  DBuf<unsigned> d_novf;   // dada2b_ctx::upload_gen the k-mer tables were built for
  int nown = 0;
  // the shard (raw it * scr_world + scr_rank) and SM count the k-mer screen works with: the context's in a run, the caller's in
  // the stage hook dada2b_test_screen
  int scr_rank = 0, scr_world = 1, scr_sms = 1;
  bool fallback_only = false;         // DADA2B_FALLBACK (test switch): general kernels only
  bool two_phase = false;              // bound pass first, exact lambda for the survivors only (plain gap costs)
  // round tail (dd_round2.cu): every rank keeps the stored comparisons and runs shuffle / p-update / bud scan for its own raws
  // only (one rank: every raw); sharded runs add per pass one all-reduce of the cluster read deltas, per round one all-gather of
  // the ranks' reports (bud candidates, move counts) and, when raws moved, one of the move lists.
  int tail_last = -1;                    // last shuffle pass launched in the current round
  int tail_smem_clusters = 0;            // rounds with at most this many clusters stage the tail's per-cluster state in shared memory
  DBuf<uint32_t> d_moves_all;
  PBuf<uint32_t> h_moves_all;
  TailState ts{};
  DBuf<uint32_t> t_head, t_prev, t_nmove, t_bt, t_btp;
  DBuf<int> t_delta;
  DBuf<unsigned> t_done;
  DBuf<BlkBest> t_blk;
  void tail_sync_caps();
  int fwd_slots = 0;
  unsigned long long est_active = 0;
  size_t cl_cap = 0;
  unsigned long long cs_count = 0;
  // host membership (Bi::raw with slot order) and cluster records
  // members / slot_of / cluster_of_h / cl_reads_h belong to the REPLAY side (worker thread when async_replay), cl_center_h / birth /
  // nclust_h to the round loop.  The round loop only reads the replay side after drain_replay().
  std::vector<std::vector<uint32_t>> members;
  std::vector<uint32_t> slot_of, cluster_of_h, cl_center_h, cl_reads_h;
  std::vector<Birth> birth;
  int nclust_h = 0;
  // b_shuffle2's container updates and b_bud's pop / new cluster are pure host bookkeeping (O(moves), but ~30 ms of a 1e6-unique
  // run): the device reports everything the next bud decision needs unless it is an exact tie, so the updates
  // are queued to a worker and applied while the GPU runs the next round.  kind: 0 moves, 1 bud, 2 cluster 0's member arrays.
  struct ReplayEvent { int kind; std::vector<uint32_t> mv; std::vector<uint32_t> pass_end; uint32_t r, from, ni; };
  bool async_replay = false;
  std::thread rworker;
  std::mutex rmu;
  std::condition_variable rcv, rdone;
  std::deque<ReplayEvent> rq;
  bool rbusy = false, rquit = false;
  void apply_moves(const uint32_t *mv, size_t n);
  void apply_bud(uint32_t r, uint32_t from);
  void init_members();
  void push_event(ReplayEvent &&e);
  void drain_replay();
  void stop_replay();
  ~Run() { stop_replay(); }
  // align launch geometry
  int warp_words = 0, seq_bytes = 0, H_words = 0, ops_words = 0, ptr_in_smem = 0, align_grid = 0;
  unsigned long long ptr_words = 0;
  size_t align_smem = 0, align_smem_final = 0, classify_smem = 0;
  int kord_words = 0;
  // stats
  int n_rounds = 0, n_shuffles = 0;
  unsigned long long tot_nw = 0, tot_gl = 0;
  bool count_round = false;
  long long h2d_bytes = 0, d2h_bytes = 0, launches0 = 0;
  struct Ev { cudaEvent_t a, b; int tag; };
  std::vector<Ev> evs;
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
  // final pass: T_FROW = k_nwrow<FINAL> / k_nwfwd (nsubs + path class), T_FDIAG = the diagonal list, T_FGAP = the gapped list
  enum { T_CLASSIFY = 0, T_NW, T_GL, T_FROW, T_FDIAG, T_FGAP, T_NWB, T_PRE, T_TAIL, T_N };
  long long prescreen_rows = 0;
  template <typename F> void timed(int tag, F f) {
    Ev e{cx->get_event(), cx->get_event(), tag};
    cudaEventRecord(e.a, s); f(); cudaEventRecord(e.b, s);
    evs.push_back(e);
  }
  // All host<->device copies go through a pinned arena: cudaMemcpyAsync on pageable memory is staged by the
  // driver and was observed to stall for 10-1000 ms at a time on a loaded host.
  PBuf<uint8_t> arena;
  size_t arena_off = 0;
  struct PendingD2H { void *dst; const void *src; size_t n; };
  std::vector<PendingD2H> pend;
  void sync() {
    CK(cudaStreamSynchronize(s));
    for (const PendingD2H &q : pend) memcpy(q.dst, q.src, q.n);
    pend.clear();
    arena_off = 0;
  }
  uint8_t *arena_get(size_t n) {
    n = (n + 63) & ~(size_t)63;
    if (arena_off + n > arena.cap) {
      sync();                                   // every copy staged so far has completed: the arena can be reused
      if (n > arena.cap) arena.alloc(std::max<size_t>(n, 2 * arena.cap));
    }
    uint8_t *q = arena.p + arena_off;
    arena_off += n;
    return q;
  }
  void h2d(void *d, const void *h, size_t n) {
    if (!n) return;
    h2d_bytes += (long long)n;
    uint8_t *q = arena_get(n);
    memcpy(q, h, n);
    CK(cudaMemcpyAsync(d, q, n, cudaMemcpyHostToDevice, s));
  }
  void d2h(void *h, const void *d, size_t n) {
    if (!n) return;
    d2h_bytes += (long long)n;
    uint8_t *q = arena_get(n);
    CK(cudaMemcpyAsync(q, d, n, cudaMemcpyDeviceToHost, s));
    pend.push_back(PendingD2H{h, q, n});
  }
  void d2h_pinned(void *h, const void *d, size_t n) { d2h_bytes += (long long)n; CK(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, s)); }

  void bind(dada2b_ctx *c, const dada2b_opts *op, int Q) {
    cx = c; o = op; s = c->stream; in = c->in; nraw = c->in.nraw; ncol = Q;
    scr_rank = c->rank; scr_world = c->world; scr_sms = c->num_sms;
  }
  void reset_host();
  void setup_params();
  void alloc_state();
  void ensure_cluster_cap(size_t n);
  void ensure_cs_cap(unsigned long long need);
  void read_ctr() { d2h_pinned(h_ctr.p, ctr.p, CTR_N * 8); sync(); }
  void check_dev_error();
  void launch_screen(uint32_t c, uint32_t centre_reads, bool greedy, double kdist_cutoff, bool streaming);
  void launch_compare(uint32_t i, double kdist_cutoff);
  void launch_round_tail(int first_pass, int npass);
  void launch_round_tail_inner(int first_pass, int npass);
  void sync_report();
  int replay_moves(int first_pass, int last_pass);
  int decide_bud(uint32_t *r_out, uint32_t *from_out);
  struct Pending { int apply = 0; uint32_t r = 0, from = 0, newi = 0, reads = 0; } pending;
  void finish(dada2b_out *out);
  AlignArgs align_args(int mode, int kind);
  void launch_align_jobs(int mode, AlignArgs &a, unsigned long long upper);
};

void Run::reset_host() {
  stop_replay();
  members.clear(); slot_of.clear(); cluster_of_h.clear(); cl_center_h.clear(); cl_reads_h.clear(); birth.clear(); evs.clear(); nclust_h = 0;
  n_rounds = n_shuffles = 0; tot_nw = tot_gl = 0; prescreen_rows = 0; count_round = false; h2d_bytes = d2h_bytes = 0; cs_count = 0; est_active = 0; pending = Pending();
  st = DevState{};
}
void delete_run(Run *r) { delete r; }

void Run::setup_params() {
  const dada2b_opts &op = *o;
  P.match = op.match; P.mismatch = op.mismatch; P.gap = op.gap; P.hgap = op.homo_gap; P.band = op.band_size;
  // raw_align dispatch, nwalign_endsfree.cpp:57-66
  P.homo = (!op.vectorized_alignment && op.homo_gap != op.gap && op.homo_gap <= 0) ? 1 : 0;
  if (op.vectorized_alignment) {
    int m = std::min(std::min(op.mismatch, op.gap), std::min(op.match, 0));
    P.sentinel = (int)(int16_t)(INT16_MIN - m);                  // nwalign_vectorized.cpp:106
  } else P.sentinel = -9999;                                     // nwalign_endsfree.cpp:116-117
  P.use_kmers = op.use_kmers != 0; P.gapless = op.gapless != 0; P.sse = op.SSE;
  P.kdist_cutoff = op.kdist_cutoff; P.use_quals = op.use_quals != 0; P.ncol = ncol;
  // ---- k_align shared-memory layout
  const int maxlen = in.maxlen, minlen = in.minlen;
  int lbmax, rbmax;
  if (P.band < 0) { lbmax = rbmax = maxlen; }
  else { lbmax = rbmax = std::min(P.band + (maxlen - minlen), maxlen); }
  const int Wmax = lbmax + rbmax + 1;
  // band slots of dd_nwfwd.cu for the widest pair: the length difference widens ONE side of a pair's band (nwalign_endsfree.cpp:101-111)
  fwd_slots = P.band < 0 ? 1 << 20 : std::min(2 * P.band + (maxlen - minlen) + 3, ((lbmax + 1) & ~1) + rbmax + 1);
  const int nchunk = (((Wmax + 1) >> 1) + 31) >> 5;
  seq_bytes = (maxlen + 15) & ~15;
  H_words = (Wmax + 2 + 3) & ~3;
  ops_words = ((2 * maxlen) / 16 + 2 + 3) & ~3;
  ptr_words = (unsigned long long)(2 * maxlen + 2) * 2 * nchunk;
  const int base_words = 2 * (seq_bytes / 4) + H_words + ops_words;
  const size_t fixed = (size_t)16 * ncol * 8 + (size_t)16 * ncol * 4;
  ptr_in_smem = (fixed + 4 * (size_t)(base_words + ptr_words) * 4 <= 56 * 1024) ? 1 : 0;
  warp_words = base_words + (ptr_in_smem ? (int)ptr_words : 0);
  align_smem = fixed + (size_t)4 * warp_words * 4;
  if (align_smem > 200 * 1024) throw Err{"dada2b: band/sequence length too large for the alignment kernel's shared memory."};
  CK(align_set_smem(std::max<size_t>(align_smem, 48 * 1024)));
  align_grid = cx->num_sms * 8;
  kord_words = ((maxlen + 1) / 2 + 3) & ~3;
  classify_smem = (size_t)(512 + kord_words + 8 * 512 + 8 * in.SW) * 4;
  if (classify_smem > 100 * 1024) throw Err{"dada2b: sequences too long for the k-mer screen kernel."};
}

// Keeps the round tail's per-entry / per-cluster arrays as large as the comparison store and the cluster arrays.
void Run::tail_sync_caps() {
  if (t_prev.n < st.cs_cap) {
    DBuf<uint32_t> np;
    np.alloc(st.cs_cap);
    if (cs_count && t_prev.p) CK(cudaMemcpyAsync(np.p, t_prev.p, cs_count * 4, cudaMemcpyDeviceToDevice, s));
    sync();
    t_prev.swap(np);
  }
  const size_t stride = 2 * cl_cap + 4;
  if (t_delta.n < (size_t)MAX_PASS * stride) { t_delta.alloc((size_t)MAX_PASS * stride); t_delta.zero(s); }   // cleared every round by k_tail_link
  ts.cs_prev = t_prev.p; ts.rows = t_delta.p; ts.cl_cap = (uint32_t)cl_cap; ts.row_stride = (uint32_t)stride;
}

void Run::ensure_cluster_cap(size_t n) {
  if (n <= cl_cap) return;
  size_t nc = std::max<size_t>(1024, cl_cap * 2);
  while (nc < n) nc *= 2;
  DBuf<uint32_t> r2, c2; DBuf<uint8_t> u2, k2;
  r2.alloc(nc); c2.alloc(nc); u2.alloc(nc); k2.alloc(nc);
  r2.zero(s); c2.zero(s); u2.zero(s); k2.zero(s);
  if (cl_cap) {
    CK(cudaMemcpyAsync(r2.p, cl_reads.p, cl_cap * 4, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(c2.p, cl_center.p, cl_cap * 4, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(u2.p, cl_update_e.p, cl_cap, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(k2.p, cl_check_locks.p, cl_cap, cudaMemcpyDeviceToDevice, s));
  }
  sync();
  cl_reads.swap(r2); cl_center.swap(c2); cl_update_e.swap(u2); cl_check_locks.swap(k2);
  cl_cap = nc;
  st.cl_reads = cl_reads.p; st.cl_center = cl_center.p;
  st.cl_update_e = cl_update_e.p; st.cl_check_locks = cl_check_locks.p;
}

void Run::ensure_cs_cap(unsigned long long need) {
  if (need <= st.cs_cap) return;
  if (cs_index.p && need <= cs_index.cap) {   // buffers kept from an earlier run of this context
    st.cs_index = cs_index.p; st.cs_i = cs_i.p; st.cs_ham = cs_ham.p; st.cs_lambda = cs_lambda.p; st.cs_cap = cs_index.cap;
    return;
  }
  unsigned long long nc = std::max<unsigned long long>(need, st.cs_cap * 2);
  DBuf<uint32_t> a, b, c; DBuf<double> l;
  a.alloc(nc); b.alloc(nc); c.alloc(nc); l.alloc(nc);
  if (cs_count) {
    CK(cudaMemcpyAsync(a.p, cs_index.p, cs_count * 4, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(b.p, cs_i.p, cs_count * 4, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(c.p, cs_ham.p, cs_count * 4, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(l.p, cs_lambda.p, cs_count * 8, cudaMemcpyDeviceToDevice, s));
  }
  sync();
  cs_index.swap(a); cs_i.swap(b); cs_ham.swap(c); cs_lambda.swap(l);
  st.cs_index = cs_index.p; st.cs_i = cs_i.p; st.cs_ham = cs_ham.p; st.cs_lambda = cs_lambda.p; st.cs_cap = nc;
}

void Run::alloc_state() {
  const size_t n = nraw;
  arena.alloc(std::max<size_t>(8u << 20, n * 40));
  arena_off = 0; pend.clear();
  lock.alloc(n); is_center.alloc(n); slot0.alloc(n); correct.alloc(n);
  E_minmax.alloc(n); p.alloc(n); comp_lambda.alloc(n); comp_ham.alloc(n); cluster_of.alloc(n);
  nw_list.alloc(n); gl_list.alloc(n); nsubs_final.alloc(n);
  TDBG("alloc: device arrays");
  ctr.alloc(CTR_N); h_ctr.alloc(CTR_N);
  DBG("alloc: ctr done");
  move_cap = (unsigned)(4 * n + 1024); fb_list.alloc(n);
  fallback_only = getenv("DADA2B_FALLBACK") != nullptr;   // test switch: general kernels only (no row / lane kernels, no streaming screen)
  two_phase = !P.homo;
  if (two_phase) { surv_list.alloc(n); raw_S.alloc(n); raw_rho.alloc(n); uneq_list.alloc(n + 2); uneq_ctr.alloc(1); }
  if (!fallback_only && nwrow_usable(P, in.maxlen) && P.band >= 0) {
    row_grid_cap = nwrow_exact_grid(cx->num_sms, nraw);
    row_mv.alloc(nwrow_mv_words(P.band, in.maxlen, row_grid_cap)); row_sub.alloc(nwrow_sub_halfwords(in.maxlen, row_grid_cap));
    if (!uneq_list.p) { uneq_list.alloc(n + 2); uneq_ctr.alloc(1); }
    {
      lane_max = 16384;                  // job lists of at most this many NW pairs: G lanes per pair, one launch (dd_nwlane.cu)
      if (const char *e = getenv("DADA2B_LANE_MAX")) lane_max = (unsigned long long)std::max(0LL, std::min(16384LL, atoll(e)));   // test hook: exercises every size class on small inputs
      lane_max = (lane_max + 31) & ~31ull;
      if (lane_max) { lane_mv.alloc(nwlane_mv_words(P.band, in.maxlen, (int)lane_max)); lane_sub.alloc(nwlane_sub_halfwords(in.maxlen, (int)lane_max)); }
    }
  } else { row_mv.free(); row_sub.free(); lane_max = 0; }
  prescreen = P.use_kmers && !fallback_only;
  bool read_novf = false;
  if (prescreen) {
    nown = (nraw - scr_rank + scr_world - 1) / scr_world;
    kbits.alloc((size_t)nown * 32 + 32); kmeta.alloc(nown); krep.alloc((size_t)nown * 48 + 64); cand_list.alloc(nown + 32); cand_ms.alloc(nown + 32);
    old_list.alloc(nown + 32);
    if (kbits_gen != cx->upload_gen) {       // the bitmaps and repeat lists depend on the sequences only: kept across the runs of a resident sample
      d_novf.alloc(1); d_novf.zero(s);
      launch_kmer_bits(in, scr_rank, scr_world, nown, kbits.p, kmeta.p, krep.p, d_novf.p, scr_sms, s);
      d2h(&n_ovf, d_novf.p, 4);            // launch_screen reads it: synchronised below
      kbits_gen = cx->upload_gen;
      read_novf = true;
    }
  }
  if (const char *e = getenv("DADA2B_NP")) NP = std::max(1, std::min(MAX_PASS, atoi(e)));      // tuning / test override
  tail_smem_clusters = tail_smem_clusters_max();
  if (const char *e = getenv("DADA2B_TAIL_SMEM_CLUSTERS"))     // test hook: 0 = every round's tail in global memory, as past ~32 k clusters
    tail_smem_clusters = std::min(tail_smem_clusters, std::max(0, atoi(e)));
  {
    const size_t g = (size_t)tail_grid(nraw);
    t_head.alloc(n); t_nmove.alloc(MAX_PASS); t_done.alloc(1); t_blk.alloc(g); t_bt.alloc(g * TIE_MAX); t_btp.alloc(g * TIE_MAX);
    t_nmove.zero(s); t_done.zero(s);
    ts.head = t_head.p; ts.nmove_pass = t_nmove.p; ts.done = t_done.p; ts.blk = t_blk.p; ts.blk_ties = t_bt.p; ts.blk_ties_pr = t_btp.p;
    ts.rank = cx->rank; ts.world = cx->world;
  }
  pinfo.alloc(MAX_PASS + 2); pinfo.zero(s);
  d_repmv.alloc(RR_PAD + (size_t)move_cap * 8);
  // Moves carried with the report.  One GPU: enough for nearly every round without a second copy.  Sharded: 1024 per rank (an
  // untimed choice: the all-gather moves world times as much).
  eager = cx->world > 1 ? 1024 : 8192;
  if (const char *e = getenv("DADA2B_MOVES_EAGER")) eager = (unsigned)std::max(0, atoi(e));      // test hook: 0 = every move list through its own copy
  eager = std::min(eager, move_cap);
  h_report_buf.alloc(1); h_moves_buf.alloc((size_t)move_cap * 2);
  h_report = h_report_buf.p; h_moves = h_moves_buf.p;
  memset(h_report, 0, sizeof(RoundReport));
  err.alloc((size_t)16 * ncol);
  lock.zero(s); is_center.zero(s); slot0.zero(s); correct.zero(s); p.zero(s); comp_lambda.zero(s); comp_ham.zero(s);
  cluster_of.zero(s); ctr.zero(s);
  launch_fill_f64(E_minmax.p, -999.0, n, s);                      // containers.cpp:39
  TDBG("alloc: memsets queued");
  if (read_novf) sync();
  st.lock = lock.p; st.is_center = is_center.p; st.slot0 = slot0.p; st.correct = correct.p;
  st.E_minmax = E_minmax.p; st.p = p.p; st.comp_lambda = comp_lambda.p; st.comp_ham = comp_ham.p; st.cluster_of = cluster_of.p;
  st.nw_list = nw_list.p; st.gl_list = gl_list.p;
  st.ctr = ctr.p; st.err = err.p; st.nsubs_final = nsubs_final.p;
  st.pinfo = pinfo.p; st.move_cap = move_cap;
  st.shard_rank = cx->rank; st.shard_world = cx->world;
  st.report = (RoundReport *)d_repmv.p; st.moves = (uint32_t *)(d_repmv.p + RR_PAD);
  { unsigned long long nn = n; h2d(ctr.p + CTR_CS_COUNT, &nn, 8); }  // cluster 0 owns entries [0, nraw)
  st.cs_cap = 0;
  ensure_cs_cap(2ull * n + 1024);
  TDBG("alloc: cs cap");
  ensure_cluster_cap(1024);
  st.cl_reads = cl_reads.p; st.cl_center = cl_center.p;
  st.cl_update_e = cl_update_e.p; st.cl_check_locks = cl_check_locks.p;
  cl_reads.zero(s); cl_center.zero(s); cl_update_e.zero(s); cl_check_locks.zero(s);
  TDBG("alloc: cluster cap");
  if (!ptr_in_smem) {
    ptr_scratch.alloc((size_t)ptr_words * align_grid * 4);
  }
}

void Run::check_dev_error() {
  unsigned long long e = h_ctr.p[CTR_ERR];
  if (e == ERR_LAMBDA) throw Err{"Lambda out-of-range error."};                       // cluster.cpp:184
  if (e == ERR_QUAL) throw Err{"Rounded quality exceeded range of err lookup table."};  // pval.cpp:170
  if (e == ERR_TRACE) throw Err{"N-W Align out of range."};                           // nwalign_endsfree.cpp:184
}

AlignArgs Run::align_args(int mode, int kind) {
  AlignArgs a{};
  a.in = in; a.P = P; a.st = st; a.kind = kind; a.job_mul = 1; a.job_add = 0;
  a.warp_words = warp_words; a.seq_bytes = seq_bytes; a.H_words = H_words; a.ops_words = ops_words;
  a.ptr_in_smem = ptr_in_smem; a.ptr_scratch = ptr_scratch.p; a.ptr_words = ptr_words;
  (void)mode;
  return a;
}

void Run::launch_align_jobs(int mode, AlignArgs &a, unsigned long long upper) {
  if (upper == 0) return;
  int grid = (int)std::min<unsigned long long>((upper + 3) / 4, (unsigned long long)align_grid);
  launch_align(mode, a, grid, 128, align_smem, s);
}

// raw_align's k-mer screen (nwalign_endsfree.cpp:44-56) of centre c against every raw of the shard, greedy skip included
// (cluster.cpp:127-131): shrouded pairs are counted into CTR_ALIGN / CTR_SHROUD, the others are appended to st.gl_list / st.nw_list
// (CTR_GL / CTR_NW).  The caller has zeroed the round's counters.  Used by the round and by the stage hook dada2b_test_screen.
void Run::launch_screen(uint32_t c, uint32_t centre_reads, bool greedy, double kdist_cutoff, bool streaming) {
  ClassifyArgs ca{};
  ca.in = in; ca.P = P; ca.P.kdist_cutoff = kdist_cutoff; ca.mode = 0; ca.centre_idx = c; ca.centre_reads = centre_reads;
  ca.greedy = greedy; ca.lock = st.lock; ca.nw_list = st.nw_list; ca.gl_list = st.gl_list; ca.ctr = st.ctr;
  ca.kind_out = nullptr; ca.kord_words = kord_words; ca.shard_rank = scr_rank; ca.shard_world = scr_world;
  int cgrid = std::min((nraw / scr_world + 8) / 8, scr_sms * 4);
  if (streaming) {
    // stream the 128-byte bitmap rows (TMA): every pair decided exactly (presence bound, then the exact min-sum through the raw's
    // repeated-5-mer list); gapless / NW for the pairs that are not shrouded (k_kord); the warp-per-pair screen only sees raws
    // whose list overflowed
    ca.cand_list = old_list.p; ca.cand_count = st.ctr + CTR_OLD;
    timed(T_PRE, [&]() {
      launch_prescreen(in, kbits.p, kmeta.p, krep.p, nown, scr_rank, scr_world, c, centre_reads, greedy, st.lock, kdist_cutoff, cand_list.p,
                       cand_ms.p, st.ctr + CTR_CAND, st.ctr, scr_sms, s);
    });
    prescreen_rows += nown;
    timed(T_CLASSIFY, [&]() {
      launch_kord(in, ca.P, c, cand_list.p, cand_ms.p, st.ctr + CTR_CAND, st.nw_list, st.gl_list, old_list.p, st.ctr + CTR_OLD, st.ctr, (unsigned long long)nown,
                  scr_sms, s);
      if (n_ovf) launch_classify(ca, std::min(cgrid, scr_sms), 256, classify_smem, s);      // only raws whose list overflowed can be forwarded
    });
  } else
  timed(T_CLASSIFY, [&]() { launch_classify(ca, cgrid, 256, classify_smem, s); });
}

// One round on the device, no host round trip inside:
//   [apply previous bud] -> b_compare_parallel (cluster.cpp:152-204) -> NP x b_shuffle2 -> b_p_update -> b_bud scan -> report
void Run::launch_compare(uint32_t i, double kdist_cutoff) {
  const uint32_t c = cl_center_h[i];
  ensure_cs_cap(cs_count + 2ull * (unsigned long long)nraw + 1024);
  ensure_cluster_cap((size_t)nclust_h + 2);
  tail_sync_caps();
  launch_round_begin(st, pending.apply, pending.r, pending.from, pending.newi, pending.reads, s);      // zeroes the round's counters
  pending.apply = 0;
  count_round = true;
  launch_screen(c, cx->reads[c], o->greedy != 0, kdist_cutoff, prescreen && kdist_cutoff < 1.0);
  bool fwd_done = false;
  bool fb_possible = false;   // only k_nwfwd hands pairs back (those that do not fit its register band)
  if (P.band >= 0) {       // register-resident NW kernels (dd_nwrow.cu / dd_nwlane.cu / dd_nwfwd.cu); unbanded pairs: k_align below
    FwdArgs f{};
    f.in = in; f.P = P; f.st = st; f.jobs = st.nw_list; f.njobs_ptr = st.ctr + CTR_NW;
    f.centre_idx = c; f.centre_reads = cx->reads[c]; f.cluster_i = i; f.total_reads = cx->total_reads;
    f.fb_list = fb_list.p; f.fb_count = st.ctr + CTR_FB; f.seq_bytes = seq_bytes; f.mode = 0; f.job_mul = 1; f.job_add = 0;
    {  // the fast path replaces the reference's sentinel by a larger penalty: only valid while no real score can come near it
      const long worst = (long)in.maxlen * std::max(std::abs(P.mismatch), std::abs(P.match)) + std::max(std::abs(P.gap), std::abs(P.hgap)) + 16;
      f.fast_ok = (worst < std::abs((long)P.sentinel) / 2) ? 1 : 0;
    }
    const unsigned long long fwd_hint = i == 0 ? (unsigned long long)nraw : est_active;
    if (two_phase && !P.homo) {
      // pass 1: scores + substitution counts only; lambda <= S_r * rho_r^nsubs decides which pairs can pass the store rule.
      // Round 0 (E_minmax still -999, containers.cpp:39) keeps every pair, but its diagonal-path pairs still leave for
      // k_gapless_loop, so that only real gaps reach the exact pass
      FwdArgs fbnd = f;
      fbnd.raw_S = raw_S.p; fbnd.raw_rho = raw_rho.p; fbnd.surv_list = surv_list.p; fbnd.surv_count = st.ctr + CTR_SURV;
      if (!fallback_only) { fbnd.gl_out = st.gl_list; fbnd.gl_count = st.ctr + CTR_GL; }   // diagonal-path survivors -> k_gapless_loop
      // thread-per-pair row kernel (dd_nwrow.cu) for raws as long as the centre; the others come back in uneq_list
      // rounds with few pairs: one lane-group launch does bound + exact (dd_nwlane.cu); the thread-per-pair bound pass returns at once then
      bool done_row = false, done_lane = false;
      if (lane_max && row_mv.p) timed(T_NWB, [&]() { done_lane = launch_nwlane(fbnd, uneq_list.p, st.ctr + CTR_UNEQ_B, lane_mv.p, lane_sub.p, (int)cx->len[c], lane_max, (int)lane_max, s); });
      if (row_mv.p)
        timed(T_NWB, [&]() { done_row = launch_nwrow_bound(fbnd, uneq_list.p, st.ctr + CTR_UNEQ_B, (int)cx->len[c], (unsigned long long)nraw, cx->num_sms, done_lane ? lane_max : 0ull, s); });
      if (done_row) { fbnd.jobs = uneq_list.p; fbnd.njobs_ptr = st.ctr + CTR_UNEQ_B; }
      bool done_rest = done_row && in.minlen == in.maxlen;          // every raw has the centre's length: nothing was handed back
      if (!done_rest)
        timed(T_NWB, [&]() { done_rest = launch_nwfwd(fbnd, fwd_slots, (unsigned long long)nraw, done_row ? 0 : fwd_hint, cx->num_sms, s, true); fb_possible |= done_rest; });
      // pass 2: the exact forward-carry kernel on the survivors
      if (done_rest) { f.jobs = surv_list.p; f.njobs_ptr = st.ctr + CTR_SURV; f.no_cells = 1; }
    }
    // exact pass: thread-per-pair row kernel with recorded moves + traceback (dd_nwrow.cu); what it hands back (raws not as
    // long as the centre) and every configuration it does not cover go through the lane-group forward-carry kernel
    bool ex_done = false;
    if (row_mv.p) {
      // survivors of a large round are few: the lane-group kernel (lower latency) takes lists of up to lane_max jobs, the thread-per-pair
      // kernel the rest (round 0, very large survivor sets); each returns at once when the list is not its size
      bool lane2 = false;
      if (lane_max && i > 0 && two_phase) {
        FwdArgs f2 = f;
        f2.raw_S = raw_S.p; f2.raw_rho = raw_rho.p;
        timed(T_NW, [&]() { lane2 = launch_nwlane(f2, uneq_list.p, st.ctr + CTR_UNEQ_X, lane_mv.p, lane_sub.p, (int)cx->len[c], lane_max, (int)lane_max, s); });
      }
      timed(T_NW, [&]() { ex_done = launch_nwrow_exact(f, uneq_list.p, st.ctr + CTR_UNEQ_X, row_mv.p, row_sub.p, (int)cx->len[c], (unsigned long long)nraw, row_grid_cap, s, lane2 ? lane_max : 0ull); });
      if (ex_done) { f.jobs = uneq_list.p; f.njobs_ptr = st.ctr + CTR_UNEQ_X; }
    }
    if (ex_done && in.minlen == in.maxlen) fwd_done = true;       // nothing was handed back; fb_list stays empty
    else timed(T_NW, [&]() { fwd_done = launch_nwfwd(f, fwd_slots, (unsigned long long)nraw, ex_done ? 0 : fwd_hint, cx->num_sms, s); fb_possible |= fwd_done; });
  }
  if (!fallback_only) {       // gapless comparisons: no DP, one thread per pair (dd_nwrow.cu:k_gapless_loop)
    FwdArgs g{};
    g.in = in; g.P = P; g.st = st; g.jobs = st.gl_list; g.njobs_ptr = st.ctr + CTR_GL;
    g.centre_idx = c; g.centre_reads = cx->reads[c]; g.cluster_i = i; g.total_reads = cx->total_reads;
    g.raw_S = raw_S.p; g.raw_rho = raw_rho.p;
    timed(T_GL, [&]() { launch_gapless_loop(g, two_phase ? 1 : 0, (unsigned long long)nraw, cx->num_sms, s); });
  }
  for (int kind : {KIND_NW, KIND_GAPLESS}) {
    if (kind == KIND_GAPLESS && !fallback_only) continue;
    AlignArgs a = align_args(MODE_LOOP, kind);
    a.jobs = kind == KIND_NW ? st.nw_list : st.gl_list;
    if (kind == KIND_NW && fwd_done && !fb_possible) continue;        // every NW job went through the row / lane kernels: nothing to hand back
    if (kind == KIND_NW && fwd_done) { a.jobs = fb_list.p; a.njobs_ptr = st.ctr + CTR_FB; }
    else a.njobs_ptr = st.ctr + (kind == KIND_NW ? CTR_NW : CTR_GL);
    a.centre_idx = c; a.centre_reads = cx->reads[c]; a.cluster_i = i; a.total_reads = cx->total_reads;
    timed(kind == KIND_NW ? T_NW : T_GL, [&]() { launch_align_jobs(MODE_LOOP, a, (unsigned long long)nraw); });
  }
  launch_tail_link(st, ts, cs_count, i, nraw, nclust_h, s);
}

// shuffle passes [first_pass, first_pass + npass) then p-update, bud scan and the report
void Run::launch_round_tail(int first_pass, int npass) {
  timed(T_TAIL, [&]() { launch_round_tail_inner(first_pass, npass); });
}
void Run::launch_round_tail_inner(int first_pass, int npass) {
  const int nclust = nclust_h;
  const bool smem = nclust <= tail_smem_clusters;
  for (int p = first_pass; p < first_pass + npass; p++) {
    launch_tail_pass(st, in, ts, p, nclust, smem, s);
    if (cx->world > 1) NC(g_nccl.AllReduce(ts.rows + (size_t)p * ts.row_stride, ts.rows + (size_t)p * ts.row_stride, ts.row_stride, ncclInt32, ncclSum, cx->comm, s));
  }
  tail_last = first_pass + npass - 1;          // -1 => no shuffling this round (initial cluster)
  BudParams bp{o->min_fold, o->min_hamming, o->min_abund};
  bp.skip_log = log(o->omegaA / (double)(unsigned)nraw) + 1.0;                       // decide_bud: pA = p * nraw < omegaA
  bp.skip_log_prior = log(std::max(o->omegaA / (double)(unsigned)nraw, o->omegaP)) + 1.0;   // ... or p < omegaP
  if (!(bp.skip_log == bp.skip_log)) bp.skip_log = 1e300;                              // non-positive thresholds: no shortcut
  if (!(bp.skip_log_prior == bp.skip_log_prior)) bp.skip_log_prior = 1e300;
  launch_tail_final(st, in, ts, bp, o->greedy != 0, o->detect_singletons != 0, tail_last, nclust, tail_last == MAX_PASS - 1 ? 2 : 0, smem, s);
}

// Copies every rank's report back (sharded: one all-gather first), keeps the local counters, merges the bud candidates and the
// move lists so that replay_moves / decide_bud see exactly what a single-GPU run reports.  Every rank computes the same merge.
void Run::sync_report() {
  const int W = cx->world;
  const size_t G = RR_PAD + (size_t)eager * 8;                     // per rank: the report and the head of its move list
  const uint8_t *gathered = d_repmv.p;
  if (W > 1) {
    d_gather_all.alloc((size_t)W * G);
    NC(g_nccl.AllGather(d_repmv.p, d_gather_all.p, G, ncclChar, cx->comm, s));
    gathered = d_gather_all.p;
  }
  h_gather_all.alloc((size_t)W * G);
  d2h_pinned(h_gather_all.p, gathered, (size_t)W * G);
  sync();
  rep_all.resize(W);
  for (int q = 0; q < W; q++) rep_all[q] = (const RoundReport *)(h_gather_all.p + (size_t)q * G);
  struct RepView { const std::vector<const RoundReport *> &v; const RoundReport &operator[](int q) const { return *v[q]; } } rep{rep_all};
  *h_report = rep[cx->rank];
  memcpy(h_ctr.p, h_report->ctr, sizeof(unsigned long long) * CTR_N);
  for (int q = 0; q < W; q++) h_ctr.p[CTR_ERR] = std::max(h_ctr.p[CTR_ERR], rep[q].ctr[CTR_ERR]);
  check_dev_error();
  cs_count = h_report->ctr[CTR_CS_COUNT];
  if (count_round) { tot_nw += h_report->ctr[CTR_NW]; tot_gl += h_report->ctr[CTR_GL]; count_round = false; }
  est_active = std::max<unsigned long long>(1024, 2 * h_report->ctr[CTR_NW]);
  if (cs_count > st.cs_cap) throw Err{"dada2b: comparison store overflow"};
  for (int q = 0; q < W; q++) if (rep[q].ctr[CTR_NMOVE] > move_cap) throw Err{"dada2b: move list overflow"};
  // ---- moves: rank q's list is grouped by pass through its local pinfo; merge pass by pass ----
  const int last = tail_last;
  uint32_t maxM = 0;
  for (int q = 0; q < W && last >= 0; q++) maxM = std::max(maxM, rep[q].pinfo[last + 1]);
  uint32_t gp[MAX_PASS + 2] = {0};
  if (maxM) {
    const uint32_t *src = (const uint32_t *)(h_gather_all.p + RR_PAD);      // rank q's moves: src + q * stride (u32 units)
    size_t stride = G / 4;
    if (maxM > eager) {        // a round that moved more than the report's copy carries: the whole lists, padded to the longest one
      size_t m = 65536;                // grown in powers of two and kept across runs: allocation calls stall behind the kernel driver's lock
      while (m < maxM) m *= 2;
      if (W > 1 && (size_t)W * maxM * 2 > d_moves_all.cap) d_moves_all.alloc((size_t)W * m * 2);
      if ((size_t)W * maxM * 2 > h_moves_all.cap) h_moves_all.alloc((size_t)W * m * 2);
      const uint32_t *lists = st.moves;
      if (W > 1) {
        NC(g_nccl.AllGather(st.moves, d_moves_all.p, (size_t)maxM * 8, ncclChar, cx->comm, s));
        lists = d_moves_all.p;
      }
      d2h_pinned(h_moves_all.p, lists, (size_t)W * maxM * 8);
      sync();
      src = h_moves_all.p; stride = (size_t)maxM * 2;
    }
    size_t at = 0;
    for (int p = 0; p <= last; p++) {
      for (int q = 0; q < W; q++) {
        const uint32_t b = rep[q].pinfo[p], e = rep[q].pinfo[p + 1];
        if (at + (e - b) > move_cap) throw Err{"dada2b: move list overflow"};
        memcpy(h_moves + 2 * at, src + (size_t)q * stride + 2 * (size_t)b, (size_t)(e - b) * 8);
        at += e - b;
      }
      gp[p + 1] = (uint32_t)at;
    }
  }
  for (int p = 0; p <= last + 1 && p < MAX_PASS + 2; p++) h_report->pinfo[p] = gp[p];
  h_report->ctr[CTR_NMOVE] = last >= 0 ? gp[last + 1] : 0;
  // ---- bud candidates: lexicographic (p asc, reads desc) over the ranks' local optima ----
  auto merge = [&](int iP, int iR, int iN) {
    unsigned long long gmin = ~0ull, gmax = 0;
    for (int q = 0; q < W; q++) if (rep[q].ctr[iN]) gmin = std::min(gmin, rep[q].ctr[iP]);
    for (int q = 0; q < W; q++) if (rep[q].ctr[iN] && rep[q].ctr[iP] == gmin) gmax = std::max(gmax, rep[q].ctr[iR]);
    h_report->ctr[iP] = gmin; h_report->ctr[iR] = gmax;
    return std::make_pair(gmin, gmax);
  };
  auto a = merge(CTR_PMIN, CTR_RMAX, CTR_NTIE);
  auto b = merge(CTR_PMIN_PR, CTR_RMAX_PR, CTR_NTIE_PR);
  unsigned long long nt = 0, ntp = 0;
  for (int q = 0; q < W; q++) {
    if (rep[q].ctr[CTR_NTIE] && rep[q].ctr[CTR_PMIN] == a.first && rep[q].ctr[CTR_RMAX] == a.second) {
      for (unsigned long long k = 0; k < rep[q].ctr[CTR_NTIE] && k < TIE_MAX; k++)
        if (nt + k < TIE_MAX) { h_report->tie_r[nt + k] = rep[q].tie_r[k]; h_report->tie_lam[nt + k] = rep[q].tie_lam[k]; h_report->tie_ham[nt + k] = rep[q].tie_ham[k];
                                h_report->tie_cl[nt + k] = rep[q].tie_cl[k]; h_report->tie_clreads[nt + k] = rep[q].tie_clreads[k]; }
      nt += rep[q].ctr[CTR_NTIE];
    }
    if (rep[q].ctr[CTR_NTIE_PR] && rep[q].ctr[CTR_PMIN_PR] == b.first && rep[q].ctr[CTR_RMAX_PR] == b.second) {
      for (unsigned long long k = 0; k < rep[q].ctr[CTR_NTIE_PR] && k < TIE_MAX; k++)
        if (ntp + k < TIE_MAX) { h_report->tiep_r[ntp + k] = rep[q].tiep_r[k]; h_report->tiep_lam[ntp + k] = rep[q].tiep_lam[k]; h_report->tiep_ham[ntp + k] = rep[q].tiep_ham[k];
                                 h_report->tiep_cl[ntp + k] = rep[q].tiep_cl[k]; h_report->tiep_clreads[ntp + k] = rep[q].tiep_clreads[k]; }
      ntp += rep[q].ctr[CTR_NTIE_PR];
    }
  }
  h_report->ctr[CTR_NTIE] = nt; h_report->ctr[CTR_NTIE_PR] = ntp;
}

// b_shuffle2's container updates (cluster.cpp:242-260) replayed on the host member arrays in the
// reference's order: clusters ascending, slots descending, swap-with-last pops, appends.
// Returns the number of passes that actually ran.
int Run::replay_moves(int first_pass, int last_pass) {
  int ran = 0;
  ReplayEvent ev{0, {}, {}, 0, 0, 0};
  for (int p = first_pass; p <= last_pass; p++) {
    if (p > first_pass && h_report->pinfo[p] == h_report->pinfo[p - 1]) break;   // skipped on the device (previous pass moved nothing)
    ran++; n_shuffles++;
    const uint32_t b = h_report->pinfo[p], e = h_report->pinfo[p + 1];
    if (e == b) continue;
    if (async_replay) {
      ev.mv.insert(ev.mv.end(), h_moves + 2 * (size_t)b, h_moves + 2 * (size_t)e);
      ev.pass_end.push_back((uint32_t)(ev.mv.size() / 2));
    } else apply_moves(h_moves + 2 * (size_t)b, e - b);
  }
  if (async_replay && !ev.mv.empty()) push_event(std::move(ev));
  return ran;
}

// one shuffle pass: clusters ascending, slots descending, swap-with-last pops, appends (cluster.cpp:242-260)
void Run::apply_moves(const uint32_t *mvp, size_t n) {
  struct Mv { uint32_t from, slot, r, to; };
  std::vector<Mv> mv(n);
  for (size_t k = 0; k < n; k++) {
    const uint32_t r = mvp[2 * k], to = mvp[2 * k + 1];
    mv[k] = Mv{cluster_of_h[r], slot_of[r], r, to};
  }
  std::sort(mv.begin(), mv.end(), [](const Mv &a, const Mv &b2) { return a.from != b2.from ? a.from < b2.from : a.slot > b2.slot; });
  for (const Mv &m : mv) {
    std::vector<uint32_t> &src = members[m.from];
    const uint32_t sl = slot_of[m.r];
    const uint32_t last = src.back();                          // bi_pop_raw: slot <- last
    src[sl] = last; slot_of[last] = sl; src.pop_back();
    if (sl == 0 && !async_replay) {                            // only possible when slot 0 is not the centre (unsorted input: synchronous replay)
      const uint8_t z = 0, one = 1;
      h2d(slot0.p + m.r, &z, 1);
      if (last != m.r) h2d(slot0.p + last, &one, 1);
    }
    cl_reads_h[m.from] -= cx->reads[m.r];
    std::vector<uint32_t> &dst = members[m.to];                // bi_add_raw: append
    slot_of[m.r] = (uint32_t)dst.size(); dst.push_back(m.r);
    cl_reads_h[m.to] += cx->reads[m.r];
    cluster_of_h[m.r] = m.to;
  }
}

// bi_pop_raw(from, slot of r) + b_add_bi + bi_add_raw + bi_assign_center (cluster.cpp:315-346)
void Run::apply_bud(uint32_t r, uint32_t from) {
  std::vector<uint32_t> &src = members[from];
  const uint32_t sl = slot_of[r], last = src.back();
  src[sl] = last; slot_of[last] = sl; src.pop_back();
  cl_reads_h[from] -= cx->reads[r];
  const uint32_t ni = (uint32_t)members.size();
  members.emplace_back(1, r);
  slot_of[r] = 0; cluster_of_h[r] = ni;
  cl_reads_h.push_back(cx->reads[r]);
}

// b_init (containers.cpp:78-137): every raw in cluster 0, slot = index
void Run::init_members() {
  members.assign(1, std::vector<uint32_t>(nraw));
  slot_of.resize(nraw); cluster_of_h.assign(nraw, 0);
  for (int r = 0; r < nraw; r++) { members[0][r] = r; slot_of[r] = r; }
}

void Run::push_event(ReplayEvent &&e) {
  std::unique_lock<std::mutex> lk(rmu);
  if (!rworker.joinable()) {
    rquit = false;
    rworker = std::thread([this]() {
      std::unique_lock<std::mutex> lk2(rmu);
      for (;;) {
        rcv.wait(lk2, [&] { return rquit || !rq.empty(); });
        if (rq.empty()) { if (rquit) return; continue; }
        ReplayEvent ev = std::move(rq.front());
        rq.pop_front();
        rbusy = true;
        lk2.unlock();
        if (ev.kind == 0) {
          size_t b = 0;
          for (uint32_t e2 : ev.pass_end) { apply_moves(ev.mv.data() + 2 * b, e2 - b); b = e2; }
        } else if (ev.kind == 1) apply_bud(ev.r, ev.from);
        else init_members();
        lk2.lock();
        rbusy = false;
        if (rq.empty()) rdone.notify_all();
      }
    });
  }
  rq.push_back(std::move(e));
  rcv.notify_one();
}
void Run::drain_replay() {
  if (!rworker.joinable()) return;
  std::unique_lock<std::mutex> lk(rmu);
  rdone.wait(lk, [&] { return rq.empty() && !rbusy; });
}
void Run::stop_replay() {
  if (!rworker.joinable()) return;
  { std::unique_lock<std::mutex> lk(rmu); rquit = true; rcv.notify_all(); }
  rworker.join();
  rq.clear(); rbusy = false;
}

// b_bud (cluster.cpp:274-350) decision from the device scan.  Returns the new cluster index or 0.
int Run::decide_bud(uint32_t *r_out, uint32_t *from_out) {
  const RoundReport &R = *h_report;
  unsigned long long nt = R.ctr[CTR_NTIE], ntp = R.ctr[CTR_NTIE_PR];
  std::vector<uint32_t> big, bigp;
  const uint32_t *tr = R.tie_r, *trp = R.tiep_r;
  if (nt > TIE_MAX || ntp > TIE_MAX) {
    // pathological tie set: every rank lists its own candidates at the global optimum; sharded, the lists are exchanged padded
    // to the longest one
    const int W = cx->world;
    struct RepView { const std::vector<const RoundReport *> &v; const RoundReport &operator[](int q) const { return *v[q]; } } rep{rep_all};
    std::vector<unsigned long long> na(W, 0), np(W, 0);
    unsigned long long maxn = 1;
    for (int q = 0; q < W; q++) {
      if (rep[q].ctr[CTR_NTIE] && rep[q].ctr[CTR_PMIN] == R.ctr[CTR_PMIN] && rep[q].ctr[CTR_RMAX] == R.ctr[CTR_RMAX]) na[q] = rep[q].ctr[CTR_NTIE];
      if (rep[q].ctr[CTR_NTIE_PR] && rep[q].ctr[CTR_PMIN_PR] == R.ctr[CTR_PMIN_PR] && rep[q].ctr[CTR_RMAX_PR] == R.ctr[CTR_RMAX_PR]) np[q] = rep[q].ctr[CTR_NTIE_PR];
      maxn = std::max(maxn, std::max(na[q], np[q]));
    }
    DBuf<uint32_t> &d1 = tie_d1, &d2 = tie_d2, &g1 = tie_g1, &g2 = tie_g2;       // members: no cudaMalloc / cudaFree in a steady-state pass
    d1.alloc(maxn); d2.alloc(maxn);
    unsigned long long gl[6] = {R.ctr[CTR_PMIN], R.ctr[CTR_RMAX], 0ull, R.ctr[CTR_PMIN_PR], R.ctr[CTR_RMAX_PR], 0ull};
    static_assert(CTR_RMAX == CTR_PMIN + 1 && CTR_NTIE == CTR_PMIN + 2 && CTR_PMIN_PR == CTR_PMIN + 3 && CTR_NTIE_PR == CTR_PMIN + 5, "counter layout");
    h2d(ctr.p + CTR_PMIN, gl, sizeof(gl));
    BudParams bp{o->min_fold, o->min_hamming, o->min_abund};
    launch_bud_collect_owned(st, in, ts, bp, d1.p, d2.p, (unsigned)maxn, s);
    const uint32_t *all1 = d1.p, *all2 = d2.p;
    if (W > 1) {
      g1.alloc(maxn * W); g2.alloc(maxn * W);
      NC(g_nccl.AllGather(d1.p, g1.p, (size_t)maxn * 4, ncclChar, cx->comm, s));
      NC(g_nccl.AllGather(d2.p, g2.p, (size_t)maxn * 4, ncclChar, cx->comm, s));
      all1 = g1.p; all2 = g2.p;
    }
    std::vector<uint32_t> h1(maxn * W), h2(maxn * W);
    d2h(h1.data(), all1, h1.size() * 4); d2h(h2.data(), all2, h2.size() * 4);
    sync();
    for (int q = 0; q < W; q++) {
      big.insert(big.end(), h1.begin() + (size_t)q * maxn, h1.begin() + (size_t)q * maxn + na[q]);
      bigp.insert(bigp.end(), h2.begin() + (size_t)q * maxn, h2.begin() + (size_t)q * maxn + np[q]);
    }
    if (big.size() != nt || bigp.size() != ntp) throw Err{"dada2b: inconsistent tie lists across ranks"};
    tr = big.data(); trp = bigp.data();
  }
  // The device reported the cluster and the cluster's reads of every listed candidate: a single candidate needs nothing
  // from the host's member arrays, so the replay worker may still be busy with this round's moves.  Exact ties do: wait for it.
  const bool from_report = async_replay && nt <= 1 && ntp <= 1;
  if (!from_report) drain_replay();
  auto pick = [&](const uint32_t *t, unsigned long long n) -> long {     // first in (cluster, slot) scan order
    if (n == 1) return (long)t[0];
    long best = -1;
    for (unsigned long long k = 0; k < n; k++) {
      const uint32_t r = t[k];
      if (best < 0 || cluster_of_h[r] < cluster_of_h[best] || (cluster_of_h[r] == cluster_of_h[best] && slot_of[r] < slot_of[best])) best = r;
    }
    return best;
  };
  const uint32_t c0 = cl_center_h[0];     // minraw starts as the centre of cluster 0 (p == 1), cluster.cpp:279
  auto bits2d = [](unsigned long long b) { double d; memcpy(&d, &b, 8); return d; };
  long win = -1, win_pr = -1;
  double pmin = 1.0, pmin_pr = 1.0;
  if (nt) {
    const double pv = bits2d(R.ctr[CTR_PMIN]);
    if (pv < 1.0 || (pv == 1.0 && R.ctr[CTR_RMAX] > cx->reads[c0])) { win = pick(tr, nt); pmin = pv; }
  }
  if (ntp) {
    const double pv = bits2d(R.ctr[CTR_PMIN_PR]);
    if (pv < 1.0 || (pv == 1.0 && R.ctr[CTR_RMAX_PR] > cx->reads[c0])) { win_pr = pick(trp, ntp); pmin_pr = pv; }
  }
  const double pA = pmin * (double)(unsigned)nraw, pP = pmin_pr;
  long w = -1; char type = 0; double pv = 0;
  if (pA < o->omegaA && win >= 0) { w = win; type = 'A'; pv = pA; }
  else if (pP < o->omegaP && win_pr >= 0) { w = win_pr; type = 'P'; pv = pP; }
  if (w < 0) return 0;
  const uint32_t r = (uint32_t)w;
  uint32_t from, from_reads;
  if (from_report) {
    const bool isA = type == 'A';
    from = isA ? R.tie_cl[0] : R.tiep_cl[0]; from_reads = isA ? R.tie_clreads[0] : R.tiep_clreads[0];
  } else { from = cluster_of_h[r]; from_reads = cl_reads_h[from]; }
  // the winner's comparison (raw->comp)
  double lam = 0; uint32_t ham = 0; bool have = false;
  for (unsigned long long k = 0; k < std::min<unsigned long long>(nt, TIE_MAX) && !have; k++)
    if (R.tie_r[k] == r && type == 'A') { lam = R.tie_lam[k]; ham = R.tie_ham[k]; have = true; }
  for (unsigned long long k = 0; k < std::min<unsigned long long>(ntp, TIE_MAX) && !have; k++)
    if (R.tiep_r[k] == r && type == 'P') { lam = R.tiep_lam[k]; ham = R.tiep_ham[k]; have = true; }
  if (!have) {            // only the winner's owner holds its comparison: sum all-reduce of (lambda bits, hamming) with zeros elsewhere
    DBuf<unsigned long long> &w2 = win_buf; w2.alloc(2); w2.zero(s);
    if ((int)(r % (uint32_t)cx->world) == cx->rank) {
      CK(cudaMemcpyAsync(w2.p, comp_lambda.p + r, 8, cudaMemcpyDeviceToDevice, s));
      CK(cudaMemcpyAsync(w2.p + 1, comp_ham.p + r, 4, cudaMemcpyDeviceToDevice, s));
    }
    if (cx->world > 1) NC(g_nccl.AllReduce(w2.p, w2.p, 2, ncclUint64, ncclSum, cx->comm, s));
    unsigned long long hw[2];
    d2h(hw, w2.p, 16);
    sync();
    memcpy(&lam, &hw[0], 8); ham = (uint32_t)hw[1];
  }
  const double expected = lam * (double)from_reads;
  const uint32_t ni = (uint32_t)nclust_h;                       // b_add_bi + bi_add_raw + bi_assign_center
  if (async_replay) { ReplayEvent ev{1, {}, {}, r, from, ni}; push_event(std::move(ev)); }
  else apply_bud(r, from);
  nclust_h++;
  cl_center_h.push_back(r);
  Birth b; b.type = type; b.from = from;                        // 'P': uninitialised in the reference (cluster.cpp:334-339)
  b.pval = pv; b.fold = (double)cx->reads[r] / expected; b.e = expected;
  b.comp_i = from; b.comp_index = r; b.comp_lambda = lam; b.comp_ham = ham;
  birth.push_back(b);
  pending.apply = 1; pending.r = r; pending.from = from; pending.newi = ni; pending.reads = cx->reads[r];
  *r_out = r; *from_out = from;
  return (int)ni;
}

template <typename T> T *dupv(const std::vector<T> &v) {
  T *p = (T *)malloc(std::max<size_t>(1, v.size()) * sizeof(T));
  if (!v.empty()) memcpy(p, v.data(), v.size() * sizeof(T));
  return p;
}

// Rmain.cpp:168-295: final subs, final p, output tables
void Run::finish(dada2b_out *out) {
  // DADA2B_VERBOSE: host clock per phase; the device work of a phase is waited for before its end is read
  const bool vb = getenv("DADA2B_VERBOSE") != nullptr;
  double ph[10]; int nph = 0;
  ph[nph++] = now_ms();
  // A helper sums the loop's kernel timings while the device runs the final pass (every event recorded so far has completed:
  // the loop ended with a synchronisation); ~2.5 ms of event queries at 1e6 uniques.  The guard joins it on every way out.
  const std::vector<Ev> loop_evs(evs);
  double ksum[T_N] = {}; int kcnt[T_N] = {};
  std::thread ev_helper([&]() {
    if (cudaSetDevice(cx->device) != cudaSuccess) return;
    for (const Ev &e : loop_evs) { float t = 0; if (cudaEventElapsedTime(&t, e.a, e.b) == cudaSuccess) { ksum[e.tag] += t; kcnt[e.tag]++; } }
  });
  struct Join { std::thread &t; ~Join() { if (t.joinable()) t.join(); } } join{ev_helper};
  drain_replay();
  ph[nph++] = now_ms();
  const uint32_t nclust = (uint32_t)members.size();
  const int maxlen = in.maxlen;
  if (pending.apply) { launch_round_begin(st, 1, pending.r, pending.from, pending.newi, pending.reads, s); pending.apply = 0; }
  launch_final_p(st, in, o->omegaC, s);
  trans.alloc((size_t)16 * ncol); trans.zero(s);
  cq_sum.alloc((size_t)nclust * maxlen); cq_cnt.alloc((size_t)nclust * maxlen); cq_sum.zero(s); cq_cnt.zero(s);
  st.trans = trans.p; st.cq_sum = cq_sum.p; st.cq_cnt = cq_cnt.p;
  const int n_owned = (nraw - cx->rank + cx->world - 1) / cx->world;     // raws aligned by this rank in the final pass
  bool split = false;                    // the raws are split into a diagonal and a gapped list
  {  // FinalSubsParallel: sub_new(centre, raw, use_kmers=false) for every raw
    if (P.band > 0) {
      // 1) forward-carry NW of every raw against its own centre: nsubs + "is the optimal path the pure diagonal?"
      FwdArgs f{};
      unsigned long long nn = (unsigned long long)n_owned;
      h2d(ctr.p + CTR_FB, &nn, 8);                       // job count lives in CTR_FB for this launch
      { unsigned long long z[2] = {0ull, 0ull}; h2d(ctr.p + CTR_NW, z, 16); }
      f.in = in; f.P = P; f.st = st; f.jobs = nullptr; f.njobs_ptr = st.ctr + CTR_FB;
      f.seq_bytes = seq_bytes; f.mode = 1; f.job_mul = cx->world; f.job_add = cx->rank;
      f.gl_out = st.gl_list; f.nw_out = st.nw_list; f.gl_count = st.ctr + CTR_GL; f.nw_count = st.ctr + CTR_NW;
      f.fb_list = fb_list.p; f.fb_count = st.ctr + CTR_NMOVE;   // (scratch counter; pairs that do not fit -> traceback list below)
      { unsigned long long z = 0; h2d(ctr.p + CTR_NMOVE, &z, 8); }
      const long worst = (long)in.maxlen * std::max(std::abs(P.mismatch), std::abs(P.match)) + std::max(std::abs(P.gap), std::abs(P.hgap)) + 16;
      f.fast_ok = (worst < std::abs((long)P.sentinel) / 2) ? 1 : 0;
      bool row_done = false;
      if (row_mv.p) {       // thread-per-pair row kernel when every sequence has the same length (dd_nwrow.cu), else the lane-group kernel
        CK(cudaMemsetAsync(uneq_ctr.p, 0, 8, s));
        timed(T_FROW, [&]() { row_done = launch_nwrow_final(f, uneq_list.p, uneq_ctr.p, (unsigned long long)nraw, cx->num_sms, s); });
      }
      if (row_done) split = true;
      else timed(T_FROW, [&]() { split = launch_nwfwd(f, fwd_slots, (unsigned long long)nraw, (unsigned long long)nraw, cx->num_sms, s); });
    }
    if (split) {
      // 2) per-cluster reduction over the pure-diagonal raws (dd_final.cu), 3) traceback kernel for the rest (+ pairs that did not fit)
      ft_off.alloc((size_t)nclust + 1); ft_chk.alloc((size_t)nclust + 1); ft_cur.alloc(nclust); ft_ord.alloc(std::max(n_owned, 1));
      ft_sums.alloc(final_tally_scan_words((int)nclust));
      ft_off.zero(s);
      timed(T_FDIAG, [&]() {
        launch_final_tally(in, st, st.gl_list, st.ctr + CTR_GL, (unsigned long long)n_owned, (int)nclust, ncol, ft_off.p, ft_chk.p, ft_cur.p, ft_ord.p,
                           ft_sums.p, cx->num_sms, s);
      });
      for (int pass = 1; pass < 3; pass++) {
        AlignArgs a = align_args(MODE_FINAL, KIND_NW);
        a.jobs = pass == 1 ? st.nw_list : fb_list.p;
        a.njobs_ptr = st.ctr + (pass == 1 ? CTR_NW : CTR_NMOVE);
        timed(T_FGAP, [&]() { launch_align_jobs(MODE_FINAL, a, (unsigned long long)nraw); });
      }
    } else {
      AlignArgs a = align_args(MODE_FINAL, P.band == 0 ? KIND_GAPLESS : KIND_NW);
      a.jobs = nullptr; a.njobs_ptr = nullptr; a.njobs_fixed = n_owned; a.job_mul = cx->world; a.job_add = cx->rank;
      timed(T_FGAP, [&]() { launch_align_jobs(MODE_FINAL, a, (unsigned long long)nraw); });
    }
  }
  fin_tl.alloc((size_t)5 * nclust); fin_tl.zero(s); fin_map.alloc(nraw);
  launch_cluster_tally(in, st, (int)nclust, cx->rank, cx->world, fin_tl.p, fin_map.p, cx->num_sms, s);
  if (vb) {
    read_ctr();                            // synchronises
    if (split) fprintf(stderr, "[dada2b] final pass lists: diagonal %llu, gapped %llu, handed back %llu\n", h_ctr.p[CTR_GL], h_ctr.p[CTR_NW], h_ctr.p[CTR_NMOVE]);
  }
  ph[nph++] = now_ms();
  if (cx->world > 1) {   // every rank tallied its own raws: integer sums are exact and order-independent
    NC(g_nccl.AllReduce(trans.p, trans.p, (size_t)16 * ncol, ncclInt32, ncclSum, cx->comm, s));
    NC(g_nccl.AllReduce(cq_sum.p, cq_sum.p, (size_t)nclust * maxlen, ncclUint64, ncclSum, cx->comm, s));
    NC(g_nccl.AllReduce(cq_cnt.p, cq_cnt.p, (size_t)nclust * maxlen, ncclUint64, ncclSum, cx->comm, s));
    NC(g_nccl.AllReduce(fin_tl.p, fin_tl.p, (size_t)4 * nclust, ncclUint32, ncclSum, cx->comm, s));
    // abundances arrive as non-negative int32: their int32 maximum is the unsigned one
    NC(g_nccl.AllReduce(fin_tl.p + (size_t)4 * nclust, fin_tl.p + (size_t)4 * nclust, nclust, ncclInt32, ncclMax, cx->comm, s));
    NC(g_nccl.AllReduce(fin_map.p, fin_map.p, (size_t)nraw, ncclInt32, ncclSum, cx->comm, s));     // 0 off the owner
    // final p is only meaningful on a raw's owner: zero the rest, then the sum is the full array
    launch_mask_unowned(this->p.p, correct.p, nraw, cx->rank, cx->world, s);
    NC(g_nccl.AllReduce(this->p.p, this->p.p, (size_t)nraw, ncclFloat64, ncclSum, cx->comm, s));
  }
  // birth subs: sub_new(centre of birth_comp.i, centre i, use_kmers, cutoff 1.0)   Rmain.cpp:206-209
  const uint32_t npair = nclust - 1;
  std::vector<uint32_t> bns(npair, 0);
  std::vector<uint16_t> bpos; std::vector<uint8_t> bnt0, bnt1, bq1;
  const int bcap = maxlen;
  if (npair) {
    std::vector<uint32_t> pc(npair), pr(npair);
    for (uint32_t i = 1; i < nclust; i++) { pc[i - 1] = cl_center_h[birth[i].comp_i]; pr[i - 1] = cl_center_h[i]; }
    pair_centre.alloc(npair); pair_raw.alloc(npair);
    h2d(pair_centre.p, pc.data(), npair * 4);
    h2d(pair_raw.p, pr.data(), npair * 4);
    if (cx->qual_sharded) {        // the birth subs read the quality row of every centre: owners contribute theirs, one byte-sum all-reduce
      DBuf<uint8_t> &cq = fin_cq; cq.alloc((size_t)npair * in.QS);
      launch_qrows_gather(in.qual, in.QS, pair_raw.p, (int)npair, cx->rank, cx->world, cq.p, s);
      NC(g_nccl.AllReduce(cq.p, cq.p, (size_t)npair * in.QS, ncclUint8, ncclSum, cx->comm, s));
      launch_qrows_scatter(in.qual, in.QS, pair_raw.p, (int)npair, 0, 1, cq.p, s);
      sync();
    }
    b_nsubs.alloc(npair); b_lambda.alloc(npair); b_pos.alloc((size_t)npair * bcap); b_nt0.alloc((size_t)npair * bcap);
    b_nt1.alloc((size_t)npair * bcap); b_q1.alloc((size_t)npair * bcap);
    DBuf<uint32_t> &nwl = fin_nwl, &gll = fin_gll; nwl.alloc(npair); gll.alloc(npair);
    CK(cudaMemsetAsync(ctr.p + CTR_NW, 0, 2 * 8, s));
    ClassifyArgs ca{};
    ca.in = in; ca.P = P; ca.P.kdist_cutoff = 1.0; ca.mode = 1; ca.pair_centre = pair_centre.p; ca.pair_raw = pair_raw.p;
    ca.nw_list = nwl.p; ca.gl_list = gll.p; ca.ctr = st.ctr; ca.kord_words = kord_words; ca.greedy = 0; ca.lock = st.lock;
    ca.shard_rank = 0; ca.shard_world = 1;
    // birth alignments are not counted in nalign/nshroud by the reference: the counters are kept on the device and restored afterwards
    static_assert(CTR_SHROUD == CTR_ALIGN + 1, "counter layout");
    DBuf<unsigned long long> &keep = fin_keep; keep.alloc(2);
    CK(cudaMemcpyAsync(keep.p, ctr.p + CTR_ALIGN, 2 * 8, cudaMemcpyDeviceToDevice, s));
    launch_classify(ca, (int)npair, 256, classify_smem, s);
    for (int kind : {KIND_NW, KIND_GAPLESS}) {
      AlignArgs a = align_args(MODE_BIRTH, kind);
      a.jobs = kind == KIND_NW ? nwl.p : gll.p;
      a.njobs_ptr = st.ctr + (kind == KIND_NW ? CTR_NW : CTR_GL);
      a.pair_centre = pair_centre.p; a.pair_raw = pair_raw.p;
      a.b_nsubs = b_nsubs.p; a.b_lambda = b_lambda.p; a.b_pos = b_pos.p; a.b_nt0 = b_nt0.p; a.b_nt1 = b_nt1.p; a.b_q1 = b_q1.p;
      a.b_cap = bcap; a.b_ops = nullptr; a.b_nops = nullptr; a.b_opcap = 0;
      launch_align_jobs(MODE_BIRTH, a, npair);
    }
    CK(cudaMemcpyAsync(ctr.p + CTR_ALIGN, keep.p, 2 * 8, cudaMemcpyDeviceToDevice, s));
    bpos.resize((size_t)npair * bcap); bnt0.resize((size_t)npair * bcap); bnt1.resize((size_t)npair * bcap); bq1.resize((size_t)npair * bcap);
    d2h(bns.data(), b_nsubs.p, npair * 4);
    d2h(bpos.data(), b_pos.p, bpos.size() * 2);
    d2h(bnt0.data(), b_nt0.p, bnt0.size());
    d2h(bnt1.data(), b_nt1.p, bnt1.size());
    d2h(bq1.data(), b_q1.p, bq1.size());           // completed by the post-hoc pass's first synchronisation
  }
  ph[nph++] = now_ms();
  // post-hoc cluster p-values (error.cpp:99-119)
  std::vector<double> tot_e(nclust, 0.0), cpval(nclust, 0.0);
  {
    center_cluster.alloc(nraw);
    CK(cudaMemsetAsync(center_cluster.p, 0xFF, (size_t)nraw * 4, s));     // -1 everywhere
    launch_center_cluster(center_cluster.p, st.cl_center, (int)nclust, s);
    unsigned cap = std::max<unsigned>(4096, nclust * 8);
    std::vector<uint32_t> tij; std::vector<double> tv; unsigned long long cnt = 0;
    DBuf<unsigned long long> &dcount = fin_dcount; dcount.alloc(1);
    for (;;) {
      trip_ij.alloc((size_t)cap * 2); trip_v.alloc(cap); dcount.zero(s);
      launch_posthoc_owned(st, nraw, cs_count, center_cluster.p, trip_ij.p, trip_v.p, cap, dcount.p, cx->rank, cx->world, s);
      d2h(&cnt, dcount.p, 8);
      sync();
      if (cnt <= cap) break;
      cap = (unsigned)cnt + 16;
    }
    if (cx->world > 1) {       // every rank found the triples of the centres it owns: exchange them (counts first, then padded payloads)
      const int W = cx->world;
      DBuf<unsigned long long> &dall = fin_dall; dall.alloc(W);
      NC(g_nccl.AllGather(dcount.p, dall.p, 1, ncclUint64, cx->comm, s));
      std::vector<unsigned long long> cq(W);
      d2h(cq.data(), dall.p, (size_t)W * 8);
      sync();
      unsigned long long maxc = 1, tot = 0;
      for (int q = 0; q < W; q++) { maxc = std::max(maxc, cq[q]); tot += cq[q]; }
      DBuf<uint32_t> &sij = fin_sij, &gij = fin_gij; DBuf<double> &sv = fin_sv, &gv = fin_gv;
      sij.alloc((size_t)maxc * 2); sv.alloc((size_t)maxc); sij.zero(s); sv.zero(s);
      if (cnt) {
        CK(cudaMemcpyAsync(sij.p, trip_ij.p, cnt * 8, cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(sv.p, trip_v.p, cnt * 8, cudaMemcpyDeviceToDevice, s));
      }
      gij.alloc((size_t)maxc * 2 * W); gv.alloc((size_t)maxc * W);
      NC(g_nccl.AllGather(sij.p, gij.p, (size_t)maxc * 8, ncclChar, cx->comm, s));
      NC(g_nccl.AllGather(sv.p, gv.p, (size_t)maxc * 8, ncclChar, cx->comm, s));
      std::vector<uint32_t> hij((size_t)maxc * 2 * W); std::vector<double> hv((size_t)maxc * W);
      d2h(hij.data(), gij.p, hij.size() * 4); d2h(hv.data(), gv.p, hv.size() * 8);
      sync();
      tij.clear(); tv.clear();
      for (int q = 0; q < W; q++) {
        tij.insert(tij.end(), hij.begin() + (size_t)q * maxc * 2, hij.begin() + (size_t)q * maxc * 2 + cq[q] * 2);
        tv.insert(tv.end(), hv.begin() + (size_t)q * maxc, hv.begin() + (size_t)q * maxc + cq[q]);
      }
      cnt = tot;
    } else {
    tij.resize(cnt * 2); tv.resize(cnt);
    if (cnt) {
      d2h(tij.data(), trip_ij.p, cnt * 8);
      d2h(tv.data(), trip_v.p, cnt * 8);
      sync();
    }
    }
    std::vector<size_t> ord(cnt);
    for (size_t k = 0; k < cnt; k++) ord[k] = k;
    std::sort(ord.begin(), ord.end(), [&](size_t x, size_t y) { return tij[2 * x] < tij[2 * y]; });   // ascending source cluster i
    for (size_t k : ord) tot_e[tij[2 * k + 1]] += tv[k];
    std::vector<int> rr(nclust), pp(nclust, 1);
    for (uint32_t i = 0; i < nclust; i++) rr[i] = (int)cx->reads[cl_center_h[i]];
    pa_reads.alloc(nclust); pa_prior.alloc(nclust); pa_E.alloc(nclust); pa_out.alloc(nclust);
    h2d(pa_reads.p, rr.data(), nclust * 4);
    h2d(pa_prior.p, pp.data(), nclust * 4);
    h2d(pa_E.p, tot_e.data(), nclust * 8);
    launch_calc_pA_vec(pa_reads.p, pa_E.p, pa_prior.p, pa_out.p, (int)nclust, s);
    d2h(cpval.data(), pa_out.p, nclust * 8);
  }
  if (vb) sync();
  ph[nph++] = now_ms();
  // cluster-sized results, $map and $pval: staged in the pinned arena, one synchronisation for all of them
  std::vector<int> htrans((size_t)16 * ncol); std::vector<unsigned long long> hsum((size_t)nclust * maxlen), hcnt((size_t)nclust * maxlen);
  std::vector<uint32_t> tl((size_t)5 * nclust);
  {
    const size_t need = htrans.size() * 4 + (hsum.size() + hcnt.size()) * 8 + tl.size() * 4 + (size_t)nraw * 12 + 6 * 64;
    if (arena_off + need > arena.cap) { sync(); if (need > arena.cap) arena.alloc(need); }   // nothing staged below waits for room
  }
  d2h(htrans.data(), trans.p, htrans.size() * 4);
  d2h(hsum.data(), cq_sum.p, hsum.size() * 8);
  d2h(hcnt.data(), cq_cnt.p, hcnt.size() * 8);
  d2h(tl.data(), fin_tl.p, tl.size() * 4);
  auto stage = [&](const void *d, size_t n) { d2h_bytes += (long long)n; uint8_t *q = arena_get(n); CK(cudaMemcpyAsync(q, d, n, cudaMemcpyDeviceToHost, s)); return q; };
  const double *hp = (const double *)stage(p.p, (size_t)nraw * 8);
  const int32_t *hmap = (const int32_t *)stage(fin_map.p, (size_t)nraw * 4);
  read_ctr();                                     // synchronises; nothing below touches the arena
  check_dev_error();
  ph[nph++] = now_ms();

  out->nclust = nclust; out->nraw = nraw; out->maxlen = maxlen; out->Q = ncol;
  out->n_align = (int64_t)h_ctr.p[CTR_ALIGN]; out->n_shroud = (int64_t)h_ctr.p[CTR_SHROUD];
  out->n_nw = (int64_t)tot_nw; out->n_gapless = (int64_t)tot_gl; out->nw_cells = (int64_t)h_ctr.p[CTR_CELLS];
  out->n_rounds = n_rounds; out->n_shuffles = n_shuffles;
  // ---- $clustering (error.cpp:9-127)
  std::string cseq; std::vector<int64_t> coff(1, 0);
  std::vector<int32_t> ab(nclust), n0(nclust), n1(nclust), nunq(nclust), bfrom(nclust), bham(nclust);
  std::vector<double> bpval(nclust), bfold(nclust), bqave(nclust);
  for (uint32_t i = 0; i < nclust; i++) {
    ab[i] = (int32_t)tl[i]; n0[i] = (int32_t)tl[nclust + i]; n1[i] = (int32_t)tl[2 * (size_t)nclust + i]; nunq[i] = (int32_t)tl[3 * (size_t)nclust + i];
  }
  const uint32_t *mxr = tl.data() + 4 * (size_t)nclust;    // largest abundance among a cluster's members (correct or not)
  // The representative sequences are read back from the packed rows on the device (a run that gets here saw nothing but ACGT,
  // nt2int would have stopped it): no host copy of the input strings is kept.  Pinned buffer of its own -- the arena is in use.
  std::vector<long> max_raw(nclust, -1);           // error.cpp:20-27: the first member (Bi::raw order) holding the largest abundance
  uint32_t nrep = 0;
  for (uint32_t i = 0; i < nclust; i++)
    if (mxr[i] > 0) for (uint32_t r : members[i]) if (cx->reads[r] == mxr[i]) { max_raw[i] = r; nrep++; break; }
  const size_t rowb = (size_t)in.SW * 4;
  if (nrep) {
    fin_rep_h.alloc((size_t)nrep * (4 + rowb) + 64);
    uint32_t *rows_h = (uint32_t *)fin_rep_h.p;
    uint32_t k = 0;
    for (uint32_t i = 0; i < nclust; i++) if (max_raw[i] >= 0) rows_h[k++] = (uint32_t)max_raw[i];
    fin_rep_rows.alloc(nrep); fin_rep_d.alloc((size_t)nrep * rowb);
    h2d_bytes += (long long)nrep * 4; d2h_bytes += (long long)(nrep * rowb);
    CK(cudaMemcpyAsync(fin_rep_rows.p, rows_h, (size_t)nrep * 4, cudaMemcpyHostToDevice, s));
    launch_qrows_gather((const uint8_t *)in.seq2, (int)rowb, fin_rep_rows.p, (int)nrep, -1, 1, fin_rep_d.p, s);
    CK(cudaMemcpyAsync(fin_rep_h.p + (((size_t)nrep * 4 + 63) & ~(size_t)63), fin_rep_d.p, (size_t)nrep * rowb, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  ph[nph++] = now_ms();
  const uint32_t *rep_words = (const uint32_t *)(fin_rep_h.p + (((size_t)nrep * 4 + 63) & ~(size_t)63));
  uint32_t rep_k = 0;
  for (uint32_t i = 0; i < nclust; i++) {
    if (max_raw[i] >= 0) {
      const uint32_t *w = rep_words + (size_t)rep_k++ * in.SW;
      const int L = cx->len[max_raw[i]];
      for (int b = 0; b < L; b++) cseq.push_back("ACGT"[(w[b >> 4] >> (2 * (b & 15))) & 3]);
    }
    coff.push_back((int64_t)cseq.size());
    if (i == 0) { bpval[i] = na_real(); bfrom[i] = INT_MIN; bfold[i] = na_real(); bham[i] = INT_MIN; bqave[i] = na_real(); }
    else {
      bfrom[i] = (int32_t)birth[i].from + 1; bpval[i] = birth[i].pval; bfold[i] = birth[i].fold; bham[i] = (int32_t)birth[i].comp_ham;
      double q_ave = 0.0; const uint32_t ns = bns[i - 1];
      for (uint32_t k = 0; k < ns && k < (uint32_t)bcap; k++) q_ave += bq1[(size_t)(i - 1) * bcap + k];
      q_ave = q_ave / ((double)ns);
      bqave[i] = q_ave;
    }
  }
  out->cl_seq_concat = (char *)malloc(cseq.size() + 1); memcpy(out->cl_seq_concat, cseq.data(), cseq.size()); out->cl_seq_concat[cseq.size()] = 0;
  out->cl_seq_off = dupv(coff);
  out->cl_abundance = dupv(ab); out->cl_n0 = dupv(n0); out->cl_n1 = dupv(n1); out->cl_nunq = dupv(nunq);
  out->cl_pval = dupv(cpval); out->cl_birth_from = dupv(bfrom); out->cl_birth_pval = dupv(bpval); out->cl_birth_fold = dupv(bfold);
  out->cl_birth_ham = dupv(bham); out->cl_birth_qave = dupv(bqave);
  // ---- $birth_subs (error.cpp:261-300)
  std::vector<int32_t> bs_pos, bs_clust; std::vector<char> bs_ref, bs_sub; std::vector<double> bs_qual;
  for (uint32_t i = 1; i < nclust; i++)
    for (uint32_t k = 0; k < bns[i - 1] && k < (uint32_t)bcap; k++) {
      const size_t o2 = (size_t)(i - 1) * bcap + k;
      bs_pos.push_back(bpos[o2] + 1); bs_ref.push_back("ACGT"[bnt0[o2]]); bs_sub.push_back("ACGT"[bnt1[o2]]);
      bs_qual.push_back((double)bq1[o2]); bs_clust.push_back((int32_t)i + 1);
    }
  out->n_birth_subs = (int32_t)bs_pos.size();
  out->bs_pos = dupv(bs_pos); out->bs_clust = dupv(bs_clust); out->bs_ref = dupv(bs_ref); out->bs_sub = dupv(bs_sub); out->bs_qual = dupv(bs_qual);
  // ---- $subqual: device row-major [16][ncol] -> column-major 16 x ncol (error.cpp:131-172)
  std::vector<int32_t> sq((size_t)16 * ncol);
  for (int t = 0; t < 16; t++) for (int q = 0; q < ncol; q++) sq[t + 16 * (size_t)q] = htrans[(size_t)t * ncol + q];
  out->subqual = dupv(sq); out->subqual_ncol = ncol;
  // ---- $clusterquals (error.cpp:225-258)
  std::vector<double> cq((size_t)maxlen * nclust);
  for (uint32_t i = 0; i < nclust; i++) {
    const int seqlen = cx->len[cl_center_h[i]];
    for (int pos = 0; pos < maxlen; pos++) {
      const size_t k = (size_t)i * maxlen + pos;
      cq[pos + (size_t)maxlen * i] = pos < seqlen ? (double)hsum[k] / (double)(unsigned)hcnt[k] : na_real();
    }
  }
  out->clusterquals = dupv(cq);
  ph[nph++] = now_ms();
  // ---- $map, $pval (Rmain.cpp:239-279)
  out->map = (int32_t *)malloc(std::max<size_t>(1, nraw) * sizeof(int32_t));
  out->pval = (double *)malloc(std::max<size_t>(1, nraw) * sizeof(double));
  parallel_for((size_t)nraw, [&](size_t lo, size_t hi) {
    memcpy(out->map + lo, hmap + lo, (hi - lo) * sizeof(int32_t));
    memcpy(out->pval + lo, hp + lo, (hi - lo) * sizeof(double));
  });
  ph[nph++] = now_ms();
  // ---- timing / traffic diagnostics
  CK(cudaEventRecord(ev_end, s));
  CK(cudaEventSynchronize(ev_end));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, ev_begin, ev_end));
  out->ms_device = ms;
  ev_helper.join();
  double sum[T_N] = {}; int cnt[T_N] = {};
  for (int t = 0; t < T_N; t++) { sum[t] = ksum[t]; cnt[t] = kcnt[t]; }
  for (size_t k = loop_evs.size(); k < evs.size(); k++) {        // the final pass's
    const Ev &e = evs[k]; float t = 0;
    if (cudaEventElapsedTime(&t, e.a, e.b) == cudaSuccess) { sum[e.tag] += t; cnt[e.tag]++; }
  }
  if (getenv("DADA2B_VERBOSE")) fprintf(stderr, "[dada2b] loop NW: bound pass %.3f ms (%d launches), exact %.3f ms (%d launches)\n", sum[T_NWB], cnt[T_NWB], sum[T_NW], cnt[T_NW]);
  out->ms_k_prescreen = sum[T_PRE]; out->n_k_prescreen = cnt[T_PRE]; out->prescreen_rows = prescreen_rows;
  out->ms_k_nw_bound = sum[T_NWB]; out->n_k_nw_bound = cnt[T_NWB]; out->ms_k_nw_exact = sum[T_NW]; out->n_k_nw_exact = cnt[T_NW];
  out->ms_k_tail = sum[T_TAIL]; out->n_k_tail = cnt[T_TAIL];
  out->ms_k_final_row = sum[T_FROW]; out->ms_k_final_diag = sum[T_FDIAG]; out->ms_k_final_gapped = sum[T_FGAP];
  out->n_k_final_row = cnt[T_FROW]; out->n_k_final_diag = cnt[T_FDIAG]; out->n_k_final_gapped = cnt[T_FGAP];
  sum[T_NW] += sum[T_NWB]; cnt[T_NW] += cnt[T_NWB];
  sum[T_CLASSIFY] += sum[T_PRE]; cnt[T_CLASSIFY] += cnt[T_PRE];
  out->ms_k_classify = sum[T_CLASSIFY]; out->ms_k_align_nw = sum[T_NW]; out->ms_k_align_gl = sum[T_GL]; out->ms_k_align_final = sum[T_FROW] + sum[T_FDIAG] + sum[T_FGAP];
  out->n_k_classify = cnt[T_CLASSIFY]; out->n_k_align_nw = cnt[T_NW]; out->n_k_align_gl = cnt[T_GL]; out->n_k_align_final = cnt[T_FROW] + cnt[T_FDIAG] + cnt[T_FGAP];
  out->n_final_nw = (P.band == 0) ? 0 : nraw;
  out->gpu_launches = launches_count() - launches0;
  out->h2d_bytes = h2d_bytes; out->d2h_bytes = d2h_bytes;
  ph[nph++] = now_ms();
  if (vb) fprintf(stderr, "[dada2b] finish host ms: drain replay %.2f, final pass %.2f, birth subs %.2f, post-hoc %.2f, D2H %.2f, "
                  "representatives %.2f, cluster outputs %.2f, map/pval %.2f, kernel timings %.2f\n",
                  ph[1] - ph[0], ph[2] - ph[1], ph[3] - ph[2], ph[4] - ph[3], ph[5] - ph[4], ph[6] - ph[5], ph[7] - ph[6], ph[8] - ph[7], ph[9] - ph[8]);
}

dada2b_out *do_run(dada2b_ctx *cx, const double *err_cm, int Q, const dada2b_opts *o) {
  const double t0 = now_ms();
  g_t0 = t0;
  g_watch.last_end = 0;
  CK(cudaSetDevice(cx->device));
  if (Q < 1) throw Err{"Error matrix must have 16 rows."};
  if (cx->bad_nt) throw Err{o->use_kmers ? "Unexpected nucleotide." : "Non-ACGT sequences in compute_lambda."};
  if (o->use_quals && cx->maxq > Q - 1) throw Err{"Rounded quality exceeded range of err lookup table."};
  if (!cx->run) cx->run = new Run();
  Run &R = *cx->run;
  R.reset_host();
  R.bind(cx, o, Q);
  DBG("run: begin");
  cx->ev_next = 0;
  R.launches0 = launches_count();
  R.ev_begin = cx->get_event(); R.ev_end = cx->get_event();
  TDBG("begin");
  R.setup_params();
  TDBG("params set");
  R.alloc_state();
  TDBG("state allocated");
  if (getenv("DADA2B_SYNCDEBUG")) fprintf(stderr, "[dada2b] state allocated; warp_words=%d ptr_in_smem=%d align_smem=%zu grid=%d\n", R.warp_words, R.ptr_in_smem, R.align_smem, R.align_grid);
  CK(cudaEventRecord(R.ev_begin, R.s));
  {  // cluster.cpp:162-170: row-major copy of the error matrix
    std::vector<double> e((size_t)16 * Q);
    for (int r = 0; r < 16; r++) for (int c = 0; c < Q; c++) e[(size_t)r * Q + c] = err_cm[r + 16 * (size_t)c];
    R.h2d(R.err.p, e.data(), e.size() * 8);
    if (R.two_phase) launch_raw_bounds(R.in, R.err.p, Q, o->use_quals != 0, R.raw_S.p, R.raw_rho.p, cx->rank, cx->world, R.s);
  }
  // b_new / b_init (containers.cpp:78-137): one cluster holding every raw in index order; its centre is the first raw with the
  // largest abundance (bi_assign_center), found when the abundances were uploaded
  if (cx->reads_argmax < 0) throw Err{"dada2b: all abundances are zero."};
  const uint32_t c0 = (uint32_t)cx->reads_argmax;
  R.nclust_h = 1;
  R.cl_center_h.push_back(c0); R.cl_reads_h.push_back(cx->total_reads);
  R.birth.emplace_back(); R.birth[0].e = cx->total_reads;
  {
    const uint8_t one = 1;
    R.h2d(R.is_center.p + c0, &one, 1);
    R.h2d(R.slot0.p + 0, &one, 1);
    R.h2d(R.cl_reads.p, &cx->total_reads, 4);
    R.h2d(R.cl_center.p, &c0, 4);
    R.h2d(R.cl_update_e.p, &one, 1); R.h2d(R.cl_check_locks.p, &one, 1);
  }
  // host bookkeeping off the critical path (see Run::ReplayEvent): needs every cluster's centre at slot 0 (abundance-sorted input,
  // what derepFastq produces); DADA2B_SYNC_REPLAY is a test hook.  The member arrays of cluster 0 are then filled by the replay
  // worker while round 0 runs: they are first read by a replayed event or after drain_replay().
  R.async_replay = c0 == 0 && getenv("DADA2B_SYNC_REPLAY") == nullptr;
  if (R.async_replay) R.push_event(Run::ReplayEvent{2, {}, {}, 0, 0, 0});
  else R.init_members();
  TDBG("cluster 0 initialised");
  const double t1 = now_ms();
  const bool dbg = o->verbose || getenv("DADA2B_VERBOSE");
  // run_dada (Rmain.cpp:297-336)
  R.launch_compare(0, 1.0);
  R.launch_round_tail(0, 0);                 // initial cluster: b_p_update + first b_bud scan
  R.sync_report();
  if (dbg) fprintf(stderr, "[dada2b] round 0 done: %.2f ms, cs=%llu\n", now_ms() - t1, R.cs_count);
  const int max_clust = o->max_clust < 1 ? R.nraw : o->max_clust;
  uint32_t wr = 0, wfrom = 0;
  int newi;
  double h_enq = 0, h_wait = 0, h_replay = 0, h_decide = 0;      // host time per phase of a round (verbose diagnostics)
  for (;;) {
    const double td = now_ms();
    if (!(R.nclust_h < max_clust && (newi = R.decide_bud(&wr, &wfrom)))) break;
    const double tr = now_ms();
    h_decide += tr - td;
    R.launch_compare((uint32_t)newi, o->kdist_cutoff);
    R.launch_round_tail(0, R.NP);
    const double te = now_ms();
    R.sync_report();
    const double tw = now_ms();
    int last = R.NP - 1;
    int ran = R.replay_moves(0, last);
    h_enq += te - tr; h_wait += tw - te; h_replay += now_ms() - tw;
    while (!R.h_report->converged && last + 1 < MAX_PASS) {      // rare: more than NP passes needed: one more pass at a time
      last++;
      R.launch_round_tail(last, 1);          // at pass MAX_SHUFFLE - 1 the tail proceeds regardless (dada.h:30, Rmain.cpp:322-325)
      R.sync_report();
      ran += R.replay_moves(last, last);
    }
    R.n_rounds++;
    if (dbg) fprintf(stderr, "[dada2b] C%d seed=%u: round %.3f ms (%d passes), cs=%llu nw=%llu gl=%llu moves=%llu\n", newi,
                     R.cl_center_h[newi], now_ms() - tr, ran, R.cs_count, R.h_report->ctr[CTR_NW], R.h_report->ctr[CTR_GL],
                     R.h_report->ctr[CTR_NMOVE]);
  }
  if (dbg) fprintf(stderr, "[dada2b] loop done: %d clusters; screened %llu, shrouded %llu; host ms: enqueue %.2f, wait for the device %.2f, replay moves %.2f, decide bud %.2f\n",
                   R.nclust_h, R.h_report->ctr[CTR_ALIGN], R.h_report->ctr[CTR_SHROUD], h_enq, h_wait, h_replay, h_decide);
  R.sync();
  const double t2 = now_ms();
  dada2b_out *out = (dada2b_out *)calloc(1, sizeof(dada2b_out));
  try { R.finish(out); } catch (...) { dada2b_free(out); throw; }
  const double t3 = now_ms();
  out->ms_setup = t1 - t0; out->ms_loop = t2 - t1; out->ms_final = t3 - t2; out->ms_total = t3 - t0;
  return out;
}


// ------------------------------- kernel-level test hooks -------------------------------
static void do_test_pairs(dada2b_ctx *cx, int npairs, const uint32_t *centre, const uint32_t *raw, const double *err_cm,
                          int Q, const dada2b_opts *o, int use_kmers, double kdist_cutoff, int32_t *kind, double *lambda,
                          int32_t *nsubs, uint8_t *ops, int32_t *nops, int opcap, uint16_t *pos, uint8_t *nt0,
                          uint8_t *nt1, uint8_t *q1, int subcap) {
  CK(cudaSetDevice(cx->device));
  if (cx->bad_nt) throw Err{"Unexpected nucleotide."};
  Run R;
  R.bind(cx, o, Q);
  R.setup_params();
  R.alloc_state();
  std::vector<double> e((size_t)16 * Q);
  for (int r = 0; r < 16; r++) for (int c = 0; c < Q; c++) e[(size_t)r * Q + c] = err_cm[r + 16 * (size_t)c];
  R.h2d(R.err.p, e.data(), e.size() * 8);
  cudaStream_t s = R.s;
  R.pair_centre.alloc(npairs); R.pair_raw.alloc(npairs);
  R.h2d(R.pair_centre.p, centre, (size_t)npairs * 4);
  R.h2d(R.pair_raw.p, raw, (size_t)npairs * 4);
  R.b_nsubs.alloc(npairs); R.b_nops.alloc(npairs); R.b_lambda.alloc(npairs); R.kind_out.alloc(npairs);
  R.b_pos.alloc((size_t)npairs * subcap); R.b_nt0.alloc((size_t)npairs * subcap); R.b_nt1.alloc((size_t)npairs * subcap);
  R.b_q1.alloc((size_t)npairs * subcap); R.b_ops.alloc((size_t)npairs * opcap);
  R.b_nsubs.zero(s); R.b_nops.zero(s); R.b_lambda.zero(s); R.b_ops.zero(s); R.b_pos.zero(s); R.b_nt0.zero(s); R.b_nt1.zero(s); R.b_q1.zero(s);
  DBuf<uint32_t> nwl, gll; nwl.alloc(npairs); gll.alloc(npairs);
  ClassifyArgs ca{};
  ca.in = R.in; ca.P = R.P; ca.P.use_kmers = use_kmers; ca.P.kdist_cutoff = kdist_cutoff; ca.mode = 1;
  ca.pair_centre = R.pair_centre.p; ca.pair_raw = R.pair_raw.p; ca.nw_list = nwl.p; ca.gl_list = gll.p; ca.ctr = R.st.ctr;
  ca.kord_words = R.kord_words; ca.kind_out = R.kind_out.p; ca.lock = R.st.lock; ca.shard_rank = 0; ca.shard_world = 1;
  launch_classify(ca, npairs, 256, R.classify_smem, s);
  for (int kd : {KIND_NW, KIND_GAPLESS}) {
    AlignArgs a = R.align_args(MODE_BIRTH, kd);
    a.jobs = kd == KIND_NW ? nwl.p : gll.p;
    a.njobs_ptr = R.st.ctr + (kd == KIND_NW ? CTR_NW : CTR_GL);
    a.pair_centre = R.pair_centre.p; a.pair_raw = R.pair_raw.p;
    a.b_nsubs = R.b_nsubs.p; a.b_lambda = R.b_lambda.p; a.b_pos = R.b_pos.p; a.b_nt0 = R.b_nt0.p; a.b_nt1 = R.b_nt1.p;
    a.b_q1 = R.b_q1.p; a.b_cap = subcap; a.b_ops = R.b_ops.p; a.b_nops = R.b_nops.p; a.b_opcap = opcap;
    R.launch_align_jobs(MODE_BIRTH, a, npairs);
  }
  std::vector<uint8_t> hk(npairs); std::vector<uint32_t> hns(npairs), hno(npairs);
  R.d2h(hk.data(), R.kind_out.p, npairs);
  R.d2h(hns.data(), R.b_nsubs.p, (size_t)npairs * 4);
  R.d2h(hno.data(), R.b_nops.p, (size_t)npairs * 4);
  R.d2h(lambda, R.b_lambda.p, (size_t)npairs * 8);
  R.d2h(ops, R.b_ops.p, (size_t)npairs * opcap);
  R.d2h(pos, R.b_pos.p, (size_t)npairs * subcap * 2);
  R.d2h(nt0, R.b_nt0.p, (size_t)npairs * subcap);
  R.d2h(nt1, R.b_nt1.p, (size_t)npairs * subcap);
  R.d2h(q1, R.b_q1.p, (size_t)npairs * subcap);
  R.read_ctr();
  R.check_dev_error();
  for (int k = 0; k < npairs; k++) {
    kind[k] = hk[k];
    nsubs[k] = hk[k] == KIND_SHROUD ? -1 : (int32_t)hns[k];
    nops[k] = (int32_t)hno[k];
    if (hk[k] == KIND_SHROUD) lambda[k] = 0.0;             // compute_lambda of a NULL sub, pval.cpp:150-152
  }
}


// Loop aligners one pair at a time (include/dada2b_test.h): the pair is compared as cluster 0 would (E_minmax = -999: always
// stored, slot = raw index), so (lambda, hamming) can be read back from the comparison store.
static void do_test_loop_nw(dada2b_ctx *cx, int which, int npairs, const uint32_t *centre, const uint32_t *raw, const double *err_cm, int Q,
                            const dada2b_opts *o, uint64_t njobs_hint, double *lambda, int32_t *nsubs, int32_t *handled) {
  CK(cudaSetDevice(cx->device));
  if (cx->bad_nt) throw Err{"Unexpected nucleotide."};
  Run R;
  R.bind(cx, o, Q);
  R.setup_params();
  R.alloc_state();
  cudaStream_t s = R.s;
  std::vector<double> e((size_t)16 * Q);
  for (int r = 0; r < 16; r++) for (int c = 0; c < Q; c++) e[(size_t)r * Q + c] = err_cm[r + 16 * (size_t)c];
  R.h2d(R.err.p, e.data(), e.size() * 8);
  if (R.two_phase) launch_raw_bounds(R.in, R.err.p, Q, o->use_quals != 0, R.raw_S.p, R.raw_rho.p, cx->rank, cx->world, s);
  DBuf<uint32_t> job, uneq, nsb; DBuf<unsigned long long> cnt;
  job.alloc(1); uneq.alloc(4); nsb.alloc(R.nraw); cnt.alloc(4);
  for (int k = 0; k < npairs; k++) {
    const uint32_t c = centre[k], r = raw[k];
    handled[k] = 0; lambda[k] = 0.0; nsubs[k] = -1;
    if (c >= (uint32_t)R.nraw || r >= (uint32_t)R.nraw) throw Err{"dada2b_test_loop_nw: index out of range"};
    launch_fill_f64(R.E_minmax.p, -999.0, R.nraw, s);
    CK(cudaMemsetAsync(R.cs_ham.p + r, 0xFF, 4, s));
    CK(cudaMemsetAsync(nsb.p + r, 0xFF, 4, s));
    cnt.zero(s); R.ctr.zero(s);
    const unsigned long long one = 1;
    R.h2d(cnt.p, &one, 8);                       // cnt[0] = job count, cnt[1] = handed-back count, cnt[2] = survivors
    R.h2d(job.p, &r, 4);
    FwdArgs f{};
    f.in = R.in; f.P = R.P; f.st = R.st; f.jobs = job.p; f.njobs_ptr = cnt.p;
    f.centre_idx = c; f.centre_reads = cx->reads[c]; f.cluster_i = 0; f.total_reads = cx->total_reads;
    f.fb_list = uneq.p; f.fb_count = cnt.p + 1; f.seq_bytes = R.seq_bytes; f.mode = 0; f.job_mul = 1; f.job_add = 0;
    const long worst = (long)R.in.maxlen * std::max(std::abs(R.P.mismatch), std::abs(R.P.match)) + std::max(std::abs(R.P.gap), std::abs(R.P.hgap)) + 16;
    f.fast_ok = (worst < std::abs((long)R.P.sentinel) / 2) ? 1 : 0;
    f.raw_S = R.raw_S.p; f.raw_rho = R.raw_rho.p; f.surv_list = uneq.p + 2; f.surv_count = cnt.p + 2;
    bool launched = false;
    if (which == 0 && R.row_mv.p) launched = launch_nwrow_exact(f, uneq.p, cnt.p + 1, R.row_mv.p, R.row_sub.p, (int)cx->len[c], 1, R.row_grid_cap, s);
    else if (which == 1 && R.lane_mv.p) launched = launch_nwlane(f, uneq.p, cnt.p + 1, R.lane_mv.p, R.lane_sub.p, (int)cx->len[c], R.lane_max, (int)R.lane_max, s);
    else if (which == 2 && R.P.band >= 0) launched = launch_nwfwd(f, R.fwd_slots, 1, njobs_hint, cx->num_sms, s);
    else if (which == 3 && R.row_mv.p && R.two_phase) launched = launch_nwrow_bound(f, uneq.p, cnt.p + 1, (int)cx->len[c], 1, cx->num_sms, 0ull, s, nsb.p);
    if (!launched) continue;
    unsigned long long hc[3]; double lam; uint32_t ham, nsv;
    R.d2h(hc, cnt.p, 24); R.d2h(&lam, R.cs_lambda.p + r, 8); R.d2h(&ham, R.cs_ham.p + r, 4); R.d2h(&nsv, nsb.p + r, 4);
    R.read_ctr();
    R.check_dev_error();
    if (hc[1] != 0) continue;                    // handed on to another kernel
    handled[k] = 1;
    if (which == 3) { nsubs[k] = (int32_t)nsv; }
    else { lambda[k] = lam; nsubs[k] = (int32_t)ham; }
  }
}

// Per-raw factors of the two-phase bound (include/dada2b_test.h): k_raw_bounds over the raws of shard (rank, world), launched as
// do_run launches it; the other raws keep NaN.
static void do_test_raw_bounds(dada2b_ctx *cx, const double *err_cm, int Q, int use_quals, int rank, int world, double *S, double *rho) {
  CK(cudaSetDevice(cx->device));
  if (Q < 1) throw Err{"Error matrix must have 16 rows."};
  if (world < 1 || rank < 0 || rank >= world) throw Err{"dada2b_test_raw_bounds: bad rank/world"};
  if (use_quals && cx->maxq > Q - 1) throw Err{"Rounded quality exceeded range of err lookup table."};
  const size_t n = (size_t)cx->in.nraw;
  std::vector<double> e((size_t)16 * Q);
  for (int r = 0; r < 16; r++) for (int c = 0; c < Q; c++) e[(size_t)r * Q + c] = err_cm[r + 16 * (size_t)c];
  DBuf<double> d_err, d_S, d_rho;
  d_err.alloc(e.size()); d_S.alloc(n); d_rho.alloc(n);
  CK(cudaMemcpyAsync(d_err.p, e.data(), e.size() * 8, cudaMemcpyHostToDevice, cx->stream));
  const double nan = std::numeric_limits<double>::quiet_NaN();
  launch_fill_f64(d_S.p, nan, n, cx->stream); launch_fill_f64(d_rho.p, nan, n, cx->stream);
  launch_raw_bounds(cx->in, d_err.p, Q, use_quals != 0, d_S.p, d_rho.p, rank, world, cx->stream);
  CK(cudaMemcpyAsync(S, d_S.p, n * 8, cudaMemcpyDeviceToHost, cx->stream));
  CK(cudaMemcpyAsync(rho, d_rho.p, n * 8, cudaMemcpyDeviceToHost, cx->stream));
  CK(cudaStreamSynchronize(cx->stream));
}

// The bound pass of one round (include/dada2b_test.h): ONE launch of one bound-testing loop kernel over the caller's job list, with
// the caller's E_minmax per raw and cluster index, as Run::launch_compare launches it.  Every list the kernel writes is read back and
// checked: each raw at most once over all lists, only jobs, counts within the job count.
static void do_test_bound(dada2b_ctx *cx, int which, uint32_t centre, uint32_t cluster_i, int64_t njobs, const uint32_t *jobs, const double *e_minmax,
                          const double *err_cm, int Q, const dada2b_opts *o, uint64_t njobs_hint, int32_t *outcome, int32_t *nsubs, double *lambda,
                          double *e_after, int64_t *counters) {
  CK(cudaSetDevice(cx->device));
  if (cx->bad_nt) throw Err{"Unexpected nucleotide."};
  if (Q < 1) throw Err{"Error matrix must have 16 rows."};
  if (o->use_quals && cx->maxq > Q - 1) throw Err{"Rounded quality exceeded range of err lookup table."};
  if (which < 0 || which > 3) throw Err{"dada2b_test_bound: which must be 0 (k_nwrow<BOUND>), 1 (k_nwlane), 2 (k_nwfwd) or 3 (k_gapless_loop)"};
  if (cluster_i < 1) throw Err{"dada2b_test_bound: cluster_i must be >= 1 (cluster 0 never tests the bound)"};
  const size_t n = (size_t)cx->in.nraw;
  if (centre >= n) throw Err{"dada2b_test_bound: centre out of range"};
  if (njobs < 1 || (size_t)njobs > n) throw Err{"dada2b_test_bound: njobs must be in 1 .. nraw"};
  std::vector<int64_t> job_of(n, -1);
  for (int64_t k = 0; k < njobs; k++) {
    if (jobs[k] >= n) throw Err{"dada2b_test_bound: job out of range"};
    if (job_of[jobs[k]] >= 0) throw Err{"dada2b_test_bound: a raw appears twice in the job list"};
    job_of[jobs[k]] = k;
  }
  Run R;
  R.bind(cx, o, Q);
  R.setup_params();
  R.alloc_state();
  if (!R.two_phase) throw Err{"dada2b_test_bound: homopolymer gap costs have no bound pass"};
  cudaStream_t s = R.s;
  {
    std::vector<double> e((size_t)16 * Q);
    for (int r = 0; r < 16; r++) for (int c = 0; c < Q; c++) e[(size_t)r * Q + c] = err_cm[r + 16 * (size_t)c];
    R.h2d(R.err.p, e.data(), e.size() * 8);
  }
  launch_raw_bounds(R.in, R.err.p, Q, o->use_quals != 0, R.raw_S.p, R.raw_rho.p, cx->rank, cx->world, s);
  R.h2d(R.E_minmax.p, e_minmax, n * 8);
  R.ensure_cs_cap(n + (unsigned long long)njobs + 1024);    // cluster 0 owns entries [0, nraw); a later cluster takes slots by atomics
  const uint64_t nj = (uint64_t)njobs;
  DBuf<uint32_t> d_jobs, l_back, l_surv, l_gl, d_ns; DBuf<unsigned long long> cnt;
  d_jobs.alloc(nj); l_back.alloc(nj + 2); l_surv.alloc(nj); l_gl.alloc(nj); d_ns.alloc(n); cnt.alloc(4);
  R.h2d(d_jobs.p, jobs, nj * 4);
  cnt.zero(s);
  R.h2d(cnt.p, &nj, 8);                               // cnt[0] = job count, [1] handed back, [2] survivors, [3] gapless-listed
  CK(cudaMemsetAsync(d_ns.p, 0xFF, n * 4, s));
  FwdArgs f{};
  f.in = R.in; f.P = R.P; f.st = R.st; f.jobs = d_jobs.p; f.njobs_ptr = cnt.p;
  f.centre_idx = centre; f.centre_reads = cx->reads[centre]; f.cluster_i = cluster_i; f.total_reads = cx->total_reads;
  f.fb_list = l_back.p; f.fb_count = cnt.p + 1; f.seq_bytes = R.seq_bytes; f.mode = 0; f.job_mul = 1; f.job_add = 0;
  {
    const long worst = (long)R.in.maxlen * std::max(std::abs(R.P.mismatch), std::abs(R.P.match)) + std::max(std::abs(R.P.gap), std::abs(R.P.hgap)) + 16;
    f.fast_ok = (worst < std::abs((long)R.P.sentinel) / 2) ? 1 : 0;
  }
  f.raw_S = R.raw_S.p; f.raw_rho = R.raw_rho.p; f.surv_list = l_surv.p; f.surv_count = cnt.p + 2;
  const int len1 = (int)cx->len[centre];
  bool launched = false;
  if (which == 0) {
    f.gl_out = l_gl.p; f.gl_count = cnt.p + 3;
    launched = launch_nwrow_bound(f, l_back.p, cnt.p + 1, len1, nj, cx->num_sms, 0ull, s, d_ns.p);
  } else if (which == 1) {
    if (!R.lane_max || !R.lane_mv.p) throw Err{"dada2b_test_bound: k_nwlane is not set up for this configuration"};
    if (nj > R.lane_max) throw Err{"dada2b_test_bound: more jobs than k_nwlane takes (lane_max)"};
    f.ns_out = d_ns.p;
    launched = launch_nwlane(f, l_back.p, cnt.p + 1, R.lane_mv.p, R.lane_sub.p, len1, R.lane_max, (int)R.lane_max, s);
  } else if (which == 2) {
    if (R.P.band < 0) throw Err{"dada2b_test_bound: k_nwfwd needs a band"};
    f.ns_out = d_ns.p;
    launched = launch_nwfwd(f, R.fwd_slots, nj, njobs_hint, cx->num_sms, s, true);
  } else {
    f.ns_out = d_ns.p;
    launch_gapless_loop(f, 1, nj, cx->num_sms, s);
    launched = true;
  }
  if (!launched) throw Err{"dada2b_test_bound: the kernel does not take this configuration"};
  unsigned long long hc[4];
  std::vector<double> E2(n);
  std::vector<uint32_t> ns(n);
  R.d2h(hc, cnt.p, 32); R.d2h(E2.data(), R.E_minmax.p, n * 8); R.d2h(ns.data(), d_ns.p, n * 4);
  R.read_ctr();
  R.check_dev_error();
  const unsigned long long nstored = R.h_ctr.p[CTR_CS_COUNT] - n;
  if (hc[0] != nj || hc[1] > nj || hc[2] > nj || hc[3] > nj || nstored > nj || hc[1] + hc[2] + hc[3] > nj)
    throw Err{"dada2b_test_bound: a list count is out of range"};
  std::vector<uint32_t> back(hc[1]), surv(hc[2]), gl(hc[3]), cs_idx(nstored), cs_ham(nstored), cs_i(nstored);
  std::vector<double> cs_lam(nstored);
  R.d2h(back.data(), l_back.p, hc[1] * 4); R.d2h(surv.data(), l_surv.p, hc[2] * 4); R.d2h(gl.data(), l_gl.p, hc[3] * 4);
  R.d2h(cs_idx.data(), R.st.cs_index + n, nstored * 4); R.d2h(cs_ham.data(), R.st.cs_ham + n, nstored * 4);
  R.d2h(cs_i.data(), R.st.cs_i + n, nstored * 4); R.d2h(cs_lam.data(), R.st.cs_lambda + n, nstored * 8);
  R.sync();
  const double nan = std::numeric_limits<double>::quiet_NaN();
  for (int64_t k = 0; k < njobs; k++) { outcome[k] = -1; nsubs[k] = -1; lambda[k] = nan; }
  auto mark = [&](uint32_t r, int32_t v, const char *what) {
    if (r >= n || job_of[r] < 0) throw Err{std::string("dada2b_test_bound: a raw that is no job appears in the ") + what};
    if (outcome[job_of[r]] >= 0) throw Err{std::string("dada2b_test_bound: a raw appears twice in the lists (") + what + ")"};
    outcome[job_of[r]] = v;
  };
  for (uint32_t r : surv) mark(r, 1, "survivor list");
  for (uint32_t r : gl) mark(r, 2, "gapless list");
  for (uint32_t r : back) mark(r, 3, "hand-back list");
  for (size_t k = 0; k < nstored; k++) {
    if (cs_i[k] != cluster_i) throw Err{"dada2b_test_bound: a stored comparison carries another cluster index"};
    mark(cs_idx[k], 4, "comparison store");
    lambda[job_of[cs_idx[k]]] = cs_lam[k];
    if (cs_ham[k] != (ns[cs_idx[k]] & 0x7FFFFFFFu)) throw Err{"dada2b_test_bound: the stored hamming differs from the bound pass's nsubs"};
  }
  for (int64_t k = 0; k < njobs; k++) {
    const uint32_t r = jobs[k], w = ns[r];
    const bool written = w != 0xFFFFFFFFu;
    if (written) nsubs[k] = (int32_t)(w & 0x7FFFFFFFu);
    if (outcome[k] == 3) {
      if (written) throw Err{"dada2b_test_bound: a handed-back job was aligned"};
      continue;
    }
    if (!written) throw Err{"dada2b_test_bound: a job was neither aligned nor handed back"};
    if (which == 0) { if (outcome[k] < 0) outcome[k] = 0; continue; }      // k_nwrow<BOUND> writes the bare count
    const bool passed = (w & 0x80000000u) != 0;
    if (which == 2 && passed != (outcome[k] == 1)) throw Err{"dada2b_test_bound: k_nwfwd's survivor list and its bound decision disagree"};
    if (which != 2 && outcome[k] == 4 && !passed) throw Err{"dada2b_test_bound: a job that failed the bound was stored"};
    if (outcome[k] < 0) outcome[k] = passed ? 5 : 0;
  }
  for (size_t r = 0; r < n; r++) e_after[r] = E2[r];
  counters[0] = (int64_t)hc[2]; counters[1] = (int64_t)hc[3]; counters[2] = (int64_t)hc[1]; counters[3] = (int64_t)nstored;
}

// The k-mer screen of one round (include/dada2b_test.h): Run::launch_screen, the round's own launch sequence, for shard (rank, world)
// with the bitmaps of that shard built into this call's Run; the per-raw decision is read back from the gapless / NW lists.
static void do_test_screen(dada2b_ctx *cx, uint32_t centre, const dada2b_opts *o, double kdist_cutoff, uint32_t centre_reads, const uint8_t *lock,
                           int rank, int world, int max_sms, int path, int32_t *kind, int32_t *minsum, int64_t *counters) {
  CK(cudaSetDevice(cx->device));
  if (cx->bad_nt) throw Err{"Unexpected nucleotide."};
  if (world < 1 || rank < 0 || rank >= world) throw Err{"dada2b_test_screen: bad rank/world"};
  if (path != 0 && path != 1) throw Err{"dada2b_test_screen: path must be 0 (product selection) or 1 (k_classify)"};
  if (max_sms < 0) throw Err{"dada2b_test_screen: max_sms must be >= 0"};
  if (centre >= (uint32_t)cx->in.nraw) throw Err{"dada2b_test_screen: centre out of range"};
  Run R;
  R.bind(cx, o, 1);                                      // nothing is aligned: one quality column sizes the unused error table
  R.scr_rank = rank; R.scr_world = world;
  if (max_sms > 0) R.scr_sms = std::min(R.scr_sms, max_sms);
  R.setup_params();
  R.alloc_state();                                       // zeroes the counters and the locks, builds the shard's bitmaps
  const size_t n = (size_t)R.nraw;
  if (lock) R.h2d(R.lock.p, lock, n);
  const bool streaming = path == 0 && R.prescreen && kdist_cutoff < 1.0;
  R.launch_screen(centre, centre_reads, o->greedy != 0, kdist_cutoff, streaming);
  R.read_ctr();
  R.check_dev_error();
  const unsigned long long ngl = R.h_ctr.p[CTR_GL], nnw = R.h_ctr.p[CTR_NW], ncand = streaming ? R.h_ctr.p[CTR_CAND] : 0;
  if (ngl + nnw > n || ncand > (unsigned long long)R.nown) throw Err{"dada2b_test_screen: list count out of range"};
  std::vector<uint32_t> gl(ngl), nw(nnw), cand(ncand);
  std::vector<uint16_t> cms(ncand);
  R.d2h(gl.data(), R.st.gl_list, ngl * 4); R.d2h(nw.data(), R.st.nw_list, nnw * 4);
  R.d2h(cand.data(), R.cand_list.p, ncand * 4); R.d2h(cms.data(), R.cand_ms.p, ncand * 2);
  R.sync();
  for (size_t r = 0; r < n; r++) { kind[r] = (int)(r % world) == rank ? 0 : -1; minsum[r] = -1; }
  auto owned = [&](uint32_t r) {
    if (r >= n || kind[r] < 0) throw Err{"dada2b_test_screen: a raw of another rank was screened"};
  };
  for (int k : {KIND_GAPLESS, KIND_NW})
    for (uint32_t r : k == KIND_GAPLESS ? gl : nw) {
      owned(r);
      if (kind[r] != 0) throw Err{"dada2b_test_screen: a raw appears twice in the gapless / NW lists"};
      kind[r] = k;
    }
  for (size_t k = 0; k < ncand; k++) {
    owned(cand[k]);
    if (minsum[cand[k]] != -1) throw Err{"dada2b_test_screen: a raw appears twice in the candidate list"};
    minsum[cand[k]] = cms[k];
  }
  counters[0] = (int64_t)R.h_ctr.p[CTR_ALIGN]; counters[1] = (int64_t)R.h_ctr.p[CTR_SHROUD];
  counters[2] = (int64_t)ngl; counters[3] = (int64_t)nnw;
}

static void do_test_calc_pA(int n,const int32_t *reads, const double *E, const int32_t *prior, double *out) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw Err{"dada2b: no CUDA device available (this library has no CPU path)."};
  DBuf<int> r, p; DBuf<double> e, o;
  r.alloc(n); p.alloc(n); e.alloc(n); o.alloc(n);
  CK(cudaMemcpy(r.p, reads, (size_t)n * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(p.p, prior, (size_t)n * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e.p, E, (size_t)n * 8, cudaMemcpyHostToDevice));
  launch_calc_pA_vec(r.p, e.p, p.p, o.p, n, 0);
  CK(cudaMemcpy(out, o.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
}

}  // namespace

extern "C" {

int dada2b_test_pairs(dada2b_ctx *ctx, int32_t npairs, const uint32_t *centre, const uint32_t *raw, const double *err,
                      int32_t Q, const dada2b_opts *opts, int32_t use_kmers, double kdist_cutoff, int32_t *kind,
                      double *lambda, int32_t *nsubs, uint8_t *ops, int32_t *nops, int32_t opcap, uint16_t *pos,
                      uint8_t *nt0, uint8_t *nt1, uint8_t *q1, int32_t subcap, char errbuf[DADA2B_ERRLEN]) {
  try { do_test_pairs(ctx, npairs, centre, raw, err, Q, opts, use_kmers, kdist_cutoff, kind, lambda, nsubs, ops, nops, opcap, pos, nt0, nt1, q1, subcap); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}
int dada2b_test_loop_nw(dada2b_ctx *ctx, int32_t which, int32_t npairs, const uint32_t *centre, const uint32_t *raw, const double *err,
                        int32_t Q, const dada2b_opts *opts, uint64_t njobs_hint, double *lambda, int32_t *nsubs, int32_t *handled,
                        char errbuf[DADA2B_ERRLEN]) {
  try { do_test_loop_nw(ctx, which, npairs, centre, raw, err, Q, opts, njobs_hint, lambda, nsubs, handled); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}
int dada2b_test_raw_bounds(dada2b_ctx *ctx, const double *err, int32_t Q, int32_t use_quals, int32_t rank, int32_t world, double *S, double *rho,
                           char errbuf[DADA2B_ERRLEN]) {
  try { do_test_raw_bounds(ctx, err, Q, use_quals, rank, world, S, rho); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}
int dada2b_test_bound(dada2b_ctx *ctx, int32_t which, uint32_t centre, uint32_t cluster_i, int64_t njobs, const uint32_t *jobs, const double *e_minmax,
                      const double *err, int32_t Q, const dada2b_opts *opts, uint64_t njobs_hint, int32_t *outcome, int32_t *nsubs, double *lambda,
                      double *e_after, int64_t *counters, char errbuf[DADA2B_ERRLEN]) {
  try { do_test_bound(ctx, which, centre, cluster_i, njobs, jobs, e_minmax, err, Q, opts, njobs_hint, outcome, nsubs, lambda, e_after, counters); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}
int dada2b_test_screen(dada2b_ctx *ctx, uint32_t centre, const dada2b_opts *opts, double kdist_cutoff, uint32_t centre_reads,
                       const uint8_t *lock, int32_t rank, int32_t world, int32_t max_sms, int32_t path, int32_t *kind, int32_t *minsum,
                       int64_t *counters, char errbuf[DADA2B_ERRLEN]) {
  try { do_test_screen(ctx, centre, opts, kdist_cutoff, centre_reads, lock, rank, world, max_sms, path, kind, minsum, counters); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}
int dada2b_test_calc_pA(int32_t n, const int32_t *reads, const double *E, const int32_t *prior, double *out,
                        char errbuf[DADA2B_ERRLEN]) {
  try { do_test_calc_pA(n, reads, E, prior, out); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}

void dada2b_default_opts(dada2b_opts *o) {            // R/dada.R:1-26
  memset(o, 0, sizeof *o);
  o->match = 5; o->mismatch = -4; o->gap = -8; o->use_kmers = 1; o->kdist_cutoff = 0.42; o->band_size = 16;
  o->omegaA = 1e-40; o->omegaP = 1e-4; o->omegaC = 1e-40; o->detect_singletons = 0; o->max_clust = 0;
  o->min_fold = 1; o->min_hamming = 1; o->min_abund = 1; o->use_quals = 1; o->final_consensus = 0;
  o->vectorized_alignment = 1; o->homo_gap = -8; o->multithread = 1; o->verbose = 0; o->SSE = 2; o->gapless = 1; o->greedy = 1;
}

int dada2b_nccl_unique_id(char id[DADA2B_NCCL_ID_BYTES], char errbuf[DADA2B_ERRLEN]) {
  try {
    std::string why;
    if (!g_nccl.load(why)) throw Err{why};
    static_assert(sizeof(ncclUniqueId) <= DADA2B_NCCL_ID_BYTES, "id buffer");
    ncclUniqueId u;
    NC(g_nccl.GetUniqueId(&u));
    memset(id, 0, DADA2B_NCCL_ID_BYTES);
    memcpy(id, &u, sizeof u);
    return 0;
  } catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
}

int dada2b_comm_init(dada2b_ctx *ctx, int32_t rank, int32_t world, const char id[DADA2B_NCCL_ID_BYTES], char errbuf[DADA2B_ERRLEN]) {
  try {
    if (world < 1 || rank < 0 || rank >= world) throw Err{"dada2b: bad rank/world"};
    if (world == 1) { ctx->rank = 0; ctx->world = 1; ctx->upload_gen++; return 0; }
    std::string why;
    if (!g_nccl.load(why)) throw Err{why};
    CK(cudaSetDevice(ctx->device));
    ncclUniqueId u;
    memcpy(&u, id, sizeof u);
    NC(g_nccl.CommInitRank(&ctx->comm, world, u, rank));
    ctx->rank = rank; ctx->world = world; ctx->upload_gen++;      // the owned rows changed
    return 0;
  } catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
}

int dada2b_upload(const dada2b_in *in, int32_t device, dada2b_ctx **ctx, char errbuf[DADA2B_ERRLEN]) {
  *ctx = nullptr;
  try { *ctx = do_upload(in, device); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}

int dada2b_reupload(dada2b_ctx *ctx, const dada2b_in *in, char errbuf[DADA2B_ERRLEN]) {
  try { do_upload(in, ctx->device, ctx); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}

int dada2b_run_resident(dada2b_ctx *ctx, const double *err, int32_t Q, const dada2b_opts *opts, dada2b_out **out,
                        char errbuf[DADA2B_ERRLEN]) {
  *out = nullptr;
  try { *out = do_run(ctx, err, Q, opts); return 0; }
  catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
}

void dada2b_ctx_free(dada2b_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  for (auto e : ctx->ev_pool) cudaEventDestroy(e);
  delete_run(ctx->run);
  if (ctx->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->comm);
  delete ctx;
}

// One-shot call.  The device/pinned workspace of the previous call on this thread is kept and reused
// (grow-only), like a caching allocator: repeated dada_uniques() calls -- the per-sample loop of
// R/dada.R:266 -- do not pay cudaMalloc/cudaMallocHost again.
int dada2b_run(const dada2b_in *in, const dada2b_opts *opts, dada2b_out **out, char errbuf[DADA2B_ERRLEN]) {
  static thread_local dada2b_ctx *ws = nullptr;
  *out = nullptr;
  try {
    int dev = 0;
    if (ws) dev = ws->device;
    ws = do_upload(in, dev, ws);
  } catch (Err &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.msg.c_str()); return 1; }
  catch (std::exception &e) { snprintf(errbuf, DADA2B_ERRLEN, "%s", e.what()); return 2; }
  int rc = dada2b_run_resident(ws, in->err, in->Q, opts, out, errbuf);
  if (!rc && *out) (*out)->h2d_bytes += ws->upload_h2d;
  return rc;
}

void dada2b_free(dada2b_out *o) {
  if (!o) return;
  free(o->cl_seq_concat); free(o->cl_seq_off); free(o->cl_abundance); free(o->cl_n0); free(o->cl_n1); free(o->cl_nunq);
  free(o->cl_pval); free(o->cl_birth_from); free(o->cl_birth_pval); free(o->cl_birth_fold); free(o->cl_birth_ham);
  free(o->cl_birth_qave); free(o->bs_pos); free(o->bs_ref); free(o->bs_sub); free(o->bs_qual); free(o->bs_clust);
  free(o->subqual); free(o->clusterquals); free(o->map); free(o->pval); free(o);
}

}  // extern "C"
