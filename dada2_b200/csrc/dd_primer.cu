// Primer removal on the H100 (include/dada2b_primer.h).  Product code.
//
// Replaces the matching block of removePrimers (R/filter.R:118-213) for one file.  Every decision is made on integers:
// mismatch counts, hit positions and window ends, so the output is exact (DESIGN.md 19).
// Launch sequence of one call (dada2b_remove_primers and the hit hook run the same one):
//   k_flt_alpha    (flt_check_reads) one thread per base: letters upper-case IUPAC, qualities 0..93; the host stops
//                  the call on a bad one
//   k_prm_hits     one warp per read, 32 placements per step: the four scans (forward and reverse primer, each against the
//                  read and -- as rc(primer) against the read, positions mirrored -- against its reverse complement).  The
//                  read's letters become four 4-bit IUPAC base planes (A C G T) and a "single base" plane, built by
//                  ballots over 96 positions; a lane's placement compares the primer's planes with the read's 64-bit
//                  window (AND, OR, popc).  Placements off the read's ends see padding letters that match nothing.
//                  Out: per scan the hit count, the first and the last hit; whole-file flags by atomicOr
//   k_prm_decide   one thread per read: the whole-file skip, flip, the first forward / last reverse hit, the trim window
//                  -> reason code, flags, survivor count and length
//   scans          exclusive u64 scans of the survivor counts / lengths (output in input order)
//   k_prm_emit     one warp per survivor: the window, reverse-complemented where flipped, at its output offset
#include "../../include/dada2b_primer.h"
#include "dd_flt.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace dd2 {

constexpr int PRM_WARPS = 8;                    // warps per block of the per-read kernels

__host__ __device__ __forceinline__ unsigned prm_mask(char c) {   // IUPAC base set: A=1 C=2 G=4 T=8 (Biostrings' DNA codes)
  switch (c) {
    case 'A': return 1u; case 'C': return 2u; case 'G': return 4u; case 'T': return 8u;
    case 'R': return 5u; case 'Y': return 10u; case 'S': return 6u; case 'W': return 9u; case 'K': return 12u; case 'M': return 3u;
    case 'B': return 14u; case 'D': return 13u; case 'H': return 11u; case 'V': return 7u; case 'N': return 15u;
    default: return 0u;
  }
}

// One pattern scanned against the read: bit i of plane[b] is set when primer letter i contains base b.  fixed: the
// primer is A/C/G/T only, and a read letter matches only when it is the same single base.  Placements are padded
// shifts lo .. lo + nsh - 1 (per read: nsh = L + 2 pad - P + 1), where padded position t is read position t - PAD.
struct PrmPat {
  unsigned long long plane[4];
  int P, pad, fixed;
};
struct PrmArgs {
  int n, k, PAD;
  const char *seq; const long long *off;
  PrmPat pat[4];                        // forward, reverse, rc(forward), rc(reverse); P = 0: absent
  dada2b_primer_hit *hits;              // [n][4]
  unsigned *flags;                      // bit 0 a forward hit as read, 1 a reverse hit as read, 2 several hits in a scan
                                        // as read, 3 several hits in a scan of the reverse complement
};

__global__ void __launch_bounds__(PRM_WARPS * 32) k_prm_hits(PrmArgs a) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * PRM_WARPS;
  for (int i = blockIdx.x * PRM_WARPS + (threadIdx.x >> 5); i < a.n; i += nw) {
    const long long o = a.off[i];
    const char *s = a.seq + o;
    const int L = (int)(a.off[i + 1] - o);
    int cnt[4], lo[4], hi[4], first[4], last[4];
    int top = -1;                                          // largest placement of any pattern
#pragma unroll
    for (int p = 0; p < 4; p++) {
      cnt[p] = 0; first[p] = INT_MAX; last[p] = INT_MIN;
      lo[p] = a.PAD - a.pat[p].pad;
      hi[p] = a.pat[p].P ? lo[p] + L + 2 * a.pat[p].pad - a.pat[p].P : lo[p] - 1;
      top = max(top, hi[p]);
    }
    unsigned w[3][5];                                      // planes A C G T single of padded positions [b, b + 96)
    auto load = [&](int t0, unsigned *pl) {
      const int r = t0 + lane - a.PAD;
      const unsigned m = (r >= 0 && r < L) ? prm_mask(s[r]) : 0u;
#pragma unroll
      for (int bb = 0; bb < 4; bb++) pl[bb] = __ballot_sync(FULL, (m >> bb) & 1u);
      pl[4] = __ballot_sync(FULL, __popc(m) == 1);
    };
    if (top >= 0) { load(0, w[0]); load(32, w[1]); }
    for (int b = 0; b <= top; b += 32) {
      load(b + 64, w[2]);
      unsigned long long W[5];
#pragma unroll
      for (int j = 0; j < 5; j++) {
        const unsigned long long x = w[0][j] | ((unsigned long long)w[1][j] << 32);
        W[j] = lane ? (x >> lane) | ((unsigned long long)w[2][j] << (64 - lane)) : x;
      }
      const int sp = b + lane;
#pragma unroll
      for (int p = 0; p < 4; p++) {
        const PrmPat &q = a.pat[p];
        unsigned long long m = (q.plane[0] & W[0]) | (q.plane[1] & W[1]) | (q.plane[2] & W[2]) | (q.plane[3] & W[3]);
        if (q.fixed) m &= W[4];
        const int mism = q.P - __popcll(m);
        if (sp >= lo[p] && sp <= hi[p] && mism <= a.k) { cnt[p]++; first[p] = min(first[p], sp); last[p] = max(last[p], sp); }
      }
#pragma unroll
      for (int j = 0; j < 5; j++) { w[0][j] = w[1][j]; w[1][j] = w[2][j]; }
    }
#pragma unroll
    for (int p = 0; p < 4; p++) {
      for (int x = 16; x; x >>= 1) {
        cnt[p] += __shfl_xor_sync(FULL, cnt[p], x);
        first[p] = min(first[p], __shfl_xor_sync(FULL, first[p], x));
        last[p] = max(last[p], __shfl_xor_sync(FULL, last[p], x));
      }
    }
    if (lane == 0) {
      dada2b_primer_hit *h = a.hits + (size_t)i * 4;
#pragma unroll
      for (int p = 0; p < 4; p++) {
        dada2b_primer_hit r{cnt[p], 0, 0, 0, 0};
        if (cnt[p]) {
          const int P = a.pat[p].P;
          const int f1 = first[p] - a.PAD + 1, l1 = last[p] - a.PAD + 1;          // 1-based starts on the read
          // scans 2 and 3: rc(primer) at read [s, s+P-1] is the primer at [L+2-s-P, L+1-s] on the reverse complement, so
          // the read's last hit is the reverse complement's first
          r.first_start = p < 2 ? f1 : L + 2 - l1 - P;
          r.last_start = p < 2 ? l1 : L + 2 - f1 - P;
          r.first_end = r.first_start + P - 1; r.last_end = r.last_start + P - 1;
        }
        h[p] = r;
      }
      const unsigned fl = (cnt[0] ? 1u : 0u) | (cnt[1] ? 2u : 0u) | (cnt[0] > 1 || cnt[1] > 1 ? 4u : 0u) | (cnt[2] > 1 || cnt[3] > 1 ? 8u : 0u);
      if (fl & ~*(volatile unsigned *)a.flags) atomicOr(a.flags, fl);
    }
  }
}

struct PrmDecide {
  int n, has_rev, trim_fwd, trim_rev, orient;
  const long long *off;
  const dada2b_primer_hit *hits;
  const unsigned *flags;
  int *win;                             // [n][2]: 0-based start and length of the kept window in the oriented read
};

// Rules 4-7 of DESIGN.md 19 (R/filter.R:157-212).  acc rows of n+1 u64 (last entry 0): 0 kept, 1 kept length.
__global__ void __launch_bounds__(256) k_prm_decide(PrmDecide d, uint8_t *reason, uint8_t *flags, unsigned long long *acc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t R = (size_t)d.n + 1;
  if (i > d.n) return;
  if (i == d.n) { acc[i] = 0ull; acc[R + i] = 0ull; return; }
  const unsigned ff = *d.flags;
  const dada2b_primer_hit *h = d.hits + (size_t)i * 4;
  const int L = (int)(d.off[i + 1] - d.off[i]);
  int why = 0, fl = 0, first = 0, last = 0;
  if (!(ff & 1u) || (d.has_rev && !(ff & 2u))) {
    why = DADA2B_PRIMER_SKIPPED;                            // :157-158, before any flipping
  } else {
    const bool flip = d.orient && !h[0].count && h[2].count;                     // :181
    const dada2b_primer_hit &hf = h[flip ? 2 : 0], &hr = h[flip ? 3 : 1];
    fl = (flip ? DADA2B_PRIMER_FLIPPED : 0) | (hf.count > 1 ? DADA2B_PRIMER_MULTI_FWD : 0) |
         (d.has_rev && hr.count > 1 ? DADA2B_PRIMER_MULTI_REV : 0);
    if (!hf.count) why = DADA2B_PRIMER_NO_FWD;
    else if (d.has_rev && !hr.count) why = DADA2B_PRIMER_NO_REV;
    else {
      first = d.trim_fwd ? hf.first_end + 1 : 1;                                  // the first forward hit
      last = d.has_rev && d.trim_rev ? hr.last_start - 1 : L;                     // the last reverse hit
      if (!(last > first)) why = DADA2B_PRIMER_EMPTY;
    }
  }
  reason[i] = (uint8_t)why; flags[i] = (uint8_t)fl;
  const bool keep = !why;
  d.win[2 * (size_t)i] = keep ? first - 1 : 0;
  d.win[2 * (size_t)i + 1] = keep ? last - first + 1 : 0;
  acc[i] = keep; acc[R + i] = keep ? (unsigned long long)(last - first + 1) : 0ull;
}

struct PrmOut { char *seq; uint8_t *qual; long long *off; int32_t *src; };

__global__ void __launch_bounds__(PRM_WARPS * 32) k_prm_emit(int n, const char *seq, const uint8_t *qual, const long long *off, const uint8_t *reason,
                                                             const uint8_t *flags, const int *win, const unsigned long long *acc, PrmOut out) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * PRM_WARPS;
  const size_t R = (size_t)n + 1;
  for (int i = blockIdx.x * PRM_WARPS + (threadIdx.x >> 5); i < n; i += nw) {
    if (reason[i]) continue;
    const unsigned long long pos = acc[i], o = acc[R + i];
    const long long ro = off[i];
    const FltView v{seq + ro, qual + ro, (int)(off[i + 1] - ro), (flags[i] & DADA2B_PRIMER_FLIPPED) != 0};
    flt_copy_window(v, win[2 * (size_t)i], win[2 * (size_t)i + 1], out.seq + o, out.qual + o, lane);
    if (lane == 0) { out.src[pos] = i; out.off[pos] = (long long)o; }
  }
}

}  // namespace dd2

using namespace dd2;

namespace {

std::string check_primer(const char *p, const char *what) {
  if (!p || !*p) throw BErr{std::string("dada2b: the ") + what + " primer is empty."};
  const std::string s = p;
  for (char c : s)
    if (!prm_mask(c)) throw BErr{std::string("dada2b: the ") + what + " primer must be upper-case IUPAC letters (A C G T R Y S W K M B D H V N)."};
  if (s.size() > DADA2B_PRIMER_MAXLEN)
    throw BErr{std::string("dada2b: the ") + what + " primer is longer than " + std::to_string(DADA2B_PRIMER_MAXLEN) + " nt."};
  return s;
}

PrmPat make_pat(const std::string &s, int k) {
  PrmPat q{};
  q.P = (int)s.size();
  q.pad = q.P <= k ? q.P - 1 : k;                          // -min_shift of Biostrings' naive inexact matcher
  q.fixed = is_acgt(s);                                    // C_isACGT(primer) (src/evaluate.cpp:184)
  for (int i = 0; i < q.P; i++) {
    const unsigned m = prm_mask(s[i]);
    for (int b = 0; b < 4; b++) if ((m >> b) & 1u) q.plane[b] |= 1ull << i;
  }
  return q;
}

std::string revcomp(const std::string &s) {
  std::string r(s.rbegin(), s.rend());
  for (char &c : r) c = flt_comp(c);
  return r;
}

// The one launch sequence of dada2b_remove_primers and dada2b_test_primer_hits (hook != NULL: the hit records are
// copied out).
int run_primers(const dada2b_derep_in *rd, const dada2b_primer_opts *opts, int32_t device, dada2b_primer_out **out, dada2b_primer_hit *hook,
                char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  dada2b_primer_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!rd || !opts || (!out && !hook)) throw BErr{"dada2b: NULL argument."};
    if (out) *out = nullptr;
    if (opts->allow_indels)
      throw BErr{"dada2b: allow.indels=TRUE is not supported (Biostrings' choice among equal-edit placements is not restated)."};
    if (opts->max_mismatch < 0) throw BErr{"dada2b: max.mismatch must be >= 0."};
    const std::string pf = check_primer(opts->primer_fwd, "forward");
    const bool has_rev = opts->primer_rev != nullptr;
    const std::string pr = has_rev ? check_primer(opts->primer_rev, "reverse") : std::string();
    need_device(device);
    const int n = rd->nreads;
    if (n < 0) throw BErr{"dada2b: negative read count."};
    PrmArgs a{};
    a.n = n; a.k = opts->max_mismatch;
    a.pat[0] = make_pat(pf, a.k); a.pat[2] = make_pat(revcomp(pf), a.k);
    if (has_rev) { a.pat[1] = make_pat(pr, a.k); a.pat[3] = make_pat(revcomp(pr), a.k); }
    for (auto &q : a.pat) a.PAD = std::max(a.PAD, q.pad);
    res = (dada2b_primer_out *)calloc(1, sizeof(dada2b_primer_out));
    res->nreads = n;
    res->reason = (uint8_t *)malloc(std::max(n, 1)); res->flags = (uint8_t *)malloc(std::max(n, 1));
    if (n == 0) {                                          // no read has a hit: the file is skipped
      res->skipped = 1;
      res->src = (int32_t *)malloc(4);
      res->seq_concat = (char *)malloc(1); res->qual_concat = (uint8_t *)malloc(1); res->seq_off = (int64_t *)calloc(1, 8);
      res->ms_total = bnow_ms() - t0;
      if (out) { *out = res; res = nullptr; }
      else { dada2b_primer_free(res); res = nullptr; }
      return 0;
    }
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
    long long h2d = 0, d2h = 0, kbytes = 0, launches = 0;
    std::vector<long long> off;
    const long long nbytes = rebase(n, rd->seq_off, off);
    const long long o0 = rd->seq_off[0];
    BBuf<char> d_seq; BBuf<uint8_t> d_qual; BBuf<long long> d_off; BBuf<unsigned> d_err, d_flags;
    BCK(cudaEventRecord(ev[0], s));
    d_seq.alloc(std::max<long long>(nbytes, 1)); d_qual.alloc(std::max<long long>(nbytes, 1)); d_off.alloc((size_t)n + 1);
    BCK(cudaMemcpyAsync(d_seq.p, rd->seq_concat + o0, nbytes, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_qual.p, rd->qual_concat + o0, nbytes, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_off.p, off.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, s));
    h2d += 2 * nbytes + ((long long)n + 1) * 8;
    d_err.alloc(1); d_flags.alloc(1);
    BCK(cudaMemsetAsync(d_err.p, 0, 4, s));
    BCK(cudaMemsetAsync(d_flags.p, 0, 4, s));
    BCK(cudaEventRecord(ev[1], s));
    if (nbytes) {
      const char *sp = d_seq.p; const uint8_t *qp = d_qual.p; unsigned *ep = d_err.p;
      flt_check_reads(sp, qp, nbytes, ep, s);
      launches++; kbytes += 2 * nbytes;
    }
    {
      unsigned bad = 0;
      BCK(cudaMemcpyAsync(&bad, d_err.p, 4, cudaMemcpyDeviceToHost, s));
      BCK(cudaStreamSynchronize(s));
      if (bad & 4u) throw BErr{"dada2b: reads must be upper-case IUPAC letters (A C G T R Y S W K M B D H V N)."};
      if (bad & 8u) throw BErr{"dada2b: quality values must be 0..93."};
    }
    int nsm = 0;
    BCK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
    const unsigned wgrid = (unsigned)std::max(1, std::min((n + PRM_WARPS - 1) / PRM_WARPS, nsm * 16));
    BBuf<dada2b_primer_hit> d_hits; BBuf<uint8_t> d_reason, d_fl; BBuf<int> d_win; BBuf<unsigned long long> d_acc;
    d_hits.alloc((size_t)n * 4); d_reason.alloc(n); d_fl.alloc(n); d_win.alloc((size_t)n * 2);
    const size_t R = (size_t)n + 1;
    d_acc.alloc(R * 2);
    a.seq = d_seq.p; a.off = d_off.p; a.hits = d_hits.p; a.flags = d_flags.p;
    k_prm_hits<<<wgrid, PRM_WARPS * 32, 0, s>>>(a);
    PrmDecide dc{n, has_rev ? 1 : 0, opts->trim_fwd ? 1 : 0, opts->trim_rev ? 1 : 0, opts->orient ? 1 : 0, d_off.p, d_hits.p, d_flags.p, d_win.p};
    uint8_t *reason_p = d_reason.p, *fl_p = d_fl.p;
    unsigned long long *acc_p = d_acc.p;
    k_prm_decide<<<(unsigned)((R + 255) / 256), 256, 0, s>>>(dc, reason_p, fl_p, acc_p);
    launches += 2;
    const long long hb = (long long)n * 4 * (long long)sizeof(dada2b_primer_hit);
    kbytes += nbytes + (long long)R * 8 + hb + hb + (long long)R * 8 + 2LL * n + 8LL * n + (long long)R * 2 * 8;
    FltScan scan; scan.s = s;
    for (int k = 0; k < 2; k++) scan(acc_p + k * R, R);
    launches += scan.launches; kbytes += (long long)R * 2 * 8 * 4;
    unsigned long long tot[2] = {0, 0};
    unsigned ff = 0;
    for (int k = 0; k < 2; k++) BCK(cudaMemcpyAsync(&tot[k], d_acc.p + k * R + n, 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&ff, d_flags.p, 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));
    const long long nout = (long long)tot[0], obytes = (long long)tot[1];
    res->nout = (int32_t)nout;
    res->skipped = !(ff & 1u) || (has_rev && !(ff & 2u));
    res->multi = !res->skipped && ((ff & 4u) || (opts->orient && (ff & 8u)));
    BBuf<char> o_seq; BBuf<uint8_t> o_qual; BBuf<long long> o_off; BBuf<int32_t> o_src;
    o_src.alloc(std::max<long long>(nout, 1)); o_seq.alloc(std::max<long long>(obytes, 1)); o_qual.alloc(std::max<long long>(obytes, 1));
    o_off.alloc((size_t)nout + 1);
    if (nout) {
      PrmOut po{o_seq.p, o_qual.p, o_off.p, o_src.p};
      const char *sp = d_seq.p; const uint8_t *qp = d_qual.p; const long long *op = d_off.p; const int *wp = d_win.p;
      k_prm_emit<<<wgrid, PRM_WARPS * 32, 0, s>>>(n, sp, qp, op, reason_p, fl_p, wp, acc_p, po);
      launches++;
      kbytes += 2LL * n + nout * (8 + 16 + 4 + 8 + 16) + 4 * obytes;
    }
    BCK(cudaEventRecord(ev[2], s));
    BCK(cudaMemcpyAsync(res->reason, d_reason.p, n, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->flags, d_fl.p, n, cudaMemcpyDeviceToHost, s));
    res->src = (int32_t *)malloc((size_t)std::max<long long>(nout, 1) * 4);
    res->seq_concat = (char *)malloc(std::max<long long>(obytes, 1));
    res->qual_concat = (uint8_t *)malloc(std::max<long long>(obytes, 1));
    res->seq_off = (int64_t *)malloc(((size_t)nout + 1) * 8);
    BCK(cudaMemcpyAsync(res->src, o_src.p, (size_t)nout * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->seq_concat, o_seq.p, obytes, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->qual_concat, o_qual.p, obytes, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->seq_off, o_off.p, (size_t)nout * 8, cudaMemcpyDeviceToHost, s));
    d2h += 2LL * n + nout * 12 + 2 * obytes;
    if (hook) {
      BCK(cudaMemcpyAsync(hook, d_hits.p, (size_t)hb, cudaMemcpyDeviceToHost, s));
      d2h += hb;
    }
    BCK(cudaEventRecord(ev[3], s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    res->seq_off[nout] = obytes;
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
  if (res) dada2b_primer_free(res);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

}  // namespace

extern "C" {

void dada2b_primer_default_opts(dada2b_primer_opts *o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));                               // removePrimers (R/filter.R:81-85)
  o->max_mismatch = 2; o->allow_indels = 0; o->trim_fwd = 1; o->trim_rev = 1; o->orient = 1;
}

void dada2b_primer_free(dada2b_primer_out *o) {
  if (!o) return;
  free(o->reason); free(o->flags); free(o->src); free(o->seq_concat); free(o->seq_off); free(o->qual_concat);
  free(o);
}

int dada2b_remove_primers(const dada2b_derep_in *reads, const dada2b_primer_opts *opts, int32_t device, dada2b_primer_out **out,
                          char errbuf[DADA2B_ERRLEN]) {
  if (!out) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "dada2b: NULL argument."); return 1; }
  return run_primers(reads, opts, device, out, nullptr, errbuf);
}

int dada2b_test_primer_hits(const dada2b_derep_in *reads, const dada2b_primer_opts *opts, int32_t device, dada2b_primer_hit *out,
                            char errbuf[DADA2B_ERRLEN]) {
  if (!out) { if (errbuf) snprintf(errbuf, DADA2B_ERRLEN, "dada2b: NULL argument."); return 1; }
  return run_primers(reads, opts, device, nullptr, out, errbuf);
}

}  // extern "C"
