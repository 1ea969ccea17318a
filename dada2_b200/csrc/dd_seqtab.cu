// Sequence-table merge on the H100 (include/dada2b_seqtab.h).  Product code.
//
// Replaces the column work of mergeSequenceTables (R/multiSample.R:290-364): the first-occurrence union of the tables'
// column names (:321), tryRC's earlier-reverse-complement test and re-orientation (:322-335), the accumulation of
// every table into the dense result (:337-343) and its column order (:345-352).  Integer work only.  Launch sequence:
//   k_st_pack        every column name -> a forward key and, with try_rc, a reverse-complement key: MSB-first 4-bit
//                    IUPAC codes (8 per word, 0 = padding), then the length, in dd_sort.cuh's [n][KW + 1] layout.
//                    Forward keys are rows 0..C-1 in input order, rc keys rows C..2C-1.  A bad letter sets its bit.
//   radix sort       Sorter's stable LSD passes over (length, last word ... first word): equal sequences are adjacent,
//                    and inside a segment forward keys come first, in input order
//   k_dr_heads, scan segment ids
//   k_st_segs        per sorted key: its segment, the segment's first forward member (the sequence's first occurrence
//                    in R's seqs), and whether the next forward member of the segment lies in the same table
//   k_st_cols        per column: rc_flag (the segment of its rc key has a first forward member before its own first
//                    member), the target segment, collapsed tables, output column candidates; scan -> output columns
//                    in first-seen order
//   k_st_target      per column: its output column, or -1 when superseded (a later column of the same name in the same
//                    table wins, unless the table was collapsed by collapseNoMismatch(identicalOnly = TRUE))
//   -- one host synchronisation: ncol_out, n_rc, bad letters --
//   k_st_accumulate  every cell of every table into an int64 [nrow_out][ncol_out] accumulator; atomics only for tables
//                    whose cells can meet another cell (an output row shared with another table, or a collapsed table)
//   k_st_colsum      column sums, non-zero counts, int32 overflow flag, the complemented sort key
//   radix sort       stable, of the output columns by that key (ties keep first-seen order)
//   k_st_gather      the ordered int32 matrix and the name sources
#include "../../include/dada2b_seqtab.h"
#include "dd_sort.cuh"
#include "dd_flt.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace dd2 {

constexpr uint32_t ST_NONE = 0xffffffffu;
constexpr unsigned ST_NEG = 1u, ST_OVERFLOW = 2u;        // bits of the error word

// 4-bit IUPAC code, one bit per base (A 1, C 2, G 4, T 8; an ambiguity code is the OR of its bases, N = 15); 0 for a
// letter outside the alphabet.  The complement swaps A<->T and C<->G, i.e. reverses the four bits.
__device__ __forceinline__ unsigned st_code(unsigned char c) {
  switch (c) {
    case 'A': return 1; case 'C': return 2; case 'G': return 4; case 'T': return 8;
    case 'M': return 3; case 'R': return 5; case 'S': return 6; case 'V': return 7; case 'W': return 9; case 'Y': return 10;
    case 'H': return 11; case 'K': return 12; case 'D': return 13; case 'B': return 14; case 'N': return 15;
    default: return 0;
  }
}
__device__ __forceinline__ unsigned st_comp(unsigned x) { return ((x & 1u) << 3) | ((x & 2u) << 1) | ((x & 4u) >> 1) | ((x & 8u) >> 3); }

// table of element x given the tables' start offsets off[0..ntab) (strictly increasing: every table is non-empty)
__device__ __forceinline__ int st_tab(const long long *off, int ntab, long long x) {
  int lo = 0, hi = ntab - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (off[mid] <= x) lo = mid; else hi = mid - 1; }
  return lo;
}

struct StPack { const char *names; const long long *off; unsigned ncol, nkey; int KW; uint32_t *keys; unsigned long long *bad; };
__global__ void __launch_bounds__(256) k_st_pack(StPack a) {
  const size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int S = a.KW + 1;
  if (x >= (size_t)a.nkey * S) return;
  const unsigned k = (unsigned)(x / S); const int w = (int)(x % S);
  const bool rc = k >= a.ncol;
  const unsigned j = rc ? k - a.ncol : k;
  const long long o = a.off[j];
  const int len = (int)(a.off[j + 1] - o);
  if (w == a.KW) { a.keys[x] = (uint32_t)len; return; }
  uint32_t v = 0;
  for (int b = 0; b < 8; b++) {
    const int p = 8 * w + b;
    if (p >= len) break;
    const unsigned char c = (unsigned char)a.names[o + (rc ? len - 1 - p : p)];
    unsigned code = st_code(c);
    if (!code && !rc) atomicOr(&a.bad[c >> 6], 1ull << (c & 63));
    if (rc) code = st_comp(code);
    v |= code << (28 - 4 * b);
  }
  a.keys[x] = v;
}

struct StSegs {
  const uint32_t *idx, *head, *seg; unsigned n, ncol; const long long *col_off; int ntab;
  uint32_t *seg_of, *seg_first; uint8_t *next_same;
};
__global__ void __launch_bounds__(256) k_st_segs(StSegs a) {
  const unsigned p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n) return;
  const uint32_t id = a.idx[p], s = a.seg[p] + a.head[p] - 1;
  a.seg_of[id] = s;
  if (a.head[p]) a.seg_first[s] = id < a.ncol ? id : ST_NONE;       // forward keys sort first inside a segment
  if (id < a.ncol) {
    uint8_t same = 0;
    if (p + 1 < a.n && !a.head[p + 1]) {
      const uint32_t nx = a.idx[p + 1];
      same = nx < a.ncol && st_tab(a.col_off, a.ntab, nx) == st_tab(a.col_off, a.ntab, id);
    }
    a.next_same[id] = same;
  }
}

struct StCols {
  unsigned ncol; int try_rc; const uint32_t *seg_of, *seg_first; const long long *col_off; int ntab;
  uint32_t *tgt_seg, *first, *colnum, *collapsed; unsigned long long *n_rc;
};
__global__ void __launch_bounds__(256) k_st_cols(StCols a) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.ncol) return;
  const uint32_t sf = a.seg_of[j], f = a.seg_first[sf];
  uint32_t tgt = sf;
  bool flag = false;
  if (a.try_rc) {
    const uint32_t sr = a.seg_of[a.ncol + j], fr = a.seg_first[sr];
    if (fr != ST_NONE && fr < f) { flag = true; tgt = sr; }        // a palindrome has sr == sf, fr == f: never flagged
  }
  a.tgt_seg[j] = tgt;
  const uint32_t is_first = (f == j && !flag) ? 1u : 0u;
  a.first[j] = is_first; a.colnum[j] = is_first;
  if (flag) {
    a.collapsed[st_tab(a.col_off, a.ntab, j)] = 1u;
    if (f == j) atomicAdd(a.n_rc, 1ull);
  }
}

struct StTarget {
  unsigned ncol; const uint32_t *tgt_seg, *seg_first, *first, *colnum, *collapsed; const uint8_t *next_same;
  const long long *col_off; int ntab; int32_t *out_col; uint32_t *name_src;
};
__global__ void __launch_bounds__(256) k_st_target(StTarget a) {
  const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.ncol) return;
  const bool superseded = a.next_same[j] && !a.collapsed[st_tab(a.col_off, a.ntab, j)];
  a.out_col[j] = superseded ? -1 : (int32_t)a.colnum[a.seg_first[a.tgt_seg[j]]];
  if (a.first[j]) a.name_src[a.colnum[j]] = j;
}

struct StAcc {
  const int32_t *entries; long long ncells; const long long *cell_off, *col_off, *row_off; int ntab;
  const int32_t *row_out, *out_col; const uint32_t *collapsed; const uint8_t *shared;
  unsigned ncol_out; unsigned long long *acc; unsigned *err;
};
__global__ void __launch_bounds__(256) k_st_accumulate(StAcc a) {
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < a.ncells; x += (long long)gridDim.x * blockDim.x) {
    const int32_t v = a.entries[x];
    if (v == 0) continue;
    if (v < 0) { atomicOr(a.err, ST_NEG); continue; }
    const int t = st_tab(a.cell_off, a.ntab, x);
    const long long nc = a.col_off[t + 1] - a.col_off[t], local = x - a.cell_off[t];
    const long long r = local / nc, c = local - r * nc;
    const int32_t orow = a.row_out[a.row_off[t] + r];
    if (orow < 0) continue;
    const int32_t oc = a.out_col[a.col_off[t] + c];
    if (oc < 0) continue;
    unsigned long long *p = a.acc + (size_t)orow * a.ncol_out + oc;
    if (a.shared[t] || a.collapsed[t]) atomicAdd(p, (unsigned long long)v);
    else *p += (unsigned long long)v;                              // the only cell of any table that reaches *p
  }
}

__global__ void __launch_bounds__(256) k_st_colsum(const unsigned long long *acc, unsigned nrow, unsigned ncol, int order_by, uint32_t *key,
                                                   unsigned *err) {
  const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ncol) return;
  unsigned long long sum = 0;
  uint32_t nz = 0;
  bool big = false;
  for (unsigned r = 0; r < nrow; r++) {
    const unsigned long long v = acc[(size_t)r * ncol + k];
    sum += v; nz += v != 0; big |= v > (unsigned long long)INT32_MAX;
  }
  if (big || sum > (unsigned long long)INT32_MAX) atomicOr(err, ST_OVERFLOW);     // no big cell: sum < nrow * 2^31
  key[k] = ~(order_by == DADA2B_ORDER_NSAMPLES ? nz : (uint32_t)sum);               // ascending ~v == descending v
}

__global__ void __launch_bounds__(256) k_st_gather(const unsigned long long *acc, unsigned nrow, unsigned ncol, const uint32_t *ord,
                                                   const uint32_t *name_src, int32_t *out, int32_t *src_out) {
  const long long n = (long long)nrow * ncol;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += (long long)gridDim.x * blockDim.x) {
    const long long r = x / ncol, k = x - r * ncol;
    const uint32_t c = ord[k];
    out[x] = (int32_t)acc[(size_t)r * ncol + c];
    if (r == 0) src_out[k] = (int32_t)name_src[c];
  }
}

static unsigned st_blocks(long long n) { return (unsigned)std::max<long long>(1, std::min<long long>((n + 255) / 256, 1 << 20)); }

}  // namespace dd2

using namespace dd2;

extern "C" {

void dada2b_merge_seqtabs_free(dada2b_seqtab_merge_out *o) {
  if (!o) return;
  free(o->name_src); free(o->mat); free(o);
}

int dada2b_merge_seqtabs(const dada2b_seqtab_merge_in *in, int32_t device, dada2b_seqtab_merge_out **out, char errbuf[DADA2B_ERRLEN]) {
  const double t0 = bnow_ms();
  cudaStream_t s = nullptr;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  dada2b_seqtab_merge_out *res = nullptr;
  int rc = 0;
  std::string msg;
  try {
    if (!in || !out) throw BErr{"dada2b: NULL argument."};
    *out = nullptr;
    const int T = in->ntab;
    if (T < 1) throw BErr{"dada2b: no sequence tables."};
    if (!in->nrow || !in->ncol || !in->names || !in->name_off || !in->row_out || !in->entries) throw BErr{"dada2b: NULL argument."};
    if (in->nrow_out < 1) throw BErr{"dada2b: the merged table needs at least one row."};
    if (in->order_by < DADA2B_ORDER_NONE || in->order_by > DADA2B_ORDER_NSAMPLES) throw BErr{"dada2b: order_by must be 0, 1 or 2."};
    // ---- host checks of the caller's layout (O(tables + columns + rows)) ----
    std::vector<long long> col_off(T + 1, 0), row_off(T + 1, 0), cell_off(T + 1, 0);
    for (int t = 0; t < T; t++) {
      if (in->nrow[t] < 1 || in->ncol[t] < 1) throw BErr{"dada2b: every sequence table needs at least one row and one column."};
      col_off[t + 1] = col_off[t] + in->ncol[t];
      row_off[t + 1] = row_off[t] + in->nrow[t];
      cell_off[t + 1] = cell_off[t] + (long long)in->nrow[t] * in->ncol[t];
    }
    const long long C = col_off[T], R = row_off[T], ncells = cell_off[T];
    const int nk = in->try_rc ? 2 : 1;
    if (C * nk >= (long long)ST_NONE) throw BErr{"dada2b: too many columns."};
    long long maxlen = 0;
    for (long long c = 0; c < C; c++) {
      const long long l = in->name_off[c + 1] - in->name_off[c];
      if (l <= 0) throw BErr{"dada2b: column (sequence) names must not be empty."};
      if (l > INT_MAX / 2) throw BErr{"dada2b: column name too long."};
      maxlen = std::max(maxlen, l);
    }
    // a table whose rows share no output row with another row (of any table) adds without atomics
    std::vector<int32_t> row_uses(in->nrow_out, 0);
    for (long long r = 0; r < R; r++) {
      const int32_t o = in->row_out[r];
      if (o < -1 || o >= in->nrow_out) throw BErr{"dada2b: row_out out of range."};
      if (o >= 0) row_uses[o]++;
    }
    std::vector<uint8_t> shared(T, 0);
    for (int t = 0; t < T; t++)
      for (long long r = row_off[t]; r < row_off[t + 1]; r++) if (in->row_out[r] >= 0 && row_uses[in->row_out[r]] > 1) shared[t] = 1;
    const long long n0 = in->name_off[0], nbytes = in->name_off[C] - n0;
    std::vector<long long> name_off((size_t)C + 1);
    for (long long c = 0; c <= C; c++) name_off[c] = in->name_off[c] - n0;
    const int KW = (int)((maxlen + 7) / 8), S = KW + 1;
    const unsigned ncol = (unsigned)C, nkey = (unsigned)(C * nk);

    need_device(device);
    BCK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (auto &e : ev) BCK(cudaEventCreate(&e));
    long long launches = 0, h2d = 0, d2h = 0;
    BBuf<char> d_names; BBuf<long long> d_name_off, d_col_off, d_row_off, d_cell_off; BBuf<int32_t> d_row_out, d_entries;
    BBuf<uint8_t> d_shared, d_next_same;
    BBuf<uint32_t> d_keys, d_idx, d_idx2, d_head, d_seg, d_seg_of, d_seg_first, d_tgt, d_first, d_colnum, d_collapsed, d_name_src;
    BBuf<int32_t> d_out_col; BBuf<unsigned long long> d_flags;       // [0..4) bad-letter bits, [4] n_rc, [5] error word
    d_names.alloc(nbytes); d_name_off.alloc(C + 1); d_col_off.alloc(T + 1); d_row_off.alloc(T + 1); d_cell_off.alloc(T + 1);
    d_row_out.alloc(R); d_entries.alloc(ncells); d_shared.alloc(T); d_next_same.alloc(ncol);
    d_keys.alloc((size_t)nkey * S); d_idx.alloc(nkey); d_idx2.alloc(nkey); d_head.alloc(nkey); d_seg.alloc(nkey); d_seg_of.alloc(nkey);
    d_seg_first.alloc(nkey); d_tgt.alloc(ncol); d_first.alloc(ncol); d_colnum.alloc(ncol); d_collapsed.alloc(T); d_name_src.alloc(ncol);
    d_out_col.alloc(ncol); d_flags.alloc(6);
    BCK(cudaEventRecord(ev[0], s));
    BCK(cudaMemcpyAsync(d_names.p, in->names + n0, nbytes, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_name_off.p, name_off.data(), (C + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_col_off.p, col_off.data(), (T + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_row_off.p, row_off.data(), (T + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_cell_off.p, cell_off.data(), (T + 1) * 8, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_row_out.p, in->row_out, R * 4, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_entries.p, in->entries, ncells * 4, cudaMemcpyHostToDevice, s));
    BCK(cudaMemcpyAsync(d_shared.p, shared.data(), T, cudaMemcpyHostToDevice, s));
    h2d = nbytes + (C + 1) * 8 + 3LL * (T + 1) * 8 + R * 4 + ncells * 4 + T;
    BCK(cudaMemsetAsync(d_flags.p, 0, 6 * 8, s));
    BCK(cudaMemsetAsync(d_collapsed.p, 0, (size_t)T * 4, s));
    BCK(cudaEventRecord(ev[1], s));
    // ---- keys, sort, segments ----
    Sorter so; so.s = s;
    {
      StPack pa{d_names.p, d_name_off.p, ncol, nkey, KW, d_keys.p, d_flags.p};
      k_st_pack<<<(unsigned)(((size_t)nkey * S + 255) / 256), 256, 0, s>>>(pa);
      uint32_t *ip = d_idx.p;
      k_iota<<<(nkey + 255) / 256, 256, 0, s>>>(ip, nkey);
      launches += 2;
    }
    uint32_t *a = d_idx.p, *b = d_idx2.p;
    int lbytes = 0;
    while (lbytes < 4 && (maxlen >> (8 * lbytes)) != 0) lbytes++;
    for (int by = 0; by < lbytes; by++) { so.pass(RsPass{d_keys.p, S, KW, 8 * by}, a, b, nkey); std::swap(a, b); }
    for (int w = KW - 1; w >= 0; w--)
      for (int by = 0; by < 4; by++) { so.pass(RsPass{d_keys.p, S, w, 8 * by}, a, b, nkey); std::swap(a, b); }
    {
      const uint32_t *kp = d_keys.p; uint32_t *hp = d_head.p;
      k_dr_heads<<<(nkey + 255) / 256, 256, 0, s>>>(kp, S, a, nkey, hp);
      launches += 1;
    }
    BCK(cudaMemcpyAsync(d_seg.p, d_head.p, (size_t)nkey * 4, cudaMemcpyDeviceToDevice, s));
    so.scan(d_seg.p, nkey);
    {
      StSegs sg{a, d_head.p, d_seg.p, nkey, ncol, d_col_off.p, T, d_seg_of.p, d_seg_first.p, d_next_same.p};
      k_st_segs<<<(nkey + 255) / 256, 256, 0, s>>>(sg);
      StCols cl{ncol, in->try_rc ? 1 : 0, d_seg_of.p, d_seg_first.p, d_col_off.p, T, d_tgt.p, d_first.p, d_colnum.p, d_collapsed.p,
                d_flags.p + 4};
      k_st_cols<<<(ncol + 255) / 256, 256, 0, s>>>(cl);
      launches += 2;
    }
    so.scan(d_colnum.p, ncol);
    {
      StTarget tg{ncol, d_tgt.p, d_seg_first.p, d_first.p, d_colnum.p, d_collapsed.p, d_next_same.p, d_col_off.p, T, d_out_col.p,
                  d_name_src.p};
      k_st_target<<<(ncol + 255) / 256, 256, 0, s>>>(tg);
      launches += 1;
    }
    BCK(cudaEventRecord(ev[2], s));
    uint32_t last[2];
    unsigned long long flags[5];
    BCK(cudaMemcpyAsync(&last[0], d_colnum.p + (ncol - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&last[1], d_first.p + (ncol - 1), 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(flags, d_flags.p, 5 * 8, cudaMemcpyDeviceToHost, s));
    BCK(cudaStreamSynchronize(s));                                   // the one synchronisation: ncol_out
    for (int c = 0; c < 256; c++)
      if ((flags[c >> 6] >> (c & 63)) & 1ull) {
        char l[16];
        if (c > 32 && c < 127) snprintf(l, sizeof l, "'%c'", (char)c); else snprintf(l, sizeof l, "byte 0x%02x", c);
        throw BErr{std::string("dada2b: column (sequence) names must be upper-case IUPAC letters (ACGTMRWSYKVHDBN); found ") + l + "."};
      }
    const unsigned ncol_out = last[0] + last[1], nrow_out = (unsigned)in->nrow_out;
    const long long nout = (long long)nrow_out * ncol_out;
    // ---- accumulate, order, gather ----
    BBuf<unsigned long long> d_acc; BBuf<uint32_t> d_key, d_ord, d_ord2; BBuf<int32_t> d_mat, d_src;
    d_acc.alloc(nout); d_key.alloc(ncol_out); d_ord.alloc(ncol_out); d_ord2.alloc(ncol_out); d_mat.alloc(nout); d_src.alloc(ncol_out);
    BCK(cudaEventRecord(ev[3], s));
    BCK(cudaMemsetAsync(d_acc.p, 0, (size_t)nout * 8, s));
    {
      StAcc ac{d_entries.p, ncells, d_cell_off.p, d_col_off.p, d_row_off.p, T, d_row_out.p, d_out_col.p, d_collapsed.p, d_shared.p, ncol_out,
               d_acc.p, (unsigned *)(d_flags.p + 5)};
      k_st_accumulate<<<st_blocks(ncells), 256, 0, s>>>(ac);
      const unsigned long long *ap = d_acc.p; uint32_t *kp = d_key.p, *op = d_ord.p; unsigned *ep = (unsigned *)(d_flags.p + 5);
      const int order = in->order_by;
      k_st_colsum<<<(ncol_out + 255) / 256, 256, 0, s>>>(ap, nrow_out, ncol_out, order, kp, ep);
      k_iota<<<(ncol_out + 255) / 256, 256, 0, s>>>(op, ncol_out);
      launches += 3;
    }
    uint32_t *oa = d_ord.p, *ob = d_ord2.p;
    if (in->order_by != DADA2B_ORDER_NONE)
      for (int by = 0; by < 4; by++) { so.pass(RsPass{d_key.p, 1, 0, 8 * by}, oa, ob, ncol_out); std::swap(oa, ob); }
    {
      const unsigned long long *ap = d_acc.p; const uint32_t *srcp = d_name_src.p; int32_t *mp = d_mat.p, *sp = d_src.p;
      k_st_gather<<<st_blocks(nout), 256, 0, s>>>(ap, nrow_out, ncol_out, oa, srcp, mp, sp);
      launches += 1;
    }
    BCK(cudaEventRecord(ev[4], s));
    res = (dada2b_seqtab_merge_out *)calloc(1, sizeof(dada2b_seqtab_merge_out));
    if (!res) throw BErr{"dada2b: out of host memory."};
    res->name_src = (int32_t *)malloc((size_t)ncol_out * 4);
    res->mat = (int32_t *)malloc((size_t)nout * 4);
    if (!res->name_src || !res->mat) throw BErr{"dada2b: out of host memory."};
    unsigned err = 0;
    BCK(cudaMemcpyAsync(res->mat, d_mat.p, (size_t)nout * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(res->name_src, d_src.p, (size_t)ncol_out * 4, cudaMemcpyDeviceToHost, s));
    BCK(cudaMemcpyAsync(&err, d_flags.p + 5, 4, cudaMemcpyDeviceToHost, s));
    d2h = nout * 4 + (long long)ncol_out * 4 + 4 + 8 + 5 * 8;
    BCK(cudaEventRecord(ev[5], s));
    BCK(cudaStreamSynchronize(s));
    BCK(cudaGetLastError());
    if (err & ST_NEG) throw BErr{"dada2b: sequence table entries must be >= 0."};
    if (err & ST_OVERFLOW) throw BErr{"dada2b: a merged table entry or column sum exceeds the int32 range (R would return NA)."};
    res->ncol_out = (int32_t)ncol_out;
    res->n_rc = (int64_t)flags[4];
    float ms = 0, ms2 = 0;
    BCK(cudaEventElapsedTime(&ms, ev[0], ev[1])); res->ms_h2d = ms;
    BCK(cudaEventElapsedTime(&ms, ev[1], ev[2])); BCK(cudaEventElapsedTime(&ms2, ev[3], ev[4])); res->ms_kernels = ms + ms2;
    BCK(cudaEventElapsedTime(&ms, ev[4], ev[5])); res->ms_d2h = ms;
    BCK(cudaEventElapsedTime(&ms, ev[0], ev[5])); res->ms_device = ms;
    res->gpu_launches = launches + so.launches; res->h2d_bytes = h2d; res->d2h_bytes = d2h;
    res->ms_total = bnow_ms() - t0;
    *out = res; res = nullptr;
  } catch (BErr &e) { msg = e.msg; rc = 1; }
  catch (std::exception &e) { msg = e.what(); rc = 1; }
  for (auto &e : ev) if (e) cudaEventDestroy(e);
  if (s) cudaStreamDestroy(s);
  if (res) dada2b_merge_seqtabs_free(res);
  if (rc && errbuf) snprintf(errbuf, DADA2B_ERRLEN, "%s", msg.c_str());
  return rc;
}

}  // extern "C"
