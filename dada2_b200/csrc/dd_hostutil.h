// Host-side helpers shared by the drivers of dd_bimera.cu and dd_merge.cu (product code).
#pragma once
#include "dd_bimera.cuh"
#include <algorithm>
#include <chrono>
#include <climits>
#include <string>
#include <vector>

namespace dd2 {

struct BErr { std::string msg; };
#define BCK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) throw BErr{std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " #x}; } while (0)

template <typename T> struct BBuf {
  T *p = nullptr; size_t n = 0;
  BBuf() = default;
  BBuf(const BBuf &) = delete;
  BBuf &operator=(const BBuf &) = delete;
  void alloc(size_t count) { release(); n = count; if (count) BCK(cudaMalloc(&p, count * sizeof(T))); }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
  ~BBuf() { release(); }
};

inline double bnow_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }


// 2-bit packing of A/C/G/T sequences (same layout as DevIn::seq2: 16 bases per word, rows of SW words) + upload.
inline void upload_packed_seqs(int nseq, const char *seq_concat, const int64_t *seq_off, cudaStream_t s, BBuf<uint32_t> &d_seq2,
                               BBuf<uint16_t> &d_len, std::vector<uint16_t> &len, BimSeqs &sq, long long &h2d, const char *what) {
  if (nseq <= 0) throw BErr{"Zero input sequences."};
  len.resize(nseq);
  int maxlen = 0, minlen = INT_MAX;
  for (int i = 0; i < nseq; i++) {
    const int64_t l = seq_off[i + 1] - seq_off[i];
    if (l < 0) throw BErr{"Bad sequence offsets."};
    if (l >= 9999) throw BErr{"Input sequences exceed the maximum allowed string length."};
    if (l == 0) throw BErr{"Empty sequences cannot be aligned."};
    len[i] = (uint16_t)l; maxlen = std::max(maxlen, (int)l); minlen = std::min(minlen, (int)l);
  }
  sq.n = nseq; sq.maxlen = maxlen; sq.minlen = minlen; sq.SW = ((maxlen + 15) / 16 + 3) & ~3;
  std::vector<uint32_t> packed((size_t)nseq * sq.SW, 0u);
  bool bad = false;
  for (int r = 0; r < nseq; r++) {
    const char *sp = seq_concat + seq_off[r];
    uint32_t *row = packed.data() + (size_t)r * sq.SW;
    for (int p = 0; p < len[r]; p++) {
      unsigned code;
      switch (sp[p]) { case 'A': code = 0; break; case 'C': code = 1; break; case 'G': code = 2; break; case 'T': code = 3; break;
                       default: code = 0; bad = true; }
      row[p >> 4] |= code << (2 * (p & 15));
    }
  }
  if (bad) throw BErr{std::string("dada2b: ") + what + " needs A/C/G/T sequences (2-bit packed on the device)."};
  d_seq2.alloc(packed.size()); d_len.alloc(nseq);
  BCK(cudaMemcpyAsync(d_seq2.p, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, s));
  BCK(cudaMemcpyAsync(d_len.p, len.data(), (size_t)nseq * 2, cudaMemcpyHostToDevice, s));
  BCK(cudaStreamSynchronize(s));                 // `packed` is pageable and goes out of scope
  h2d += (long long)packed.size() * 4 + (long long)nseq * 2;
  sq.seq2 = d_seq2.p; sq.len = d_len.p;
}

// Per-warp shared-memory layout of a warp-per-pair nw_warp kernel (k_merge_pairs, k_col_align, k_nwalign): the two
// unpacked rows, the diagonal scores H, the move string, three column masks for eval_pair_warp and, when it fits in 96 KB
// per block of four warps, the move matrix; otherwise that goes to a global scratch row per warp.  All sizes in 32-bit
// words except seq_bytes and smem.
struct NwWarpLayout {
  int warp_words, seq_bytes, H_words, ops_words, mask_words, ptr_in_smem;
  unsigned long long ptr_words;
  size_t smem;                                   // dynamic shared memory of a 128-thread block
};

inline NwWarpLayout nw_warp_layout(int maxlen, int minlen, int band) {
  NwWarpLayout L;
  const int lbmax = band < 0 ? maxlen : std::min(band + (maxlen - minlen), maxlen), rbmax = lbmax;
  const int Wmax = lbmax + rbmax + 1;
  const int nchunk = (((Wmax + 1) >> 1) + 31) >> 5;
  L.seq_bytes = (maxlen + 15) & ~15;
  L.H_words = (Wmax + 2 + 3) & ~3;
  L.ops_words = ((2 * maxlen) / 16 + 2 + 3) & ~3;
  L.mask_words = ((2 * maxlen + 31) / 32 + 2 + 3) & ~3;
  L.ptr_words = (unsigned long long)(2 * maxlen + 2) * 2 * nchunk;
  const int base_words = 2 * (L.seq_bytes / 4) + L.H_words + L.ops_words + 3 * L.mask_words;
  L.ptr_in_smem = (4 * ((size_t)base_words + L.ptr_words) * 4 <= 96 * 1024) ? 1 : 0;
  L.warp_words = base_words + (L.ptr_in_smem ? (int)L.ptr_words : 0);
  L.smem = (size_t)4 * L.warp_words * 4;
  if (L.smem > 200 * 1024) throw BErr{"dada2b: band/sequence length too large for the alignment kernel's shared memory."};
  return L;
}

// Copies the layout into a kernel's argument struct (fields of the same names).
template <typename A> inline void set_layout(A &a, const NwWarpLayout &L) {
  a.warp_words = L.warp_words; a.seq_bytes = L.seq_bytes; a.H_words = L.H_words; a.ops_words = L.ops_words;
  a.mask_words = L.mask_words; a.ptr_in_smem = L.ptr_in_smem; a.ptr_words = L.ptr_words;
}

}  // namespace dd2
