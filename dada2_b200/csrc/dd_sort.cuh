// Sequence-set building blocks shared by dereplication (dd_derep.cu) and sample pooling (dd_pool.cu).  Product code.
//   k_dr_pack      sequences -> MSB-first 2-bit keys (16 bases per word, then the length): integer order == lexical order
//   Sorter         stable LSD radix sort of an index array by byte digits, and an exclusive u32 scan
//   k_dr_heads     head[p] = 1 where sorted element p starts a new distinct sequence; k_dr_rank inverts a permutation
//   k_dr_to_ctx    fills a dada() context's packed arrays from device-side uniques (dd_ctx.h)
// The kernels and Sorter's launches live in dd_derep.cu.
#pragma once
#include "dd_hostutil.h"

namespace dd2 {

constexpr int RS_TILE = 2048;          // elements per (one-warp) block of a radix pass

// digit of element `id` in this pass: byte `shift/8` of keys[id * stride + word]
struct RsPass { const uint32_t *keys; int stride, word, shift; };
__device__ __forceinline__ unsigned rs_digit(const RsPass &p, uint32_t id) { return (p.keys[(size_t)id * p.stride + p.word] >> p.shift) & 255u; }

__global__ void __launch_bounds__(32) k_rs_hist(RsPass p, const uint32_t *src, unsigned n, uint32_t *hist, unsigned nb);
__global__ void __launch_bounds__(32) k_rs_scatter(RsPass p, const uint32_t *src, uint32_t *dst, unsigned n, const uint32_t *offs, unsigned nb,
                                                   const uint32_t *hist_total);
__global__ void k_rs_total(const uint32_t *hist, unsigned nb, uint32_t *total);
__global__ void __launch_bounds__(256) k_scan1(const uint32_t *in, uint32_t *out, uint32_t *sums, size_t n);
__global__ void __launch_bounds__(1024) k_scan2(uint32_t *sums, size_t nblocks);
__global__ void __launch_bounds__(256) k_scan3(uint32_t *out, const uint32_t *sums, size_t n);

struct DrIn {
  int nreads, KW, maxlen;              // KW = key words per read
  const char *seq; const uint8_t *qual; const long long *off;
  uint32_t *keys;                      // [nreads][KW + 1]: MSB-first packed bases, then the length
  unsigned long long *flags;           // [0] bad base seen
};
__global__ void __launch_bounds__(256) k_dr_pack(DrIn a);
__global__ void __launch_bounds__(256) k_iota(uint32_t *p, unsigned n);
__global__ void __launch_bounds__(256) k_dr_heads(const uint32_t *keys, int S, const uint32_t *idx, unsigned n, uint32_t *head);
__global__ void __launch_bounds__(256) k_dr_rank(const uint32_t *order, unsigned nuniq, uint32_t *rank_of);   // rank_of[order[r]] = r

// uniques -> dada(): one thread per 16-base word / per quality byte of the context's rows.  Row r is sequence rep[r] of
// (seq, off, keys); its mean qualities are quals[r * maxlen ...]; prior may be NULL (no priors).
struct DrToCtx {
  DevIn in; unsigned nuniq; int maxlen, S;
  const char *seq; const long long *off; const int32_t *rep, *abund; const double *quals; const uint32_t *keys;
  unsigned long long *maxq;
  const uint8_t *prior;
};
__global__ void __launch_bounds__(256) k_dr_to_ctx(DrToCtx a);

struct Sorter {                       // stable LSD radix sort of an index array by byte digits
  cudaStream_t s;
  BBuf<uint32_t> hist, sums, total;
  long long launches = 0;
  void scan(uint32_t *buf, size_t n);                                   // exclusive scan in place
  void pass(const RsPass &p, const uint32_t *a, uint32_t *b, unsigned n);   // sorts a[0..n) by digit `p` into b; caller swaps
};

}  // namespace dd2
