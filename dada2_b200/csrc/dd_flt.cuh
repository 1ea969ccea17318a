// Read-set building blocks shared by the read filter (dd_filter.cu) and primer removal (dd_primer.cu).  Product code.
//   flt_check_reads        one thread per base: letters upper-case IUPAC, qualities 0..93 (flags for the host)
//   FltView, flt_comp      a read as is or reverse-complemented (qualities reversed), without building the copy
//   flt_copy_window        one warp writes a window of such a view to its output offset
//   FltScan                exclusive u64 scan in place (byte offsets of a run exceed 32 bits)
// The kernels behind flt_check_reads and FltScan live in dd_filter.cu.
#pragma once
#include "dd_hostutil.h"

#include <algorithm>
#include <climits>
#include <string>
#include <vector>

namespace dd2 {

constexpr unsigned FULL = 0xffffffffu;

__host__ __device__ __forceinline__ char flt_comp(char c) {  // IUPAC complement (Biostrings' DNA_COMPLEMENT_CODE)
  switch (c) {
    case 'A': return 'T'; case 'T': return 'A'; case 'C': return 'G'; case 'G': return 'C';
    case 'R': return 'Y'; case 'Y': return 'R'; case 'K': return 'M'; case 'M': return 'K';
    case 'B': return 'V'; case 'V': return 'B'; case 'D': return 'H'; case 'H': return 'D';
    default: return c;                                        // S W N
  }
}

// A read as the stages see it: reverse-complemented (qualities reversed) where it was flipped.
struct FltView {
  const char *s; const uint8_t *q; int L; bool flip;
  __device__ char base(int p) const { return flip ? flt_comp(s[L - 1 - p]) : s[p]; }
  __device__ int qual(int p) const { return flip ? q[L - 1 - p] : q[p]; }
};

// Bases [s0, s0 + len) of v and their qualities to oseq / oqual, one warp.
__device__ __forceinline__ void flt_copy_window(const FltView &v, int s0, int len, char *oseq, uint8_t *oqual, int lane) {
  for (int j = lane; j < len; j += 32) { oseq[j] = v.base(s0 + j); oqual[j] = (uint8_t)v.qual(s0 + j); }
}

// One thread per base (k_flt_alpha): bit 2 of *err for a letter that is not upper-case IUPAC, bit 3 for a quality > 93.
void flt_check_reads(const char *seq, const uint8_t *qual, long long nbytes, unsigned *err, cudaStream_t s);

struct FltScan {                                          // in-place exclusive u64 scans on one stream
  cudaStream_t s;
  BBuf<unsigned long long> sums;
  long long launches = 0;
  void operator()(unsigned long long *v, size_t n);
};

inline bool is_acgt(const std::string &s) {
  for (char c : s) if (c != 'A' && c != 'C' && c != 'G' && c != 'T') return false;
  return true;
}

inline void need_device(int32_t device) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw BErr{"dada2b: no CUDA device available (this library has no CPU path)."};
  BCK(cudaSetDevice(device));
}

// Offsets relative to the first read; returns the bytes spanned.
inline long long rebase(int n, const int64_t *seq_off, std::vector<long long> &off) {
  off.resize((size_t)n + 1);
  const long long o0 = seq_off[0];
  for (int r = 0; r < n; r++) {
    const long long l = seq_off[r + 1] - seq_off[r];
    if (l < 0) throw BErr{"Bad sequence offsets."};
    if (l > INT_MAX / 2) throw BErr{"dada2b: read too long."};
    off[r] = seq_off[r] - o0;
  }
  off[n] = seq_off[n] - o0;
  return off[n];
}

}  // namespace dd2
