// mergePairs' fused align / evaluate / consensus kernel (dd_merge.cu), shared with the whole-sample path (dd_pairs.cu).
// Product code.
#pragma once
#include "../../include/dada2b_merge.h"
#include "dd_evalpair.cuh"
#include "dd_hostutil.h"

namespace dd2 {

struct MergeArgs {
  BimSeqs sq;
  AlnParams P;
  int trim_overhang;
  const int32_t *s1_idx, *s2_idx, *prefer;
  int npairs;
  int32_t *counts;                 // [npairs][3] match, mismatch, indel
  char *cons; int cons_stride;     // [npairs][cons_stride]
  int32_t *cons_len;               // [npairs]
  unsigned long long *ctr;         // [1] cells, [2] error flag
  int warp_words, seq_bytes, H_words, ops_words, mask_words, ptr_in_smem;
  uint32_t *ptr_scratch; unsigned long long ptr_words;
};

__global__ void __launch_bounds__(128) k_merge_pairs(MergeArgs a);

// Scores, shared-memory layout and grid of k_merge_pairs for `npairs` pairings over the packed pool `sq`; allocates the
// global traceback scratch when it does not fit in shared memory.  Fills everything of `a` but the pair / output pointers.
void merge_setup(const BimSeqs &sq, const dada2b_merge_opts *opts, int num_sms, int npairs, MergeArgs &a, size_t &smem, int &grid,
                 BBuf<uint32_t> &d_ptr);

}  // namespace dd2
