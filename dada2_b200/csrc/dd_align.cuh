// nwalign's warp-per-pair kernel (dd_align.cu), shared with isShiftDenovo's alignment step (dd_collapse.cu).  Product code.
#pragma once
#include "../../include/dada2b_align.h"
#include "dd_evalpair.cuh"
#include "dd_hostutil.h"

namespace dd2 {

struct NwAlignArgs {
  BimSeqs sq;
  AlnParams P;
  const int32_t *s1, *s2;                   // pair -> sequences (s1 = al[0], s2 = al[1])
  const uint32_t *alist;                    // pairs to align (NULL: every pair x < count)
  const unsigned long long *npairs_ptr;     // device-side count (NULL: npairs)
  unsigned long long npairs;
  const int64_t *al_off; int64_t al_base;   // rows of pair x start at al_off[x] - al_base of al1 / al2 (al1 may be NULL)
  char *al1, *al2; int32_t *al_len;
  int32_t *counts;                          // [pair][3] C_eval_pair's match, mismatch, indel (may be NULL)
  uint8_t *flag; int min_overlap;           // isShiftDenovo: flag[s1] = 1 when the pair is a shift (may be NULL)
  unsigned long long *ctr;                  // [0] cells, [2] error flag
  int warp_words, seq_bytes, H_words, ops_words, mask_words, ptr_in_smem;
  uint32_t *ptr_scratch; unsigned long long ptr_words;
};

template <bool GLOBAL> __global__ void __launch_bounds__(128) k_nwalign(NwAlignArgs a);

struct NwAlignPlan { NwAlignArgs a{}; size_t smem = 0; int grid = 1; bool global = false; BBuf<uint32_t> d_ptr; };

// Refuses vec=1 inputs whose scores leave the reference's int16 range (DESIGN.md 24).  maxlen: the longest sequence;
// maxsum: the largest len1 + len2 of a pair (global alignment only).
void check_int16(int match, int mismatch, int gap_p, int endsfree, int maxlen, long long maxsum);

// Scores, sentinel, shared-memory layout and grid of k_nwalign over the packed pool `sq`; allocates the global traceback
// scratch when the move matrix does not fit in shared memory.  Fills everything of pl.a but the pair / output pointers.
void nwalign_plan(NwAlignPlan &pl, const BimSeqs &sq, const dada2b_nwalign_opts &o, int num_sms);
void nwalign_launch(const NwAlignPlan &pl, cudaStream_t s);

}  // namespace dd2
