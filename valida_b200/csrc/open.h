#pragma once
#include "ctx.h"
#include <vector>

// 1/(x_i - z) over the committed rows [begin, begin + count) of the coset of height 2^log_H: out[l * count + (i - begin)]
int32_t vg_inverse_denominators(vgpu_ctx* ctx, uint32_t log_H, const bb::E5& z, uint64_t begin, uint64_t count, uint32_t* out);
// out-of-domain evaluation in two halves: enqueue the column sums (no host sync), then host arithmetic on the copied-back sums.
// invden: over the same rows as the part of the matrix held here, limb stride ics.
int32_t vg_eval_columns_enqueue(vgpu_ctx* ctx, const vgpu_dmat* lde, uint32_t npoints, const uint32_t* const* invden, uint64_t ics, uint32_t* d_out /* vg_eval_columns_words(w) */);
uint32_t vg_eval_columns_words(uint32_t w);
// w_first: columns [0, w_first) were summed over the coset g*H, the others over g*w_2h*H (a split proof: vg_eval_columns_first_coset(w); else w)
void vg_eval_columns_finish(const uint32_t* sums, uint64_t H, uint32_t w, uint32_t npoints, const bb::E5* z, std::vector<bb::E5>* ys /* [q][c] */, uint32_t w_first);
uint32_t vg_eval_columns_first_coset(uint32_t w);
int32_t vg_reduced_opening_accumulate(vgpu_ctx* ctx, const vgpu_dmat* lde, const bb::E5* apow_off /* alpha^(off_0 + c), host */, const bb::E5& alpha_w, uint32_t npoints,
                                      const uint32_t* const* invden, uint64_t vcs, const bb::E5* sum_y, uint32_t* ro);
int32_t vg_fri_fold(vgpu_ctx* ctx, const uint32_t* cur, uint64_t ccs, uint64_t n, uint64_t i0, uint64_t count, const bb::E5& beta,
                    const uint32_t* add_v, uint64_t acs, uint32_t* out_v, uint64_t ocs);
int32_t vg_gather_words(vgpu_ctx* ctx, const std::vector<const uint32_t*>& ptrs, std::vector<uint32_t>* out);
namespace vgh { struct Challenger; }
int32_t vg_pow_grind(vgpu_ctx* ctx, vgh::Challenger& ch, int bits, uint32_t* witness_monty);   // pow.cu
