// Device image of a vgpu_chip_desc with the LogUp randomness folded in (Montgomery words):
// alphas per interaction = r1^(bus+1) (generate_rlc_elements, machine/src/chip.rs:291-331),
// betas[j] = r2^j (chip.rs:133).
#pragma once
#include "ctx.h"

struct DevPairCol {
    uint32_t constant;
    uint32_t n_terms;
    uint32_t is_prep[VGPU_MAX_TERMS], column[VGPU_MAX_TERMS], weight[VGPU_MAX_TERMS];
};
struct DevInteraction {
    uint32_t n_fields;
    DevPairCol fields[VGPU_MAX_FIELDS];
    DevPairCol count;
    uint32_t is_send;
    bb::E5 alpha;
};
struct DevChip {
    uint32_t chip_id, width, prep_width, n_interactions;
    DevInteraction interactions[VGPU_MAX_INTERACTIONS];
    bb::E5 betas[VGPU_MAX_FIELDS];
};

int32_t vg_build_devchip(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const uint32_t challenges_canonical[15], DevChip* out);
int32_t vg_prefix_sum_columns(vgpu_ctx* ctx, uint32_t* data, uint64_t cs, uint64_t n, uint32_t ncols);
int32_t vg_ext_batch_inverse(vgpu_ctx* ctx, uint32_t* data, uint64_t cs, uint64_t h, uint32_t groups);
int32_t vg_perm_trace_enqueue(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                              const uint32_t challenges[15], vgpu_dmat** out_perm, uint32_t* d_totals, uint32_t* n_totals);
uint32_t vg_perm_totals_ranks(const vgpu_ctx* ctx);
// check.cu — check_constraints of one chip on whole traces; d_first / d_count must hold ~0 / 0 before the sweep
int32_t vg_check_enqueue(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null, const vgpu_dmat* perm,
                         const uint32_t challenges[15], unsigned long long* d_first, unsigned long long* d_count);
void vg_check_decode(const unsigned long long first_count[2], int64_t* row, uint32_t* constraint, uint64_t* failing_rows);
// the 14 chips' verdicts (first keys [14], then failing-row counts [14]) and canonical cumulative sums -> reports
void vg_check_reports(const unsigned long long* chk, const uint32_t cumsum[VGPU_NUM_CHIPS][5], vgpu_check_report out[VGPU_NUM_CHIPS]);
// check_cumulative_sums (machine/src/check_constraints.rs:87-93): the canonical sums of the 14 chips add to zero
bool vg_sums_cancel(const uint32_t cumsum[VGPU_NUM_CHIPS][5]);
