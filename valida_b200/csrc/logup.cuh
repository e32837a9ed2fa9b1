// eval_permutation_constraints (machine/src/chip.rs:210-289) for one row, written against the builder concept of airs.cuh plus
// b.z_ext(E5) (AirBuilder::assert_zero_ext) and the selector values b.first / b.last / b.trans.  One text serves the quotient sweep
// over the LDE (quotient.cu) and the constraint check over the trace (check.cu), so both number the LogUp constraints alike:
// one per interaction (rlc * phi_m - 1), then the transition, first-row and last-row constraints.
#pragma once
#include "devchip.h"
#include "airs.cuh"

namespace logup {

using bb::E5;

// VirtualPairCol::apply on one row: mrow / prow point at the row's element of column 0, columns are mcs / pcs words apart
__device__ __forceinline__ uint32_t pair_col(const DevPairCol& pc, const uint32_t* mrow, uint64_t mcs, const uint32_t* prow, uint64_t pcs) {
    uint32_t v = pc.constant;
    for (uint32_t t = 0; t < pc.n_terms; t++) {
        uint32_t x = pc.is_prep[t] ? __ldg(prow + (uint64_t)pc.column[t] * pcs) : __ldg(mrow + (uint64_t)pc.column[t] * mcs);
        v = bb::add(v, bb::mul(x, pc.weight[t]));
    }
    return v;
}
// extension element m of a flattened permutation row (base columns 5m .. 5m + 4)
__device__ __forceinline__ E5 load_e5(const uint32_t* row, uint64_t cs, uint32_t m) {
    E5 r;
#pragma unroll
    for (int l = 0; l < 5; l++) r.c[l] = __ldg(row + (uint64_t)(5 * m + l) * cs);
    return r;
}

// ml / mn, pl / pn (null without a preprocessed trace), ql / qn: main, preprocessed and permutation traces offset to the local / next
// row; mcs, pcs, qcs: their column strides.
template <class B>
__device__ __forceinline__ void eval_constraints(B& b, const DevChip& chip, const uint32_t* ml, const uint32_t* mn, uint64_t mcs,
                                                 const uint32_t* pl, const uint32_t* pn, uint64_t pcs,
                                                 const uint32_t* ql, const uint32_t* qn, uint64_t qcs, const E5& cumsum) {
    const uint32_t k = chip.n_interactions;
    const E5 phi_local = load_e5(ql, qcs, k), phi_next = load_e5(qn, qcs, k);
    E5 rhs = bb::e5_zero(), phi0 = bb::e5_zero();
    for (uint32_t m = 0; m < k; m++) {
        const DevInteraction& it = chip.interactions[m];
        bb::Lazy5 ra; ra.init();
        for (uint32_t f = 0; f < it.n_fields; f++) ra.fma_base(chip.betas[f], pair_col(it.fields[f], ml, mcs, pl, pcs));
        const E5 rlc = bb::e5_add(it.alpha, ra.value());
        const E5 pm_l = load_e5(ql, qcs, m), pm_n = load_e5(qn, qcs, m);
        b.z_ext(bb::e5_sub_base(bb::e5_mul(rlc, pm_l), bb::R1));
        const uint32_t mult_l = pair_col(it.count, ml, mcs, pl, pcs), mult_n = pair_col(it.count, mn, mcs, pn, pcs);
        const E5 tl = bb::e5_mul_base(pm_l, mult_l), tn = bb::e5_mul_base(pm_n, mult_n);
        if (it.is_send) { phi0 = bb::e5_add(phi0, tl); rhs = bb::e5_add(rhs, tn); }
        else { phi0 = bb::e5_sub(phi0, tl); rhs = bb::e5_sub(rhs, tn); }
    }
    b.z_ext(bb::e5_mul_base(bb::e5_sub(bb::e5_sub(phi_next, phi_local), rhs), b.trans.v));
    b.z_ext(bb::e5_mul_base(bb::e5_sub(phi_local, phi0), b.first.v));
    b.z_ext(bb::e5_mul_base(bb::e5_sub(phi_local, cumsum), b.last.v));
}

}  // namespace logup
