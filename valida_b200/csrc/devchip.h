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
// the cumulative sum (Montgomery) from the n per-rank totals ([rank][limb]) vg_perm_trace_enqueue left for a chip
void vg_perm_totals_fold(const uint32_t* totals, uint32_t n, uint32_t out[5]);

uint32_t vg_chip_base_constraints(uint32_t chip_id);   // quotient.cu
// every constraint of a chip in eval order: Air::eval's assertions (vg_chip_base_constraints), one per interaction, the 3 LogUp ones
inline uint32_t vg_chip_constraints(const vgpu_chip_desc* chip) { return vg_chip_base_constraints(chip->chip_id) + chip->n_interactions + 3; }
// a description of one of the machine's chips with no more interactions than a DevChip holds
inline bool vg_chip_ok(const vgpu_chip_desc* chip) { return chip && chip->chip_id < VGPU_NUM_CHIPS && chip->n_interactions <= VGPU_MAX_INTERACTIONS; }
// The preprocessed trace of machine chip i (prep[0] / prep[1]: chips 1 / 12), null for the others.
inline const vgpu_dmat* vg_machine_prep(const vgpu_dmat* const prep[2], int i) { return i == 1 ? prep[0] : i == 12 ? prep[1] : nullptr; }
// check.cu — refuses, before anything is enqueued and alike on every rank, what the check sweep cannot read (perm may be null;
// shards: this rank's row shards are accepted)
int32_t vg_check_shapes(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep, const vgpu_dmat* perm, bool shards);
// check.cu — n <= 7 strided copies of n words each, (src, scs) -> (dst, dcs), in one launch of the check's boundary-row copy kernel
struct VgCopySeg { const uint32_t* src; uint64_t scs; uint32_t* dst; uint64_t dcs; uint32_t n; };
int32_t vg_copy_segments(vgpu_ctx* ctx, const VgCopySeg* segs, int n);
// explain.cu — the main columns chip_id's Air::eval reads on the local row and on the next row (bit c % 64 of word c / 64): the unions
// of the constraint catalogue's cells
void vg_air_reads(uint32_t chip_id, uint64_t local[2], uint64_t next[2]);
// check.cu — the same for the 14 + 2 traces of a machine witness (their permutation traces not yet built); `what` names the call
int32_t vg_check_machine(vgpu_ctx* ctx, const char* what, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2]);

// check.cu — the permutation traces of a machine witness (14 chips, prep[0] / prep[1] the preprocessed traces of chips 1 / 12) and,
// when `check`, check_constraints of every chip on this rank's run: vgpu_check_witness and prove's debug mode.  perm(i) enqueues
// chip i's permutation trace; sweep(i) (checking only) its check, which reads the trace before later work on the stream.  finish()
// runs the split chips' windows and the verdict all-gather, then brings the LogUp totals and the verdicts back with ONE copy and one
// synchronisation.  main, prep and challenges must outlive the object.
class CheckSet;
class VgMachineCheck {
  public:
    VgMachineCheck(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2], const uint32_t challenges[15],
                   bool check);
    ~VgMachineCheck();
    const vgpu_dmat* prep_for(int i) const { return vg_machine_prep(prep_, i); }
    int32_t alloc();                                  // reads the traces' heights; enqueues nothing unless checking
    int32_t perm(int i, VgMat* out);
    int32_t sweep(int i, const vgpu_dmat* perm);
    // sums: the cumulative sums (Montgomery); report: the same canonical and each chip's verdict (none failing unless checking)
    int32_t finish(uint32_t sums[VGPU_NUM_CHIPS][5], vgpu_check_report report[VGPU_NUM_CHIPS]);

  private:
    vgpu_ctx* ctx_;
    const vgpu_dmat* const* main_;
    const vgpu_dmat* const* prep_;
    const uint32_t* challenges_;
    std::unique_ptr<CheckSet> set_;                   // null unless checking
    VgBuf res_;                                       // the verdicts (checking only), then the LogUp totals [chip][rank][limb]
    size_t tot_at_ = 0;                               // words
    uint32_t slots_ = 0, nt_[VGPU_NUM_CHIPS] = {};
};
// check_cumulative_sums (machine/src/check_constraints.rs:87-93): the canonical sums of the 14 chips add to zero
bool vg_sums_cancel(const vgpu_check_report report[VGPU_NUM_CHIPS]);
