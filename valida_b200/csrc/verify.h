// Internal interface between the proof-level verifier (host/verifier.cc) and the per-chip
// out-of-domain constraint check (verify.cu).
#pragma once
#include "ctx.h"
#include "host/proof.h"

// *ok = the folded constraints at zeta equal Z_H(zeta) * quotient(zeta).  Returns non-zero only on API errors.
int32_t vg_verify_chip_constraints(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgh::ChipProof& cp, const bb::E5& zeta,
                                   const bb::E5& alpha, const uint32_t perm_challenges_canonical[15], bool* ok);
