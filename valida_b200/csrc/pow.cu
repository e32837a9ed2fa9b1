// K11 — proof-of-work grinding on the device: DuplexChallenger::grind(bits) of p3-challenger as used by p3-fri's prover
// (FriConfig{proof_of_work_bits: 8}, basic/src/bin/valida.rs:385-390) [P3-UNVERIFIED: the reference searches with rayon's
// find_any and may return any witness; this search returns the SMALLEST one, which the verifier's check_witness accepts
// like any other].  One thread per candidate: overlay the candidate on the sponge state, run Poseidon-16 (poseidon.cuh,
// constants from shared memory as broadcast reads), test the low bits of the last lane.
// ~2000 candidates cost one launch (~50 us) where the host search took ~3 ms of otherwise idle GPU time per proof.
#include "ctx.h"
#include "poseidon.cuh"
#include "host/challenger.h"

namespace {

__global__ void __launch_bounds__(256) pow_grind_kernel(const uint32_t* __restrict__ consts /* 480 rc + 256 mds, Montgomery */, const uint32_t* __restrict__ base_state,
                                                       uint32_t slot, uint32_t w0, uint32_t count, uint32_t mask, uint32_t* __restrict__ result) {
    __shared__ uint32_t sc[p16::CONST_WORDS];
    p16::load_consts(sc, consts);
    __syncthreads();
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= count) return;
    const uint32_t w = w0 + gid;
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 16; i++) s[i] = base_state[i];
#pragma unroll
    for (int i = 0; i < 16; i++) if ((uint32_t)i == slot) s[i] = bb::to_monty(w);
    p16::permute(s, sc, sc + p16::RC_WORDS);
    if ((bb::from_monty(s[15]) & mask) == 0) atomicMin(result, w);
}

}  // namespace

// The context's Poseidon-16 constants on the device (480 round constants + the MDS, Montgomery; then 17 words of grinding
// scratch), uploaded on first use after vgpu_set_challenger.
int32_t vg_poseidon_consts(vgpu_ctx* ctx, uint32_t** out) {
    if (!ctx->challenger_set) VG_FAIL(ctx, "Poseidon-16: vgpu_set_challenger has not been called");
    if (!ctx->d_poseidon) {
        vgh::Poseidon16 perm;
        perm.set(ctx->poseidon_rc, ctx->poseidon_has_mds ? ctx->poseidon_mds : nullptr);
        std::vector<uint32_t> c(p16::CONST_WORDS);
        for (int i = 0; i < 480; i++) c[i] = perm.rc[i];
        for (int i = 0; i < 16; i++) for (int j = 0; j < 16; j++) c[480 + i * 16 + j] = perm.mds[i][j];
        VG_TRY(vg_alloc(ctx, (void**)&ctx->d_poseidon, (c.size() + 16 + 1) * 4));
        VG_CUDA(ctx, cudaMemcpyAsync(ctx->d_poseidon, c.data(), c.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    *out = ctx->d_poseidon;
    return 0;
}

// Smallest canonical witness w with check_witness(bits, w); the challenger is advanced exactly as grind() would.
int32_t vg_pow_grind(vgpu_ctx* ctx, vgh::Challenger& ch, int bits, uint32_t* witness_monty) {
    if (ch.input.size() >= 16) VG_FAIL(ctx, "grind: the sponge has a full input buffer");
    uint32_t* consts = nullptr;
    VG_TRY(vg_poseidon_consts(ctx, &consts));
    uint32_t* d_state = consts + p16::CONST_WORDS;
    uint32_t* d_result = d_state + 16;
    uint32_t hs[17];
    for (int i = 0; i < 16; i++) hs[i] = i < (int)ch.input.size() ? ch.input[i] : ch.state[i];
    const uint32_t slot = (uint32_t)ch.input.size(), mask = (1u << bits) - 1;
    const uint32_t batch = 2048;
    for (uint32_t w0 = 0; w0 < bb::P; w0 += batch) {
        hs[16] = 0xffffffffu;
        VG_CUDA(ctx, cudaMemcpyAsync(d_state, hs, 17 * 4, cudaMemcpyHostToDevice, ctx->stream));
        const uint32_t count = bb::P - w0 < batch ? bb::P - w0 : batch;
        pow_grind_kernel<<<(count + 255) / 256, 256, 0, ctx->stream>>>(consts, d_state, slot, w0, count, mask, d_result);
        VG_LAUNCH_CHECK(ctx);
        uint32_t found = 0;
        VG_CUDA(ctx, cudaMemcpyAsync(&found, d_result, 4, cudaMemcpyDeviceToHost, ctx->stream));
        VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (found != 0xffffffffu) {
            const uint32_t wm = bb::to_monty(found);
            if (!ch.check_witness(bits, wm)) VG_FAIL(ctx, "grind: the device's witness fails the host check");
            *witness_monty = wm;
            return 0;
        }
    }
    VG_FAIL(ctx, "grind: no witness");
}
