// Poseidon<BabyBear, CosetMds<_, 16>, 16, 5> on the device: the challenger's permutation (alpha = 5, 4 + 22 + 4 rounds, dense
// 16 x 16 MDS), defined once for proof-of-work grinding (pow.cu) and the Poseidon-16 Merkle trees (merkle.cu).  State words are
// Montgomery; the constants are the context's (vg_poseidon_consts: 480 round constants, then the MDS row-major, Montgomery), read
// by the caller from shared memory so that every lane's read of one constant is a broadcast.
#pragma once
#include "bb.cuh"

namespace p16 {

constexpr int WIDTH = 16, ROUNDS = 30, RC_WORDS = 480, CONST_WORDS = 480 + 256;

__device__ __forceinline__ uint32_t sbox5(uint32_t x) { const uint32_t x2 = bb::sqr(x), x4 = bb::sqr(x2); return bb::mul(x4, x); }

__device__ __forceinline__ void permute(uint32_t s[16], const uint32_t* rc, const uint32_t* mds) {
#pragma unroll 1
    for (int round = 0; round < ROUNDS; round++) {
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = bb::add(s[i], rc[round * 16 + i]);
        if (round >= 4 && round < 26) s[0] = sbox5(s[0]);
        else {
#pragma unroll
            for (int i = 0; i < 16; i++) s[i] = sbox5(s[i]);
        }
        uint32_t o[16];
#pragma unroll
        for (int i = 0; i < 16; i++) {
            uint64_t acc = 0;
#pragma unroll
            for (int j = 0; j < 16; j++) { acc = bb::madw(mds[i * 16 + j], s[j], acc); if ((j & 3) == 3) acc = bb::lazy_fold(acc); }
            o[i] = bb::monty_reduce64(acc);
        }
#pragma unroll
        for (int i = 0; i < 16; i++) s[i] = o[i];
    }
}

// the context's constants into shared memory (every thread of the CTA takes part; the caller synchronises)
__device__ __forceinline__ void load_consts(uint32_t* sc, const uint32_t* __restrict__ consts) {
    for (uint32_t i = threadIdx.x; i < CONST_WORDS; i += blockDim.x) sc[i] = consts[i];
}

}  // namespace p16
