// FRI parameters of the machine's proofs (basic/src/bin/valida.rs:385-390) and the Merkle digest type.  The prover
// (prover.cc) and the verifier (verifier.cc) must agree on every one of them, so both take them from here.
#pragma once
#include <array>
#include <cstdint>

constexpr int LOG_BLOWUP = 1, NUM_QUERIES = 40, POW_BITS = 8;

using Digest = std::array<uint32_t, 8>;   // canonical words
