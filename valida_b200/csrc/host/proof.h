// The proof's wire format: MachineProof (machine/src/proof.rs:13-44) and the (opened_values, proof) pair of
// TwoAdicFriPcs::open_multi_batches, as serde/ciborium writes them.  The prover encodes and the verifier decodes through
// this one module.  Host code only: no CUDA runtime call, so g++ compiles it on its own (tests/test_proof_codec.py).
//
// Field elements are kept as the wire holds them: Montgomery words and bb::E5.  Digests are canonical words, as everywhere
// else on the host (transcript, trees); the codec converts them at the edge.
#pragma once
#include "../bb.cuh"
#include "fri_config.h"
#include <vector>

namespace vgh {

struct BatchOpening { std::vector<std::vector<uint32_t>> opened_values; std::vector<Digest> opening_proof; };   // rows: [matrix][column]
struct CommitPhaseStep { bb::E5 sibling_value{}; std::vector<Digest> opening_proof; };

struct PcsProof {   // TwoAdicFriPcsProof
    std::vector<Digest> commit_phase_commits;
    std::vector<std::vector<CommitPhaseStep>> query_proofs;   // [query][FRI layer]
    bb::E5 final_poly{};
    uint32_t pow_witness = 0;
    std::vector<std::vector<BatchOpening>> query_openings;    // [query][round]
};

struct ChipProof {
    uint32_t log_degree = 0;
    std::vector<bb::E5> preprocessed_local, preprocessed_next, trace_local, trace_next, permutation_local, permutation_next, quotient_chunks;
    bb::E5 cumulative_sum{};
};

struct MachineProof {
    Digest main_trace, perm_trace, quotient_chunks;   // commitments
    PcsProof opening_proof;
    std::vector<ChipProof> chip_proofs;
};

using OpenedValues = std::vector<std::vector<std::vector<std::vector<bb::E5>>>>;   // [round][matrix][point][column]

std::vector<uint8_t> encode(const MachineProof& proof);
std::vector<uint8_t> encode_opening(const OpenedValues& values, const PcsProof& proof);
// Syntax only: exact keys and map sizes, felts below p, no trailing bytes; counts and dimensions are the caller's to check.
// An array length larger than the bytes left is refused before anything is allocated for it.
bool decode(const uint8_t* data, uint64_t len, MachineProof* out);
bool decode_opening(const uint8_t* data, uint64_t len, OpenedValues* values, PcsProof* proof);

}  // namespace vgh
