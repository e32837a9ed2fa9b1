// ORACLE — TEST INFRASTRUCTURE ONLY.  The oracle (oracle/*.h, oracle/oracle_api.cc) with its Merkle trees hashed by Poseidon-16
// instead of Keccak-256: the MMCS a Plonky3 user configures as
//   FieldMerkleTreeMmcs<Val, PaddingFreeSponge<Perm16, 16, 8, 8>, TruncatedPermutation<Perm16, 2, 8, 16>, 8>
// over the challenger's permutation, the reference for vgpu_ctx_set_merkle_hash(VGPU_MERKLE_POSEIDON16).
// [P3-UNVERIFIED: restated from the p3-symmetric definitions, not checked against a Plonky3 build]:
//  * leaf  = PaddingFreeSponge<WIDTH 16, RATE 8, OUT 8>: the state starts at zero; the concatenated rows of the matrices of one
//            height (stable order, as oracle/merkle.h) are absorbed 8 elements at a time by OVERWRITING state[0..len) of each
//            chunk, with one permutation after each chunk, a trailing partial chunk included, and none extra when 8 divides the
//            length (ceil(n/8) in all); the digest is state[0..8);
//  * node  = TruncatedPermutation<N 2, CHUNK 8, WIDTH 16>: the first 8 elements of permute(left || right);
//  * shorter matrices join as in oracle/merkle.h: node = compress(compress(left, right), hash(rows of those matrices)).
// Built as its own library (tests/poseidon_mmcs.py compiles it): oracle/merkle.h is included with its two hash-dependent
// functions renamed, merkle_commit and merkle_verify are defined here with the Poseidon-16 hash, and oracle_api.cc is compiled
// on top, so every orc_* entry point (commit, open, prove, verify) is the oracle's own text with these trees.  The permutation of
// the trees is set by orc_mmcs_set_round_constants (CosetMds, as the challenger's).
#include "../../oracle/field.h"
#include "../../oracle/keccak.h"
#include "../../oracle/poseidon.h"
#include "../../oracle/ntt.h"
#define merkle_commit keccak_merkle_commit
#define merkle_verify keccak_merkle_verify
#include "../../oracle/merkle.h"
#undef merkle_commit
#undef merkle_verify

namespace orc {

static Poseidon16 g_mmcs_perm;

static inline Digest p16_hash(const std::vector<const uint32_t*>& slices, const std::vector<size_t>& lens) {
    uint32_t s[16] = {0};
    size_t k = 0;
    for (size_t i = 0; i < slices.size(); i++)
        for (size_t j = 0; j < lens[i]; j++) {
            s[k++] = slices[i][j];
            if (k == 8) { g_mmcs_perm.permute(s); k = 0; }
        }
    if (k) g_mmcs_perm.permute(s);
    Digest d;
    std::memcpy(d.data(), s, 32);
    return d;
}
static inline Digest p16_compress(const Digest& l, const Digest& r) {
    uint32_t s[16];
    std::memcpy(s, l.data(), 32);
    std::memcpy(s + 8, r.data(), 32);
    g_mmcs_perm.permute(s);
    Digest d;
    std::memcpy(d.data(), s, 32);
    return d;
}
static inline Digest p16_hash_rows(const std::vector<const Matrix*>& mats, size_t row) {
    std::vector<const uint32_t*> sl;
    std::vector<size_t> ln;
    for (const Matrix* m : mats) { sl.push_back(m->row(row)); ln.push_back(m->width); }
    return p16_hash(sl, ln);
}

// oracle/merkle.h's merkle_commit and merkle_verify with the Poseidon-16 hash and compression
static inline MerkleTree merkle_commit(std::vector<Matrix> leaves) {
    MerkleTree t;
    t.leaves = std::move(leaves);
    std::vector<size_t> order(t.leaves.size());
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return t.leaves[a].height() > t.leaves[b].height(); });
    size_t pos = 0;
    const size_t max_h = t.leaves[order[0]].height();
    std::vector<const Matrix*> tallest;
    while (pos < order.size() && t.leaves[order[pos]].height() == max_h) tallest.push_back(&t.leaves[order[pos++]]);
    std::vector<Digest> first(max_h);
#pragma omp parallel for schedule(static) if (max_h > 256)
    for (long i = 0; i < (long)max_h; i++) first[i] = p16_hash_rows(tallest, (size_t)i);
    t.layers.push_back(std::move(first));
    while (t.layers.back().size() > 1) {
        const std::vector<Digest>& prev = t.layers.back();
        const size_t next_len = prev.size() / 2;
        std::vector<const Matrix*> inject;
        while (pos < order.size() && (1ull << log2_ceil(t.leaves[order[pos]].height())) == next_len) inject.push_back(&t.leaves[order[pos++]]);
        std::vector<Digest> next(next_len);
#pragma omp parallel for schedule(static) if (next_len > 256)
        for (long i = 0; i < (long)next_len; i++) {
            Digest d = p16_compress(prev[2 * i], prev[2 * i + 1]);
            if (!inject.empty()) d = p16_compress(d, p16_hash_rows(inject, (size_t)i));
            next[i] = d;
        }
        t.layers.push_back(std::move(next));
    }
    assert(pos == order.size());
    return t;
}

static inline bool merkle_verify(const Digest& commit, const std::vector<Dims>& dims, size_t index,
                                 const std::vector<std::vector<uint32_t>>& opened, const std::vector<Digest>& proof) {
    if (dims.size() != opened.size() || dims.empty()) return false;
    for (size_t i = 0; i < dims.size(); i++) if (opened[i].size() != dims[i].width) return false;
    std::vector<size_t> order(dims.size());
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return dims[a].height > dims[b].height; });
    size_t pos = 0;
    size_t cur = 1ull << log2_ceil(dims[order[0]].height);
    if (proof.size() != (size_t)log2_ceil(cur)) return false;
    auto hash_group = [&](size_t padded) {
        std::vector<const uint32_t*> sl;
        std::vector<size_t> ln;
        while (pos < order.size() && (1ull << log2_ceil(dims[order[pos]].height)) == padded) {
            sl.push_back(opened[order[pos]].data()); ln.push_back(opened[order[pos]].size()); pos++;
        }
        return p16_hash(sl, ln);
    };
    Digest root = hash_group(cur);
    for (const Digest& sib : proof) {
        root = (index & 1) ? p16_compress(sib, root) : p16_compress(root, sib);
        index >>= 1;
        cur >>= 1;
        if (pos < order.size() && (1ull << log2_ceil(dims[order[pos]].height)) == cur) root = p16_compress(root, hash_group(cur));
    }
    return pos == order.size() && root == commit;
}

}  // namespace orc

#include "../../oracle/oracle_api.cc"

extern "C" {

// The round constants (canonical) of the permutation the trees hash with; the MDS is CosetMds<_, 16>.
void orc_mmcs_set_round_constants(const uint32_t* rc480) {
    std::memcpy(orc::g_mmcs_perm.rc, rc480, sizeof orc::g_mmcs_perm.rc);
    orc::g_mmcs_perm.set_default_mds();
}
// The opening of leaf `index` of the tree over the matrices as given (no LDE): the opened rows concatenated in the caller's
// order into rows_out, the sibling digests (leaf level first) into path_out; returns the path length.
uint32_t orc_merkle_open(uint32_t n, const uint32_t* const* mats, const uint64_t* heights, const uint64_t* widths, uint64_t index,
                         uint32_t* rows_out, uint32_t* path_out) {
    std::vector<orc::Matrix> ms;
    for (uint32_t i = 0; i < n; i++) ms.emplace_back(std::vector<uint32_t>(mats[i], mats[i] + heights[i] * widths[i]), widths[i]);
    const orc::MerkleTree t = orc::merkle_commit(std::move(ms));
    const orc::BatchOpening o = orc::merkle_open(t, (size_t)index);
    for (auto& r : o.opened_values) { std::memcpy(rows_out, r.data(), r.size() * 4); rows_out += r.size(); }
    for (size_t i = 0; i < o.opening_proof.size(); i++) std::memcpy(path_out + 8 * i, o.opening_proof[i].data(), 32);
    return (uint32_t)o.opening_proof.size();
}

}  // extern "C"
