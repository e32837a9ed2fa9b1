// Machine::verify for proofs in the reference's wire format — the acceptance side of the boundary.
// Follows verify() (derive/src/lib.rs:492-650; hand copy basic/src/lib.rs:677-840):
//   re-commit the preprocessed traces (device, same kernels as the prover) -> replay the transcript ->
//   TwoAdicFriPcs::verify_multi_batches + p3-fri verify_query [P3-UNVERIFIED; SURVEY App. A items 14, 15]
//   -> per-chip verify_constraints (verify.cu) -> the cumulative sums of all chips add to zero.
// Everything except the preprocessed commit is host arithmetic on a ~2 MB proof (40 queries x ~25 Merkle
// paths); it exists so that a caller of this library can check what it produced without the Rust
// verifier, and so that the tests can cross-check prover and verifier against the oracle in both directions.
#include "../ctx.h"
#include "../verify.h"
#include "challenger.h"
#include "fri_config.h"
#include "proof.h"
#include <cstring>
#include <string>

using bb::E5;

namespace {

constexpr int MAX_LOG_DEGREE = 26;

// ---- Keccak-256 on the host (original 0x01 padding: p3-keccak wraps tiny-keccak's Keccak::v256) -------
const uint64_t RC[24] = {0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull, 0x000000000000808bull,
                         0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008aull, 0x0000000000000088ull,
                         0x0000000080008009ull, 0x000000008000000aull, 0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull,
                         0x8000000000008003ull, 0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull,
                         0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};
inline uint64_t rotl(uint64_t x, int n) { return n ? (x << n) | (x >> (64 - n)) : x; }
void keccak_f(uint64_t a[25]) {
    for (int round = 0; round < 24; round++) {
        uint64_t c[5], d[5], b[25];
        for (int x = 0; x < 5; x++) c[x] = a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20];
        for (int x = 0; x < 5; x++) d[x] = c[(x + 4) % 5] ^ rotl(c[(x + 1) % 5], 1);
        for (int i = 0; i < 25; i++) a[i] ^= d[i % 5];
        // rho + pi walk: lane (x, y) moves to (y, 2x + 3y) with rotation (t+1)(t+2)/2
        int x = 1, y = 0;
        b[0] = a[0];
        for (int t = 0; t < 24; t++) {
            const int nx = y, ny = (2 * x + 3 * y) % 5;
            b[nx + 5 * ny] = rotl(a[x + 5 * y], ((t + 1) * (t + 2) / 2) % 64);
            x = nx; y = ny;
        }
        for (int yy = 0; yy < 25; yy += 5)
            for (int xx = 0; xx < 5; xx++) a[yy + xx] = b[yy + xx] ^ (~b[yy + (xx + 1) % 5] & b[yy + (xx + 2) % 5]);
        a[0] ^= RC[round];
    }
}
// SerializingHasher32<Keccak256Hash>: little-endian canonical words in, 32 bytes out -> 8 words, each reduced mod p
Digest hash_canonical_words(const std::vector<uint32_t>& w) {
    uint64_t st[25] = {0};
    const size_t rate_words = 34;   // 136 bytes
    size_t i = 0;
    while (w.size() - i >= rate_words) {
        for (size_t k = 0; k < 17; k++) st[k] ^= (uint64_t)w[i + 2 * k] | ((uint64_t)w[i + 2 * k + 1] << 32);
        keccak_f(st);
        i += rate_words;
    }
    uint8_t block[136] = {0};
    size_t rem = w.size() - i;
    for (size_t k = 0; k < rem; k++) for (int b = 0; b < 4; b++) block[4 * k + b] = (uint8_t)(w[i + k] >> (8 * b));
    block[4 * rem] ^= 0x01;
    block[135] ^= 0x80;
    for (size_t k = 0; k < 17; k++) { uint64_t v = 0; for (int b = 7; b >= 0; b--) v = (v << 8) | block[8 * k + b]; st[k] ^= v; }
    keccak_f(st);
    Digest d;
    for (int k = 0; k < 4; k++) { d[2 * k] = (uint32_t)st[k] % bb::P; d[2 * k + 1] = (uint32_t)(st[k] >> 32) % bb::P; }
    return d;
}
Digest compress2(const Digest& l, const Digest& r) {
    std::vector<uint32_t> w(16);
    std::memcpy(w.data(), l.data(), 32); std::memcpy(w.data() + 8, r.data(), 32);
    return hash_canonical_words(w);
}

// The Poseidon-16 MMCS (VGPU_MERKLE_POSEIDON16) on the challenger's permutation.  PaddingFreeSponge<Perm16, 16, 8, 8>: state zero,
// each chunk of 8 words overwrites state[0 .. len) and is followed by a permutation, digest = state[0 .. 8).
Digest p16_hash(const vgh::Poseidon16& perm, const std::vector<uint32_t>& w) {
    uint32_t s[16] = {0};
    for (size_t i = 0; i < w.size(); i += 8) {
        for (size_t k = 0; k < 8 && i + k < w.size(); k++) s[k] = bb::to_monty(w[i + k]);
        perm.permute(s);
    }
    Digest d;
    for (int k = 0; k < 8; k++) d[k] = bb::from_monty(s[k]);
    return d;
}
// TruncatedPermutation<Perm16, 2, 8, 16>: permute(l || r)[0 .. 8)
Digest p16_compress(const vgh::Poseidon16& perm, const Digest& l, const Digest& r) {
    uint32_t s[16];
    for (int k = 0; k < 8; k++) { s[k] = bb::to_monty(l[k]); s[8 + k] = bb::to_monty(r[k]); }
    perm.permute(s);
    Digest d;
    for (int k = 0; k < 8; k++) d[k] = bb::from_monty(s[k]);
    return d;
}

// The context's MMCS: Keccak-256 when p16 is null, else Poseidon-16 over *p16.  Digests and words are canonical.
struct Mmcs {
    const vgh::Poseidon16* p16 = nullptr;
    Digest hash(const std::vector<uint32_t>& w) const { return p16 ? p16_hash(*p16, w) : hash_canonical_words(w); }
    Digest compress(const Digest& l, const Digest& r) const { return p16 ? p16_compress(*p16, l, r) : compress2(l, r); }
};

int log2_ceil(uint64_t n) { int l = 0; while ((1ull << l) < n) l++; return l; }

// FieldMerkleTreeMmcs::verify_batch [P3-UNVERIFIED; SURVEY App. A item 8]: matrices sorted by height (stable, tallest
// first); rows of equal padded height are hashed together; a shorter group is injected when the running height reaches it.
struct Dim { uint64_t w, h; };
bool merkle_verify_batch(const Mmcs& mmcs, const Digest& commit, const std::vector<Dim>& dims, uint64_t index,
                         const std::vector<std::vector<uint32_t>>& opened_canonical, const std::vector<Digest>& path) {
    if (dims.empty() || dims.size() != opened_canonical.size()) return false;
    std::vector<size_t> order;
    for (size_t i = 0; i < dims.size(); i++) { if (opened_canonical[i].size() != dims[i].w) return false; order.push_back(i); }
    for (size_t i = 1; i < order.size(); i++)   // stable insertion sort, descending height
        for (size_t j = i; j > 0 && dims[order[j - 1]].h < dims[order[j]].h; j--) std::swap(order[j - 1], order[j]);
    size_t pos = 0;
    int level = log2_ceil(dims[order[0]].h);
    if (path.size() != (size_t)level) return false;
    auto group = [&](int lvl) {
        std::vector<uint32_t> cat;
        while (pos < order.size() && log2_ceil(dims[order[pos]].h) == lvl) { auto& r = opened_canonical[order[pos]]; cat.insert(cat.end(), r.begin(), r.end()); pos++; }
        return mmcs.hash(cat);
    };
    Digest node = group(level);
    for (const Digest& sib : path) {
        node = (index & 1) ? mmcs.compress(sib, node) : mmcs.compress(node, sib);
        index >>= 1; level--;
        if (pos < order.size() && log2_ceil(dims[order[pos]].h) == level) node = mmcs.compress(node, group(level));
    }
    return pos == order.size() && node == commit;
}

struct RoundV { Digest commit; std::vector<Dim> dims; std::vector<std::vector<E5>> points; std::vector<std::vector<const std::vector<E5>*>> values; };

// TwoAdicFriPcs::verify_multi_batches + p3-fri verifier; 0 = accept, otherwise the verdict code of include/valida_b200.h
int32_t verify_openings(const Mmcs& mmcs, const std::vector<RoundV>& rounds, const vgh::PcsProof& pf, vgh::Challenger& ch) {
    const E5 alpha = ch.sample_ext();
    std::vector<E5> betas;
    for (const Digest& c : pf.commit_phase_commits) { ch.observe_digest_canonical(c.data()); betas.push_back(ch.sample_ext()); }
    if (pf.query_proofs.size() != (size_t)NUM_QUERIES || pf.query_openings.size() != (size_t)NUM_QUERIES) return VGPU_REJECT_SHAPE;
    if (!ch.check_witness(POW_BITS, pf.pow_witness)) return VGPU_REJECT_POW;
    const int log_max_height = (int)pf.commit_phase_commits.size() + LOG_BLOWUP;
    if (log_max_height > MAX_LOG_DEGREE + LOG_BLOWUP) return VGPU_REJECT_SHAPE;
    for (auto& rd : rounds)
        for (auto& d : rd.dims) if (log2_ceil(d.h) + LOG_BLOWUP > log_max_height) return VGPU_REJECT_SHAPE;
    std::vector<uint32_t> indices;
    for (int q = 0; q < NUM_QUERIES; q++) indices.push_back(ch.sample_bits(log_max_height));
    const uint32_t gen = bb::to_monty(bb::GEN_CANON);
    for (int q = 0; q < NUM_QUERIES; q++) {
        uint64_t index = indices[q];
        E5 ro[32], apw[32];
        for (int i = 0; i < 32; i++) { ro[i] = bb::e5_zero(); apw[i] = bb::e5_one(); }
        if (pf.query_openings[q].size() != rounds.size()) return VGPU_REJECT_SHAPE;
        for (size_t r = 0; r < rounds.size(); r++) {
            const RoundV& rd = rounds[r];
            const vgh::BatchOpening& bo = pf.query_openings[q][r];
            if (bo.opened_values.size() != rd.dims.size()) return VGPU_REJECT_SHAPE;
            std::vector<Dim> lde_dims;
            uint64_t max_h = 0;
            for (auto& d : rd.dims) { lde_dims.push_back({d.w, d.h << LOG_BLOWUP}); max_h = std::max(max_h, d.h << LOG_BLOWUP); }
            std::vector<std::vector<uint32_t>> canon_rows;
            for (auto& row : bo.opened_values) { std::vector<uint32_t> c; for (uint32_t x : row) c.push_back(bb::from_monty(x)); canon_rows.push_back(std::move(c)); }
            const uint64_t batch_index = index >> (log_max_height - log2_ceil(max_h));
            if (!merkle_verify_batch(mmcs, rd.commit, lde_dims, batch_index, canon_rows, bo.opening_proof)) return VGPU_REJECT_INPUT_MERKLE;
            for (size_t mi = 0; mi < rd.dims.size(); mi++) {
                const int lh = log2_ceil(rd.dims[mi].h) + LOG_BLOWUP;
                const uint32_t rev = bb::reverse_bits((uint32_t)(index >> (log_max_height - lh)), lh);
                const uint32_t x = bb::mul(gen, bb::pow(bb::two_adic_generator_monty(lh), rev));
                for (size_t pi = 0; pi < rd.points[mi].size(); pi++) {
                    const std::vector<E5>& at_z = *rd.values[mi][pi];
                    if (at_z.size() != bo.opened_values[mi].size()) return VGPU_REJECT_SHAPE;
                    const E5 den = bb::e5_add_base(bb::e5_neg(rd.points[mi][pi]), x);   // x - z
                    if (bb::e5_is_zero(den)) return VGPU_REJECT_SHAPE;
                    const E5 dinv = bb::e5_inv(den);
                    for (size_t c = 0; c < at_z.size(); c++) {
                        const E5 quotient = bb::e5_mul(bb::e5_add_base(bb::e5_neg(at_z[c]), bo.opened_values[mi][c]), dinv);   // (p(x) - p(z)) / (x - z)
                        ro[lh] = bb::e5_add(ro[lh], bb::e5_mul(apw[lh], quotient));
                        apw[lh] = bb::e5_mul(apw[lh], alpha);
                    }
                }
            }
        }
        // p3-fri verify_query
        const std::vector<vgh::CommitPhaseStep>& steps = pf.query_proofs[q];
        if (steps.size() != pf.commit_phase_commits.size()) return VGPU_REJECT_SHAPE;
        E5 folded = bb::e5_zero();
        uint32_t x = bb::pow(bb::two_adic_generator_monty(log_max_height), bb::reverse_bits((uint32_t)index, log_max_height));
        const uint32_t minus_one = bb::two_adic_generator_monty(1);
        size_t si = 0;
        for (int lfh = log_max_height - 1; lfh >= LOG_BLOWUP; lfh--, si++) {
            folded = bb::e5_add(folded, ro[lfh + 1]);
            const uint64_t sib = (index ^ 1) & 1, pair = index >> 1;
            E5 evals[2] = {folded, folded};
            evals[sib] = steps[si].sibling_value;
            std::vector<uint32_t> row(10);
            for (int e = 0; e < 2; e++) for (int l = 0; l < 5; l++) row[5 * e + l] = bb::from_monty(evals[e].c[l]);
            if (!merkle_verify_batch(mmcs, pf.commit_phase_commits[si], {{10, 1ull << lfh}}, pair, {row}, steps[si].opening_proof)) return VGPU_REJECT_FRI_MERKLE;
            uint32_t xs[2] = {x, x};
            xs[sib] = bb::mul(xs[sib], minus_one);
            // line through (xs[0], evals[0]), (xs[1], evals[1]) evaluated at beta; xs[1] - xs[0] = -2 xs[0]
            const uint32_t slope_den = bb::inv(bb::sub(xs[1], xs[0]));
            const E5 slope = bb::e5_mul_base(bb::e5_sub(evals[1], evals[0]), slope_den);
            folded = bb::e5_add(evals[0], bb::e5_mul(bb::e5_sub_base(betas[si], xs[0]), slope));
            index = pair;
            x = bb::sqr(x);
        }
        // The prover's last fold also adds the reduced openings of the height-2 LDEs (traces of ONE row: constant polynomials,
        // for which (p(x) - p(z)) / (x - z) is exactly 0).  The loop above never reaches them, so they are checked here: without
        // this the opened values of every one-row chip — and with them its cumulative sum — would be bound by nothing.
        if (!bb::e5_is_zero(ro[LOG_BLOWUP])) return VGPU_REJECT_FRI_FINAL;
        for (int l = 0; l < 5; l++) if (folded.c[l] != pf.final_poly.c[l]) return VGPU_REJECT_FRI_FINAL;
    }
    return VGPU_ACCEPT;
}

}  // namespace

extern "C" int32_t vgpu_verify(vgpu_ctx* ctx, const uint8_t* proof, uint64_t proof_len, const vgpu_matrix prep[2], int32_t repr, int32_t* verdict) {
    if (!ctx) return -1;
    if (!proof || !prep || !verdict) VG_FAIL(ctx, "verify: null argument");
    if (!ctx->challenger_set) VG_FAIL(ctx, "verify: vgpu_set_challenger has not been called");
    VG_TRY(vg_enter(ctx));
    *verdict = VGPU_REJECT_MALFORMED;
    vgh::MachineProof pf;
    if (!vgh::decode(proof, proof_len, &pf)) return 0;
    const std::vector<vgh::ChipProof>& chips = pf.chip_proofs;
    if (chips.size() != (size_t)VGPU_NUM_CHIPS) { *verdict = VGPU_REJECT_SHAPE; return 0; }
    for (auto& c : chips) if (c.log_degree > (uint32_t)MAX_LOG_DEGREE || c.preprocessed_local.size() || c.preprocessed_next.size()) { *verdict = VGPU_REJECT_SHAPE; return 0; }
    // the two chips with preprocessed columns have the height of those columns (program ROM, range table): a proof may not
    // shrink them (an all-one-row proof has no FRI layers at all)
    if ((1ull << chips[1].log_degree) != prep[0].height || (1ull << chips[12].log_degree) != prep[1].height) { *verdict = VGPU_REJECT_SHAPE; return 0; }

    vgh::Poseidon16 perm;
    perm.set(ctx->poseidon_rc, ctx->poseidon_has_mds ? ctx->poseidon_mds : nullptr);
    vgh::Challenger ch;
    ch.perm = &perm;
    {   // preprocessed commitment, recomputed (derive/src/lib.rs:505-517)
        uint32_t digest[8];
        vgpu_prover_data* pd = nullptr;
        // a verifier checks alone: no collective here even when the context is a rank of a split prover
        const bool was_sharding = ctx->sharding;
        ctx->sharding = false;
        const int32_t rc = vgpu_commit_batches_host(ctx, prep, 2, repr, nullptr, digest, &pd);
        const VgPd commitment(pd);               // only its root is needed
        ctx->sharding = was_sharding;
        if (rc) return rc;
        ch.observe_digest_canonical(digest);
    }
    ch.observe_digest_canonical(pf.main_trace.data());
    uint32_t perm_challenges[15];
    for (int i = 0; i < 3; i++) { E5 e = ch.sample_ext(); for (int l = 0; l < 5; l++) perm_challenges[5 * i + l] = bb::from_monty(e.c[l]); }
    ch.observe_digest_canonical(pf.perm_trace.data());
    const E5 alpha = ch.sample_ext();
    ch.observe_digest_canonical(pf.quotient_chunks.data());
    const E5 zeta = ch.sample_ext();

    std::vector<RoundV> rounds(3);
    rounds[0].commit = pf.main_trace; rounds[1].commit = pf.perm_trace; rounds[2].commit = pf.quotient_chunks;
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        const vgpu_chip_desc* chip = vgpu_basic_machine_chip(i);
        const vgh::ChipProof& c = chips[i];
        const uint64_t h = 1ull << c.log_degree;
        const E5 zg = bb::e5_mul_base(zeta, bb::two_adic_generator_monty((int)c.log_degree));
        rounds[0].dims.push_back({chip->width, h});
        rounds[1].dims.push_back({5ull * (chip->n_interactions + 1), h});
        rounds[2].dims.push_back({10, h});
        rounds[0].points.push_back({zeta, zg}); rounds[0].values.push_back({&c.trace_local, &c.trace_next});
        rounds[1].points.push_back({zeta, zg}); rounds[1].values.push_back({&c.permutation_local, &c.permutation_next});
        rounds[2].points.push_back({bb::e5_sqr(zeta)}); rounds[2].values.push_back({&c.quotient_chunks});
    }
    Mmcs mmcs;
    if (ctx->merkle_hash == VGPU_MERKLE_POSEIDON16) mmcs.p16 = &perm;
    int32_t v = verify_openings(mmcs, rounds, pf.opening_proof, ch);
    if (v != VGPU_ACCEPT) { *verdict = v; return 0; }
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        bool ok = false;
        VG_TRY(vg_verify_chip_constraints(ctx, vgpu_basic_machine_chip(i), chips[i], zeta, alpha, perm_challenges, &ok));
        if (!ok) { *verdict = VGPU_REJECT_CONSTRAINTS_CHIP0 - i; return 0; }
    }
    E5 sum = bb::e5_zero();
    for (auto& c : chips) sum = bb::e5_add(sum, c.cumulative_sum);
    if (!bb::e5_is_zero(sum)) { *verdict = VGPU_REJECT_CUMULATIVE_SUM; return 0; }
    *verdict = VGPU_ACCEPT;
    return 0;
}
