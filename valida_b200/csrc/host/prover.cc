// Machine::prove on the device — orchestration, transcript and proof assembly.
// Mirrors, step for step, the reference's prove() (derive/src/lib.rs:275-446; hand copy
// basic/src/lib.rs:147-675) and TwoAdicFriPcs::open_multi_batches / p3-fri prove
// [P3-UNVERIFIED; SURVEY App. A items 14, 15]; every observe/sample occurs in the reference's order.
// Heavy steps are the CUDA kernels of ntt.cu / merkle.cu / perm.cu / quotient.cu / open.cu; this file
// holds no field loops over trace-sized data.
#include "../ctx.h"
#include "../merkle.h"
#include "../open.h"
#include "../devchip.h"
#include "challenger.h"
#include "fri_config.h"
#include "proof.h"
#include <algorithm>
#include <chrono>
#include <cstring>
#include <map>
#include <memory>

using bb::E5;

namespace {

struct OpenRound { const vgpu_prover_data* pd; std::vector<std::vector<E5>> points; };

// Device time of a phase: an event pair on the context's stream, read back by vgpu_last_prove_phases — no host
// synchronisation inside the proof.
struct Phase {
    vgpu_ctx* ctx;
    Phase(vgpu_ctx* c, const char* n) : ctx(c) {
        vgpu_ctx::PhaseMark m{n, nullptr, nullptr};
        vg_take_event(c, &m.a);
        vg_take_event(c, &m.b);
        cudaEventRecord(m.a, c->stream);
        c->phase_marks.push_back(m);
        idx = c->phase_marks.size() - 1;
    }
    ~Phase() { cudaEventRecord(ctx->phase_marks[idx].b, ctx->stream); }
    size_t idx;
};
// host-side stretches between device work (pointer lists, CBOR): wall-clock, reported beside the device phases
struct HostPhase {
    vgpu_ctx* ctx; const char* name; std::chrono::steady_clock::time_point t0;
    HostPhase(vgpu_ctx* c, const char* n) : ctx(c), name(n), t0(std::chrono::steady_clock::now()) {}
    ~HostPhase() { ctx->host_phases.push_back({name, std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count()}); }
};
void phases_reset(vgpu_ctx* ctx) {
    for (auto& m : ctx->phase_marks) { ctx->event_pool.push_back(m.a); ctx->event_pool.push_back(m.b); }
    ctx->phase_marks.clear();
    ctx->phases.clear();
    ctx->host_phases.clear();
}

// An ext5 vector over the rows of one LDE height (reduced openings, inverse denominators, FRI layers): limb-major.
// Split proof: a vector of a height whose matrices are row shards holds this rank's run [begin, begin + count) only.
struct RowVec {
    VgBuf d;
    uint64_t n = 0, begin = 0, count = 0;      // whole length; stored run (limb stride = count)
    uint32_t* data() const { return d.as<uint32_t>(); }
    bool shard() const { return count != n; }
    const uint32_t* at(const vgpu_ctx* ctx, int limb, uint64_t i) const {   // null: another rank reports this element (see VgTree::node)
        if (!shard()) return vg_reports_replicated(ctx) ? data() + (uint64_t)limb * count + i : nullptr;
        return i >= begin && i < begin + count ? data() + (uint64_t)limb * count + (i - begin) : nullptr;
    }
};
int32_t rowvec_alloc(vgpu_ctx* ctx, uint64_t n, RowVec* v) {
    const VgRun run = vg_row_run(ctx, n);
    v->n = n; v->begin = run.begin; v->count = run.count;
    v->d = VgBuf(ctx);
    return v->d.alloc(5 * v->count * 4);
}

struct FriLayer { RowVec values; VgTree tree; };

struct PointKey {
    uint32_t log_H; uint32_t c[5];
    bool operator<(const PointKey& o) const { if (log_H != o.log_H) return log_H < o.log_H; return std::memcmp(c, o.c, 20) < 0; }
};

int log2u(uint64_t n) { int l = 0; while ((1ull << l) < n) l++; return l; }

int32_t open_multi_batches(vgpu_ctx* ctx, const std::vector<OpenRound>& rounds, vgh::Challenger& ch, vgh::OpenedValues* values, vgh::PcsProof* out) {
    const E5 alpha = ch.sample_ext();
    // alpha^c table (host; the reduced-opening kernel takes its powers through the kernel parameters)
    uint32_t max_w = 1;
    for (auto& r : rounds) for (auto* m : r.pd->ldes) max_w = std::max<uint32_t>(max_w, (uint32_t)m->gw);
    std::vector<E5> apow(max_w + 1);
    { E5 a = bb::e5_one(); for (uint32_t c = 0; c <= max_w; c++) { apow[c] = a; a = bb::e5_mul(a, alpha); } }

    std::map<PointKey, VgBuf> invden;           // (height, point) -> 1/(x - z) over this rank's rows of the coset
    RowVec ro[32];                              // reduced openings by log height
    VgBuf d_sums(ctx);
    RowVec current;                             // the FRI layer being folded
    std::vector<FriLayer> layers;
    VgBuf paths(ctx);                           // the rebuilt lower levels of the query paths (vg_tree_paths)
    uint64_t num_reduced[32] = {0};
    // Pass 1 — enqueue, for every matrix, the inverse denominators of its points and the column sums behind p_c(z_q); nothing
    // here waits for the device.  One copy brings the sums of all matrices back.
    struct Job { const vgpu_dmat* lde; uint32_t log_H, w; const std::vector<E5>* pts; const uint32_t* dens[2]; size_t sums_at; };
    std::vector<Job> jobs;
    size_t sums_words = 0;
    for (const OpenRound& rd : rounds)
        for (size_t mi = 0; mi < rd.pd->ldes.size(); mi++) {
            Job j{};
            j.lde = rd.pd->ldes[mi]; j.log_H = (uint32_t)log2u(j.lde->gh); j.w = (uint32_t)j.lde->gw; j.pts = &rd.points[mi];
            if (j.pts->empty() || j.pts->size() > 2) VG_FAIL(ctx, "open: 1 or 2 points per matrix are supported");
            if ((j.lde->dist == VG_ROWS) != vg_row_run(ctx, j.lde->gh).split) VG_FAIL(ctx, "open: a committed matrix is not distributed as its height demands");
            j.sums_at = sums_words; sums_words += vg_eval_columns_words(j.w);
            jobs.push_back(j);
        }
    VG_TRY(d_sums.alloc(sums_words * 4));
    for (Job& j : jobs) {
        RowVec& R = ro[j.log_H];
        if (!R.d) {
            VG_TRY(rowvec_alloc(ctx, j.lde->gh, &R));
            VG_CUDA(ctx, cudaMemsetAsync(R.data(), 0, 5 * R.count * 4, ctx->stream));
        }
        for (size_t q = 0; q < j.pts->size(); q++) {
            PointKey key; key.log_H = j.log_H; std::memcpy(key.c, (*j.pts)[q].c, 20);
            auto it = invden.find(key);
            if (it == invden.end()) {
                it = invden.emplace(key, VgBuf(ctx)).first;
                VG_TRY(it->second.alloc(5 * R.count * 4));
                VG_TRY(vg_inverse_denominators(ctx, j.log_H, (*j.pts)[q], R.begin, R.count, it->second.as<uint32_t>()));
            }
            j.dens[q] = it->second.as<uint32_t>();
        }
        VG_TRY(vg_eval_columns_enqueue(ctx, j.lde, (uint32_t)j.pts->size(), j.dens, R.count, d_sums.as<uint32_t>() + j.sums_at));
    }
    std::vector<uint32_t> sums(sums_words);
    VG_CUDA(ctx, cudaMemcpyAsync(sums.data(), d_sums.p, sums_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // Pass 2 — opened values on the host, then the reduced openings of every matrix (again without waiting)
    values->clear();
    {
        size_t ji = 0;
        std::vector<E5> apow_off(max_w);
        for (const OpenRound& rd : rounds) {
            values->emplace_back();
            for (size_t mi = 0; mi < rd.pd->ldes.size(); mi++, ji++) {
                const Job& j = jobs[ji];
                const uint32_t w = j.w, np = (uint32_t)j.pts->size();
                std::vector<E5> ys;
                vg_eval_columns_finish(sums.data() + j.sums_at, j.lde->gh, w, np, j.pts->data(), &ys, j.lde->dist == VG_ROWS ? vg_eval_columns_first_coset(w) : w);
                E5 sum_y[2];
                values->back().emplace_back();
                for (uint32_t q = 0; q < np; q++) {
                    E5 s = bb::e5_zero();
                    for (uint32_t c = 0; c < w; c++) s = bb::e5_add(s, bb::e5_mul(apow[c], ys[q * w + c]));
                    sum_y[q] = s;
                    values->back().back().emplace_back(ys.begin() + q * w, ys.begin() + (q + 1) * w);
                }
                // point q's terms carry alpha^(num_reduced + q * w): the power table is shifted by the first offset
                const E5 a_off = bb::e5_pow(alpha, num_reduced[j.log_H]);
                num_reduced[j.log_H] += (uint64_t)w * np;
                for (uint32_t c = 0; c < w; c++) apow_off[c] = bb::e5_mul(a_off, apow[c]);
                VG_TRY(vg_reduced_opening_accumulate(ctx, j.lde, apow_off.data(), apow[w], np, j.dens, ro[j.log_H].count, sum_y, ro[j.log_H].data()));
            }
        }
    }
    invden.clear();
    d_sums.reset();

    // ---- p3-fri prove: commit phase --------------------------------------------------------------
    // Split proof: while a layer is long enough it stays in row shards — a fold pairs neighbours (2i, 2i+1), so a rank folds its
    // own run, hashes its own leaves and sub-tree, and only the sub-roots meet; the first layer too short to split is
    // all-gathered once and folded by every rank from there on.
    int log_max = 31;
    while (log_max >= 0 && !ro[log_max].d) log_max--;
    if (log_max < LOG_BLOWUP) VG_FAIL(ctx, "open: nothing to open");
    current = std::move(ro[log_max]);
    for (int lfh = log_max - 1; lfh >= LOG_BLOWUP; lfh--) {
        layers.emplace_back();
        FriLayer& L = layers.back();
        L.values = std::move(current);
        const RowVec& cur = L.values;
        const uint64_t npairs = cur.n / 2;
        Digest root;
        VG_TRY(vg_fri_layer_commit(ctx, cur.data(), cur.count, npairs, cur.shard(), &L.tree, root.data()));
        ch.observe_digest_canonical(root.data());
        out->commit_phase_commits.push_back(root);
        E5 beta = ch.sample_ext();
        RowVec next;
        VG_TRY(rowvec_alloc(ctx, npairs, &next));
        const RowVec& add = ro[lfh];
        if (add.d && add.shard() != next.shard()) VG_FAIL(ctx, "open: reduced openings and FRI layer of height 2^%d are distributed differently", lfh);
        const uint64_t i0 = cur.shard() ? cur.begin / 2 : 0, cnt = cur.count / 2;      // outputs folded here
        VG_TRY(vg_fri_fold(ctx, cur.data(), cur.count, cur.n, i0, cnt, beta, add.d ? add.data() - add.begin : nullptr, add.count, next.data() - next.begin, next.count));
        if (cur.shard() && !next.shard()) {   // every rank folded its run into the whole-length buffer: complete it
            VG_TRY(vg_comm_group_begin(ctx));
            for (int l = 0; l < 5; l++) VG_TRY(vg_comm_allgather_runs(ctx, next.data() + (uint64_t)l * next.count, next.n, 1));
            VG_TRY(vg_comm_group_end(ctx));
        }
        current = std::move(next);
        ro[lfh] = RowVec();
    }
    {
        const RowVec& cur = current;
        if (cur.shard()) VG_FAIL(ctx, "open: the final FRI layer is still distributed");
        std::vector<uint32_t> fin(5 * cur.n);
        VG_CUDA(ctx, cudaMemcpyAsync(fin.data(), cur.data(), fin.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        E5 f0;
        for (int l = 0; l < 5; l++) f0.c[l] = fin[l * cur.n];
        for (uint64_t i = 1; i < cur.n; i++)
            for (int l = 0; l < 5; l++)
                if (fin[l * cur.n + i] != f0.c[l]) VG_FAIL(ctx, "FRI: final layer is not constant (the committed functions are not low degree)");
        out->final_poly = f0;
    }
    {
        HostPhase hp(ctx, "proof-of-work grind (device search + host check)");
        VG_TRY(vg_pow_grind(ctx, ch, POW_BITS, &out->pow_witness));
    }
    std::vector<uint64_t> indices;
    for (int q = 0; q < NUM_QUERIES; q++) indices.push_back(ch.sample_bits(log_max));

    // ---- query phase: one gather for every word the proof needs (split proof: every rank reports the words it holds) ------
    HostPhase hq(ctx, "host+device: query phase (pointer list, gather, answers)");
    // every query asks for the same NUMBER of words (its index only selects which): the 40 pointer lists, and later the 40 answers,
    // are filled by the host threads in parallel
    size_t per_query = 0;
    for (auto& L : layers) per_query += 5 + 8 * (L.tree.layer_ptr.size() - 1);
    for (const OpenRound& rd : rounds) { for (auto* m : rd.pd->ldes) per_query += m->w; per_query += 8 * (size_t)log2u(rd.pd->max_height); }
    const long nq = (long)indices.size();
    // the path levels below the kept tree layers: every tree's, of every query, rebuilt in one launch (merkle.h) — by the rank that
    // reports the leaf, as for the stored levels; tree t of query qi writes slot qi * trees + t
    std::vector<VgPathTree> trees;
    for (const FriLayer& L : layers) trees.push_back({&L.tree, nullptr, L.values.data() - L.values.begin, L.values.count});
    for (const OpenRound& rd : rounds) trees.push_back({&rd.pd->tree, rd.pd, nullptr, 0});
    auto leaf_of = [&](size_t t, uint64_t index) -> uint64_t {     // the leaf of tree t a query index opens
        if (t < layers.size()) return index >> (t + 1);
        return index >> (log_max - log2u(rounds[t - layers.size()].pd->max_height));
    };
    std::vector<VgPathReq> reqs;
    for (long qi = 0; qi < nq; qi++)
        for (size_t t = 0; t < trees.size(); t++) {
            const uint64_t leaf = leaf_of(t, indices[qi]);
            if (trees[t].tree->rebuilt() && trees[t].tree->reports(ctx, 0, leaf)) reqs.push_back({(uint32_t)t, (uint32_t)(qi * trees.size() + t), leaf});
        }
    VG_TRY(vg_tree_paths(ctx, trees, reqs, (size_t)nq * trees.size(), &paths));
    const uint32_t* path_words = paths.as<uint32_t>();
    std::vector<const uint32_t*> ptrs(per_query * (size_t)nq);
#pragma omp parallel for schedule(static) num_threads(8)
    for (long qi = 0; qi < nq; qi++) {
        const uint64_t index = indices[qi];
        const uint32_t** o = ptrs.data() + per_query * (size_t)qi;
        auto push_digest = [&](const uint32_t* d) { for (int k = 0; k < 8; k++) *o++ = d ? d + k : nullptr; };
        auto push_path = [&](size_t t) {     // the sibling digests of tree t's path, leaf level first
            const VgTree& tr = *trees[t].tree;
            const uint64_t leaf = leaf_of(t, index);
            const uint32_t* rebuilt = tr.reports(ctx, 0, leaf) ? path_words + ((size_t)qi * trees.size() + t) * VG_TREE_DROP * 8 : nullptr;
            for (size_t lvl = 0; lvl < tr.depth(); lvl++)
                push_digest(lvl < tr.rebuilt() ? (rebuilt ? rebuilt + lvl * 8 : nullptr) : tr.node(ctx, lvl, (leaf >> lvl) ^ 1));
        };
        for (size_t i = 0; i < layers.size(); i++) {
            const FriLayer& L = layers[i];
            uint64_t sib = (index >> i) ^ 1;
            for (int l = 0; l < 5; l++) *o++ = L.values.at(ctx, l, sib);
            push_path(i);
        }
        for (size_t r = 0; r < rounds.size(); r++) {
            const OpenRound& rd = rounds[r];
            int lg = log2u(rd.pd->max_height);
            uint64_t bidx = index >> (log_max - lg);
            for (auto* m : rd.pd->ldes) {
                const uint64_t row = bidx >> (lg - log2u(m->gh));
                for (uint64_t c = 0; c < m->w; c++) *o++ = vg_reported_word(ctx, m, row, c);
            }
            push_path(layers.size() + r);
        }
    }
    std::vector<uint32_t> words;
    VG_TRY(vg_gather_words(ctx, ptrs, &words));
    out->query_proofs.assign((size_t)nq, std::vector<vgh::CommitPhaseStep>());
    out->query_openings.assign((size_t)nq, std::vector<vgh::BatchOpening>());
#pragma omp parallel for schedule(static) num_threads(8)
    for (long qi = 0; qi < nq; qi++) {
        size_t pos = per_query * (size_t)qi;
        auto take_digest = [&]() { Digest d; for (int k = 0; k < 8; k++) d[k] = words[pos++]; return d; };
        std::vector<vgh::CommitPhaseStep>& steps = out->query_proofs[qi];
        steps.reserve(layers.size());
        for (size_t i = 0; i < layers.size(); i++) {
            vgh::CommitPhaseStep st;
            for (int l = 0; l < 5; l++) st.sibling_value.c[l] = words[pos++];
            const size_t depth = layers[i].tree.layer_ptr.size() - 1;
            st.opening_proof.reserve(depth);
            for (size_t lvl = 0; lvl < depth; lvl++) st.opening_proof.push_back(take_digest());
            steps.push_back(std::move(st));
        }
        for (const OpenRound& rd : rounds) {
            vgh::BatchOpening bo;
            int lg = log2u(rd.pd->max_height);
            for (auto* m : rd.pd->ldes) {
                bo.opened_values.emplace_back(words.begin() + pos, words.begin() + pos + m->w);
                pos += m->w;
            }
            for (int lvl = 0; lvl < lg; lvl++) bo.opening_proof.push_back(take_digest());
            out->query_openings[qi].push_back(std::move(bo));
        }
    }
    return 0;
}

// The encoded bytes in a buffer of their own, released by vgpu_free_bytes.
int32_t hand_off(vgpu_ctx* ctx, const std::vector<uint8_t>& bytes, uint8_t** out, uint64_t* out_len) {
    uint8_t* buf = (uint8_t*)std::malloc(bytes.size());
    if (!buf) VG_FAIL(ctx, "out of host memory");
    std::memcpy(buf, bytes.data(), bytes.size());
    *out = buf; *out_len = bytes.size();
    return 0;
}

vgh::Poseidon16* poseidon_of(vgpu_ctx* ctx) {
    if (!ctx->poseidon) {
        auto* p = new vgh::Poseidon16();
        p->set(ctx->poseidon_rc, ctx->poseidon_has_mds ? ctx->poseidon_mds : nullptr);
        ctx->poseidon = p;
    }
    return (vgh::Poseidon16*)ctx->poseidon;
}

// The debug mode checks whole traces; a split proof holds row shards, whose last row's "next" row lives on another rank.  Every rank
// refuses alike, before any collective.
int32_t debug_mode_allowed(vgpu_ctx* ctx) {
    if (ctx->debug_checks && vg_sharded(ctx))
        VG_FAIL(ctx, "prove: the debug checks run on whole traces only; turn them off or call vgpu_comm_set_sharding(ctx, 0)");
    return 0;
}

// check_constraints of every chip and check_cumulative_sums (machine/src/check_constraints.rs:87-93): an error naming every failure,
// or 0.
int32_t debug_verdict(vgpu_ctx* ctx, const vgpu_check_report rep[VGPU_NUM_CHIPS]) {
    static const char* NAMES[VGPU_NUM_CHIPS] = {"cpu", "program", "mem", "add", "sub", "mul", "div", "shift", "lt", "com", "bitwise", "output", "range", "static_data"};
    std::string msg;
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        if (rep[i].first_row < 0) continue;
        char b[160];
        snprintf(b, sizeof b, "chip %d (%s): constraint %u does not vanish on row %lld (%llu rows fail)", i, NAMES[i], rep[i].first_constraint,
                 (long long)rep[i].first_row, (unsigned long long)rep[i].failing_rows);
        msg += (msg.empty() ? "" : "; ") + std::string(b);
    }
    if (!vg_sums_cancel(rep)) msg += (msg.empty() ? "" : "; ") + std::string("cumulative sums do not cancel");
    if (msg.empty()) return 0;
    ctx->err = "prove: debug checks failed: " + msg;
    return -1;
}

}  // namespace

void vg_host_state_free(vgpu_ctx* ctx) {
    delete (vgh::Challenger*)ctx->challenger; ctx->challenger = nullptr;
    delete (vgh::Poseidon16*)ctx->poseidon; ctx->poseidon = nullptr;
}

extern "C" {

int32_t vgpu_challenger_reset(vgpu_ctx* ctx) {
    if (!ctx->challenger_set) VG_FAIL(ctx, "challenger: vgpu_set_challenger has not been called");
    delete (vgh::Poseidon16*)ctx->poseidon; ctx->poseidon = nullptr;
    delete (vgh::Challenger*)ctx->challenger;
    auto* c = new vgh::Challenger();
    c->perm = poseidon_of(ctx);
    ctx->challenger = c;
    return 0;
}
int32_t vgpu_challenger_observe(vgpu_ctx* ctx, const uint32_t* values, uint32_t n) {
    if (!ctx->challenger) VG_TRY(vgpu_challenger_reset(ctx));
    for (uint32_t i = 0; i < n; i++) ((vgh::Challenger*)ctx->challenger)->observe(bb::to_monty(values[i] % bb::P));
    return 0;
}
int32_t vgpu_challenger_sample_ext(vgpu_ctx* ctx, uint32_t out[5]) {
    if (!ctx->challenger) VG_TRY(vgpu_challenger_reset(ctx));
    E5 e = ((vgh::Challenger*)ctx->challenger)->sample_ext();
    for (int i = 0; i < 5; i++) out[i] = bb::from_monty(e.c[i]);
    return 0;
}

int32_t vgpu_open(vgpu_ctx* ctx, const vgpu_prover_data* const* rounds, uint32_t n_rounds, const uint32_t* n_points, const uint32_t* points,
                  uint8_t** out_cbor, uint64_t* out_len) {
    if (!rounds || !n_points || !points || !out_cbor || !out_len) VG_FAIL(ctx, "open: null argument");
    VG_TRY(vg_enter(ctx));
    if (!ctx->challenger) VG_TRY(vgpu_challenger_reset(ctx));
    std::vector<OpenRound> rds(n_rounds);
    size_t mi = 0, pi = 0;
    for (uint32_t r = 0; r < n_rounds; r++) {
        if (!rounds[r]) VG_FAIL(ctx, "open: round %u has no prover data", r);
        if (rounds[r]->tree.hash != ctx->merkle_hash) VG_FAIL(ctx, "open: round %u was committed with another Merkle hash than the context's", r);
        rds[r].pd = rounds[r];
        for (size_t m = 0; m < rounds[r]->ldes.size(); m++, mi++) {
            std::vector<E5> pts;
            for (uint32_t q = 0; q < n_points[mi]; q++, pi++) {
                E5 z; for (int l = 0; l < 5; l++) z.c[l] = bb::to_monty(points[5 * pi + l] % bb::P);
                pts.push_back(z);
            }
            rds[r].points.push_back(std::move(pts));
        }
    }
    vgh::OpenedValues values;
    vgh::PcsProof proof;
    VG_TRY(open_multi_batches(ctx, rds, *(vgh::Challenger*)ctx->challenger, &values, &proof));
    return hand_off(ctx, vgh::encode_opening(values, proof), out_cbor, out_len);
}

// owned_main: the caller's main traces when this call may release them once the permutation traces are built (their last
// use), or null.  vgpu_prove passes the device copies it made itself: on an 80 GB part that is what lets a 2^24-row trace
// (memory chip 2^26 rows, LDE 2^27) be proven on one GPU.
static int32_t prove_device(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                            vgpu_dmat* const* owned_main, uint8_t** proof_out, uint64_t* proof_len) {
    VG_TRY(debug_mode_allowed(ctx));
    const bool debug = ctx->debug_checks;
    if (!ctx->challenger_set) VG_FAIL(ctx, "prove: vgpu_set_challenger has not been called");
    if (!proof_out || !proof_len) VG_FAIL(ctx, "prove: null output");
    VG_TRY(vg_enter(ctx));
    if (!ctx->in_host_prove) phases_reset(ctx);
    const vgpu_chip_desc* chips[VGPU_NUM_CHIPS];
    int log_degrees[VGPU_NUM_CHIPS];
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        chips[i] = vgpu_basic_machine_chip(i);
        if (!main[i] || main[i]->gw != chips[i]->width) VG_FAIL(ctx, "prove: chip %d trace has width %llu, expected %u", i, main[i] ? (unsigned long long)main[i]->gw : 0ull, chips[i]->width);
        log_degrees[i] = log2u(main[i]->gh);
        if ((1ull << log_degrees[i]) != main[i]->gh) VG_FAIL(ctx, "prove: chip %d trace height is not a power of two", i);
    }
    if (vg_sharded(ctx)) {
        // Split proof: room in the symmetric heap for everything the three commits put there — the row shards of every tall
        // chip's main / permutation / quotient LDEs and the column buffers of the rows -> columns hand-over (counted as if never
        // released: first-fit then always finds a run) — reserved ONCE, before the first shard is live.
        std::vector<std::pair<uint64_t, uint64_t>> dm, dq, dc, dpre;
        for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
            const uint64_t h = main[i]->gh;
            dm.push_back({h, chips[i]->width}); dq.push_back({h, 5ull * (chips[i]->n_interactions + 1)}); dc.push_back({h, 10});
            if (chips[i]->preprocessed_width) dpre.push_back({h, chips[i]->preprocessed_width});
        }
        const size_t need = vg_commit_symm_need(ctx, dm) + vg_commit_symm_need(ctx, dq) + vg_commit_symm_need(ctx, dc) + vg_commit_symm_need(ctx, dpre);
        if (need) VG_TRY(vg_symm_reserve(ctx, need));
    }
    vgh::Challenger ch;
    { delete (vgh::Poseidon16*)ctx->poseidon; ctx->poseidon = nullptr; }
    ch.perm = poseidon_of(ctx);

    // a commit's prover data, owned here from the moment the commit hands it out
    auto commit = [&](const vgpu_dmat* const* mats, uint32_t n, const uint32_t* shifts, uint32_t digest_out[8], VgPd* pd) -> int32_t {
        vgpu_prover_data* p = nullptr;
        VG_TRY(vgpu_commit_batches(ctx, mats, n, shifts, digest_out, &p));
        pd->reset(p);
        return 0;
    };
    VgPd prep_pd, main_pd, perm_pd, quot_pd;
    uint32_t digest[8];
    {   // preprocessed commit (derive:299-311)
        Phase ph(ctx, "commit preprocessed");
        VG_TRY(commit(prep, 2, nullptr, digest, &prep_pd));
        ch.observe_digest_canonical(digest);
    }
    vgh::MachineProof mp;
    mp.chip_proofs.resize(VGPU_NUM_CHIPS);
    {   // main commit (313-332)
        Phase ph(ctx, "commit main");
        VG_TRY(commit(main, VGPU_NUM_CHIPS, nullptr, mp.main_trace.data(), &main_pd));
        ch.observe_digest_canonical(mp.main_trace.data());
    }
    uint32_t perm_challenges[15];
    for (int i = 0; i < 3; i++) { E5 e = ch.sample_ext(); for (int l = 0; l < 5; l++) perm_challenges[5 * i + l] = bb::from_monty(e.c[l]); }
    uint32_t cumsum[VGPU_NUM_CHIPS][5];
    {   // permutation traces (339-358)
        std::vector<VgMat> perms;
        {
            Phase ph(ctx, "permutation traces");
            // the cumulative sums of all chips come back with ONE copy (debug mode: with the check results of the 14 chips)
            VgMachineCheck mc(ctx, main, prep, perm_challenges, debug);
            VG_TRY(mc.alloc());
            perms.resize(VGPU_NUM_CHIPS);
            for (int i = 0; i < VGPU_NUM_CHIPS; i++) VG_TRY(mc.perm(i, &perms[i]));
            if (debug) {   // check_constraints (derive/src/lib.rs:246-253) while the main traces are still held
                Phase pc(ctx, "check constraints");
                for (int i = 0; i < VGPU_NUM_CHIPS; i++) VG_TRY(mc.sweep(i, perms[i].get()));
            }
            uint32_t sums[VGPU_NUM_CHIPS][5];
            vgpu_check_report rep[VGPU_NUM_CHIPS];
            VG_TRY(mc.finish(sums, rep));
            for (int i = 0; i < VGPU_NUM_CHIPS; i++)
                for (int l = 0; l < 5; l++) {
                    mp.chip_proofs[i].cumulative_sum.c[l] = sums[i][l];
                    cumsum[i][l] = rep[i].cumulative_sum[l];
                }
            if (debug) VG_TRY(debug_verdict(ctx, rep));
            // later work reuses the released blocks in stream order, i.e. after the permutation kernels that read them
            for (int i = 0; owned_main && i < VGPU_NUM_CHIPS; i++) {
                vgpu_dmat* m = owned_main[i];
                if (m->owns && !m->symm && !m->pend_stage) { vg_free(ctx, m->d); m->d = nullptr; }
            }
        }
        Phase ph(ctx, "commit permutation");
        VG_TRY(commit(vg_handles(perms).data(), VGPU_NUM_CHIPS, nullptr, mp.perm_trace.data(), &perm_pd));
        ch.observe_digest_canonical(mp.perm_trace.data());
    }
    E5 alpha = ch.sample_ext();
    uint32_t alpha_c[5];
    for (int l = 0; l < 5; l++) alpha_c[l] = bb::from_monty(alpha.c[l]);
    {   // quotients (246-270, 362-374)
        std::vector<VgMat> quots;
        {
            Phase ph(ctx, "quotient");
            int prep_idx = 0;
            for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
                const vgpu_dmat* plde = chips[i]->preprocessed_width ? prep_pd->ldes[prep_idx++] : nullptr;
                vgpu_dmat* q = nullptr;
                VG_TRY(vgpu_quotient(ctx, chips[i], (uint32_t)log_degrees[i], plde, main_pd->ldes[i], perm_pd->ldes[i], cumsum[i], perm_challenges, alpha_c, &q));
                quots.emplace_back(q);
            }
        }
        Phase ph(ctx, "commit quotient");
        uint32_t shifts[VGPU_NUM_CHIPS];
        for (int i = 0; i < VGPU_NUM_CHIPS; i++) shifts[i] = (uint32_t)(((uint64_t)bb::GEN_CANON * bb::GEN_CANON) % bb::P);   // coset_shift^(2^log_quotient_degree)
        VG_TRY(commit(vg_handles(quots).data(), VGPU_NUM_CHIPS, shifts, mp.quotient_chunks.data(), &quot_pd));
        ch.observe_digest_canonical(mp.quotient_chunks.data());
    }
    E5 zeta = ch.sample_ext();
    // openings (379-392): main & perm at [zeta, zeta*g_i], quotient at [zeta^2]; preprocessed is NOT opened
    std::vector<OpenRound> rounds(3);
    rounds[0].pd = main_pd.get(); rounds[1].pd = perm_pd.get(); rounds[2].pd = quot_pd.get();
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        E5 zg = bb::e5_mul_base(zeta, bb::two_adic_generator_monty(log_degrees[i]));
        rounds[0].points.push_back({zeta, zg});
        rounds[1].points.push_back({zeta, zg});
        rounds[2].points.push_back({bb::e5_sqr(zeta)});
    }
    vgh::OpenedValues values;
    {
        Phase ph(ctx, "open (evaluate + FRI)");
        VG_TRY(open_multi_batches(ctx, rounds, ch, &values, &mp.opening_proof));
    }
    HostPhase hc(ctx, "host: MachineProof -> CBOR");
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        vgh::ChipProof& c = mp.chip_proofs[i];
        c.log_degree = (uint32_t)log_degrees[i];
        c.trace_local = std::move(values[0][i][0]); c.trace_next = std::move(values[0][i][1]);
        c.permutation_local = std::move(values[1][i][0]); c.permutation_next = std::move(values[1][i][1]);
        c.quotient_chunks = std::move(values[2][i][0]);
    }
    return hand_off(ctx, vgh::encode(mp), proof_out, proof_len);
}

int32_t vgpu_prove_device(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                          uint8_t** proof_out, uint64_t* proof_len) {
    return prove_device(ctx, main, prep, nullptr, proof_out, proof_len);
}

int32_t vgpu_prove(vgpu_ctx* ctx, const vgpu_matrix main[VGPU_NUM_CHIPS], const vgpu_matrix prep[2], int32_t repr,
                   uint8_t** proof_out, uint64_t* proof_len) {
    // Host-buffer entry: the H2D copies run on a copy stream in the order the commits consume the traces (preprocessed,
    // then main traces tallest first — the Merkle tree hashes the tallest LDEs first and extends the shorter matrices
    // only when a tree layer of their height is reached), each transpose is deferred to the matrix's first use, so
    // copies of later matrices overlap the LDE / Keccak kernels of earlier ones.
    // Split proof: of a trace tall enough to be split a rank uploads ITS run of rows only (1 / comm_size of the bytes).
    VG_TRY(debug_mode_allowed(ctx));
    VG_TRY(vg_enter(ctx));
    std::vector<VgMat> dm(VGPU_NUM_CHIPS), dp(2);
    phases_reset(ctx);
    auto t0 = std::chrono::steady_clock::now();
    auto alloc_for = [&](const vgpu_matrix& hm, VgMat* out) {
        return vg_dmat_alloc_run(ctx, hm.height, hm.width, vg_trace_run(ctx, hm.height).split, false, out);
    };
    auto begin_upload = [&](const vgpu_matrix& hm, vgpu_dmat* m) { return vg_upload_begin(ctx, hm.data + m->row0 * hm.width, m->h, m->w, repr, m); };
    for (int i = 0; i < 2; i++) VG_TRY(alloc_for(prep[i], &dp[i]));
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) VG_TRY(alloc_for(main[i], &dm[i]));
    for (int i = 0; i < 2; i++) VG_TRY(begin_upload(prep[i], dp[i].get()));
    std::vector<int> order(VGPU_NUM_CHIPS);
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return main[a].height > main[b].height; });
    for (int i : order) VG_TRY(begin_upload(main[i], dm[i].get()));
    float up = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    ctx->phases.push_back({"upload traces (H2D enqueue; copies overlap the commits)", up});
    // traces in pageable memory are copied by the context's staging threads from here on (staging.cu)
    struct StagerGuard { vgpu_ctx* c; ~StagerGuard() { vg_stager_finish(c); } } sg{ctx};
    VG_TRY(vg_stager_start(ctx));
    ctx->in_host_prove = true;
    const std::vector<vgpu_dmat*> mains = vg_handles(dm), preps = vg_handles(dp);
    int32_t rc = prove_device(ctx, mains.data(), preps.data(), mains.data(), proof_out, proof_len);
    ctx->in_host_prove = false;
    if (rc == 0) rc = vg_stager_finish(ctx);
    return rc;
}

int32_t vgpu_ctx_set_debug_checks(vgpu_ctx* ctx, int32_t on) { ctx->debug_checks = on != 0; return 0; }

void vgpu_free_bytes(uint8_t* p) { std::free(p); }

uint32_t vgpu_last_prove_phases(const vgpu_ctx* cctx, const char** names, float* ms, uint32_t cap) {
    vgpu_ctx* ctx = const_cast<vgpu_ctx*>(cctx);
    cudaStreamSynchronize(ctx->stream);
    for (auto& m : ctx->phase_marks) {          // drain the event pairs of the last prove into (name, milliseconds)
        float e = 0;
        if (cudaEventElapsedTime(&e, m.a, m.b) != cudaSuccess) { cudaGetLastError(); e = -1.f; }
        ctx->phases.push_back({m.name, e});
        ctx->event_pool.push_back(m.a); ctx->event_pool.push_back(m.b);
    }
    ctx->phase_marks.clear();
    for (auto& hp : ctx->host_phases) ctx->phases.push_back(hp);
    ctx->host_phases.clear();
    uint32_t n = (uint32_t)ctx->phases.size();
    for (uint32_t i = 0; i < n && i < cap; i++) { names[i] = ctx->phases[i].first; ms[i] = ctx->phases[i].second; }
    return n;
}

}  // extern "C"
