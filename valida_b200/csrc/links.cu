// vgpu_bus_links: every event of a machine witness that carries the tuple of each of n items (chip, interaction, row), on both sides
// of the bus.  Events and tuples are check_buses' (bus_events.cuh).  Three steps:
//   1. item tuples: the words each item's count and fields read on its row, reported by the rank that holds the row and brought to
//      every rank by one vg_gather_words (one all-gather, summed).  The host evaluates the VirtualPairCols, orders the K distinct tuples
//      ascending by (bus, canonical fields) and uploads an open-addressed table of them: slot -> tuple, probed linearly from bucket_of;
//      keys (bus and 14 Montgomery words) compared exactly.
//   2. count: one thread per row of this rank's run of every chip (vg_reports_trace) probes the table for each event of its row and
//      adds to the tuple's event count and send or receive sum (64-bit, terms below p).  One all-gather brings every rank's.
//   3. write: only when some listed tuple has events, the same sweep writes the events of the longest prefix of tuples that fits in
//      cap, with their tuple numbers; vg_gather_lists gathers them and the host sorts each tuple's events by (chip, row, interaction).
#include "bus_events.cuh"
#include "lists.cuh"
#include "open.h"
#include <array>
#include <map>
#include <memory>
#include <tuple>

namespace {

constexpr int LINK_KEY_WORDS = 1 + VGPU_MAX_FIELDS;   // bus, then the padded fields (Montgomery)

// one listed event as the write pass leaves it, canonical words (8 words: all-gathered as such)
struct LinkRec {
    uint32_t chip, interaction;
    uint64_t row;
    uint32_t multiplicity, is_send, tuple, pad;
};
static_assert(sizeof(LinkRec) == 32, "LinkRec is 8 words");

// One chip's sweep.  Of the bucket sweeps' block it reads the rows, the buses and the chip, and it takes
//   rows.log_b / rows.cand: the table's log2 size and its slots (tuple number, BUS_NONE: empty);
//   rows.acc: per tuple [events, sum of the sends' multiplicities, sum of the receives'];
//   rows.examined / rows.wpos: the write pass writes the events of the tuples below `examined` at out[atomicAdd(wpos, 1)].
struct LParams {
    BParams rows;
    const uint32_t* keys;                          // [tuple][LINK_KEY_WORDS]
    LinkRec* out;
};

// the number of the item tuple (bus, fv), BUS_NONE when no item carries it; the table is at most half full, so a probe ends
__device__ __forceinline__ uint32_t find_tuple(const LParams& p, uint32_t bus, const uint32_t (&fv)[VGPU_MAX_FIELDS]) {
    const uint32_t mask = (1u << p.rows.log_b) - 1;
    for (uint32_t s = bucket_of(bus, fv, p.rows.log_b);; s = (s + 1) & mask) {
        const uint32_t t = __ldg(p.rows.cand + s);
        if (t == BUS_NONE) return BUS_NONE;
        const uint32_t* k = p.keys + (uint64_t)t * LINK_KEY_WORDS;
        bool eq = __ldg(k) == bus;
#pragma unroll
        for (int f = 0; f < VGPU_MAX_FIELDS; f++) eq &= __ldg(k + 1 + f) == fv[f];
        if (eq) return t;
    }
}

__global__ void __launch_bounds__(256) link_count_kernel(const __grid_constant__ LParams p) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.rows.n) return;
    row_events(p.rows, i, [&](uint32_t m, uint32_t mult, const uint32_t (&fv)[VGPU_MAX_FIELDS]) {
        const uint32_t t = find_tuple(p, p.rows.bus[m], fv);
        if (t == BUS_NONE) return;
        unsigned long long* a = p.rows.acc + 3ull * t;
        atomicAdd(a, 1ull);
        atomicAdd(a + (p.rows.chip.interactions[m].is_send ? 1 : 2), (unsigned long long)bb::from_monty(mult));
    });
}

__global__ void __launch_bounds__(256) link_write_kernel(const __grid_constant__ LParams p) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.rows.n) return;
    row_events(p.rows, i, [&](uint32_t m, uint32_t mult, const uint32_t (&fv)[VGPU_MAX_FIELDS]) {
        const uint32_t t = find_tuple(p, p.rows.bus[m], fv);
        if (t >= p.rows.examined) return;             // BUS_NONE too
        LinkRec* e = p.out + atomicAdd(p.rows.wpos, 1ull);
        *e = LinkRec{p.rows.chip.chip_id, m, p.rows.g0 + i, bb::from_monty(mult), p.rows.chip.interactions[m].is_send, t, 0};
    });
}

unsigned blocks_of(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

using Key = std::array<uint32_t, LINK_KEY_WORDS>;

}  // namespace

extern "C" int32_t vgpu_bus_links(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                                  const vgpu_bus_event* items, uint64_t n, vgpu_bus_link* links, uint64_t cap, vgpu_bus_event* events,
                                  uint64_t* n_events, uint64_t* unlisted) {
    if (!main || !prep || (n && !items)) VG_FAIL(ctx, "bus_links: null argument");
    if (!n_events || !unlisted || (n && !links) || (cap && !events)) VG_FAIL(ctx, "bus_links: null output");
    VG_TRY(vg_check_machine(ctx, "bus_links", main, prep));
    for (uint64_t i = 0; i < n; i++) {
        const vgpu_bus_event& it = items[i];
        if (it.chip >= VGPU_NUM_CHIPS) VG_FAIL(ctx, "bus_links: item %llu: chip %u is not one of the machine's %d", (unsigned long long)i, it.chip, VGPU_NUM_CHIPS);
        const uint32_t k = vgpu_basic_machine_chip(it.chip)->n_interactions;
        if (it.interaction >= k)
            VG_FAIL(ctx, "bus_links: item %llu: interaction %u is not below chip %u's %u interactions", (unsigned long long)i, it.interaction, it.chip, k);
        const uint64_t h = main[it.chip]->gh;
        if (it.row < 0 || (uint64_t)it.row >= h)
            VG_FAIL(ctx, "bus_links: item %llu: row %lld is outside chip %u's trace of height %llu", (unsigned long long)i, (long long)it.row, it.chip,
                    (unsigned long long)h);
    }
    *n_events = 0; *unlisted = 0;
    if (!n) return 0;
    VG_TRY(vg_enter(ctx));
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) VG_TRY(vg_dmat_materialize(ctx, main[i]));
    for (int j = 0; j < 2; j++) VG_TRY(vg_dmat_materialize(ctx, prep[j]));
    // 1. the words behind each item's count and fields, in pair-column and term order
    auto pair_cols = [](const vgpu_bus_event& it, auto&& f) {
        const vgpu_interaction& x = vgpu_basic_machine_chip(it.chip)->interactions[it.interaction];
        f(x.count);
        for (uint32_t k = 0; k < x.n_fields && k < VGPU_MAX_FIELDS; k++) f(x.fields[k]);
    };
    std::vector<const uint32_t*> ptrs;
    for (uint64_t i = 0; i < n; i++) {
        const vgpu_bus_event& it = items[i];
        pair_cols(it, [&](const vgpu_pair_col& pc) {
            for (uint32_t t = 0; t < pc.n_terms && t < VGPU_MAX_TERMS; t++)
                ptrs.push_back(vg_reported_word(ctx, pc.terms[t].is_preprocessed ? vg_machine_prep(prep, it.chip) : main[it.chip], (uint64_t)it.row,
                                                pc.terms[t].column));
        });
    }
    std::vector<uint32_t> words;
    VG_TRY(vg_gather_words(ctx, ptrs, &words));
    // each item's count and key (Montgomery), and the distinct keys ascending by (bus, canonical fields)
    std::vector<uint32_t> mult(n);
    std::vector<Key> key(n);
    std::map<Key, uint32_t> order;                    // canonical key -> tuple number
    size_t w = 0;
    for (uint64_t i = 0; i < n; i++) {
        const vgpu_bus_event& it = items[i];
        std::vector<uint32_t> v;
        pair_cols(it, [&](const vgpu_pair_col& pc) {
            uint32_t x = bb::to_monty(pc.constant % bb::P);
            for (uint32_t t = 0; t < pc.n_terms && t < VGPU_MAX_TERMS; t++) x = bb::add(x, bb::mul(words[w++], bb::to_monty(pc.terms[t].weight % bb::P)));
            v.push_back(x);
        });
        mult[i] = bb::from_monty(v[0]);
        key[i].fill(0);
        key[i][0] = vgpu_basic_machine_chip(it.chip)->interactions[it.interaction].bus;
        std::copy(v.begin() + 1, v.end(), key[i].begin() + 1);
        Key c = key[i];
        for (int f = 1; f < LINK_KEY_WORDS; f++) c[f] = bb::from_monty(c[f]);
        order.emplace(c, 0);
    }
    const uint32_t K = (uint32_t)order.size();
    uint32_t next = 0;
    for (auto& kv : order) kv.second = next++;
    std::vector<uint32_t> tuple_of(n), hkeys((size_t)K * LINK_KEY_WORDS);
    for (uint64_t i = 0; i < n; i++) {
        Key c = key[i];
        for (int f = 1; f < LINK_KEY_WORDS; f++) c[f] = bb::from_monty(c[f]);
        tuple_of[i] = order[c];
        std::copy(key[i].begin(), key[i].end(), hkeys.begin() + (size_t)tuple_of[i] * LINK_KEY_WORDS);
    }
    uint32_t log_t = 4;
    while ((1ull << log_t) < 2ull * K) log_t++;
    std::vector<uint32_t> slots(1ull << log_t, BUS_NONE);
    for (uint32_t t = 0; t < K; t++) {
        uint32_t f[VGPU_MAX_FIELDS];
        std::copy(hkeys.begin() + (size_t)t * LINK_KEY_WORDS + 1, hkeys.begin() + (size_t)(t + 1) * LINK_KEY_WORDS, f);
        uint32_t s = bucket_of(hkeys[(size_t)t * LINK_KEY_WORDS], f, log_t);
        while (slots[s] != BUS_NONE) s = (s + 1) & ((1u << log_t) - 1);
        slots[s] = t;
    }
    // 2. the count sweep over this rank's run of every chip
    const bool gather = vg_sharded(ctx);
    const uint32_t N = gather ? (uint32_t)ctx->comm_size : 1, me = gather ? (uint32_t)ctx->comm_rank : 0;
    VgBuf dslots(ctx), dkeys(ctx), acc(ctx);
    VG_TRY(dslots.upload(slots.data(), slots.size()));
    VG_TRY(dkeys.upload(hkeys.data(), hkeys.size()));
    VG_TRY(acc.alloc((size_t)N * 3 * K * 8));
    unsigned long long* mine = acc.as<unsigned long long>() + (uint64_t)me * 3 * K;
    VG_CUDA(ctx, cudaMemsetAsync(mine, 0, (size_t)3 * K * 8, ctx->stream));
    static const uint32_t no_challenges[15] = {};     // the sweeps read no LogUp randomness
    std::vector<std::unique_ptr<LParams>> sweeps;
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        const vgpu_chip_desc* d = vgpu_basic_machine_chip(i);
        const vgpu_dmat *m = main[i], *pr = vg_machine_prep(prep, i);
        VgRun run;
        if (!d->n_interactions || !vg_reports_trace(ctx, m->gh, &run) || !run.count) continue;
        auto p = std::make_unique<LParams>();
        BParams& b = p->rows;
        b.main = vg_run_rows(m, run); b.mcs = m->col_stride;
        b.prep = vg_run_rows(pr, run); b.pcs = pr ? pr->col_stride : 0;
        b.g0 = run.begin; b.n = run.count;
        b.log_b = log_t; b.cand = dslots.as<uint32_t>(); b.acc = mine;
        for (uint32_t k = 0; k < d->n_interactions; k++) b.bus[k] = d->interactions[k].bus;
        VG_TRY(vg_build_devchip(ctx, d, no_challenges, &b.chip));
        p->keys = dkeys.as<uint32_t>();
        sweeps.push_back(std::move(p));
    }
    auto launch = [&](void (*kernel)(LParams)) -> int32_t {
        for (auto& p : sweeps) {
            KScope ks(ctx, KC_CHECK, 4.0 * (double)p->rows.n * (double)(p->rows.chip.width + p->rows.chip.prep_width));
            kernel<<<blocks_of(p->rows.n, 256), 256, 0, ctx->stream>>>(*p);
            VG_LAUNCH_CHECK(ctx);
        }
        return 0;
    };
    VG_TRY(launch(link_count_kernel));
    if (gather) VG_TRY(vg_comm_allgather_inplace(ctx, acc.as<uint32_t>(), (uint64_t)6 * K));
    std::vector<unsigned long long> ha((size_t)N * 3 * K);
    VG_CUDA(ctx, cudaMemcpyAsync(ha.data(), acc.p, ha.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<uint64_t> count(K, 0);
    std::vector<uint32_t> sends(K, 0), receives(K, 0);
    for (uint32_t r = 0; r < N; r++)
        for (uint32_t t = 0; t < K; t++) {
            const unsigned long long* a = ha.data() + ((size_t)r * K + t) * 3;
            count[t] += a[0];
            sends[t] = bb::add(sends[t], (uint32_t)(a[1] % bb::P));
            receives[t] = bb::add(receives[t], (uint32_t)(a[2] % bb::P));
        }
    // the longest prefix of tuples whose events fit in cap
    uint32_t J = 0;
    uint64_t fit = 0;
    for (; J < K && fit + count[J] <= cap; J++) fit += count[J];
    *unlisted = K - J;
    // 3. the listed tuples' events
    std::vector<LinkRec> he(fit);
    if (fit) {
        std::vector<uint64_t> per(N, 0);
        for (uint32_t r = 0; r < N; r++)
            for (uint32_t t = 0; t < J; t++) per[r] += ha[((size_t)r * K + t) * 3];
        uint64_t gathered = 0;
        VG_TRY(vg_gather_lists(ctx, gather, per, cap, [&](LinkRec* slot) -> int32_t {
            VgBuf wpos(ctx);
            VG_TRY(wpos.alloc(8));
            VG_CUDA(ctx, cudaMemsetAsync(wpos.p, 0, 8, ctx->stream));
            for (auto& p : sweeps) { p->rows.examined = J; p->rows.wpos = wpos.as<unsigned long long>(); p->out = slot; }
            return launch(link_write_kernel);
        }, he.data(), fit, &gathered));
        if (gathered != fit) VG_FAIL(ctx, "bus_links: the write sweep listed %llu events of the %llu counted", (unsigned long long)gathered, (unsigned long long)fit);
    }
    std::sort(he.begin(), he.end(), [](const LinkRec& a, const LinkRec& b) {
        return std::tie(a.tuple, a.chip, a.row, a.interaction) < std::tie(b.tuple, b.chip, b.row, b.interaction);
    });
    std::vector<uint64_t> first(K, UINT64_MAX);
    for (uint64_t t = 0, e = 0; t < J; e += count[t++]) first[t] = e;
    for (uint64_t e = 0; e < fit; e++) events[e] = vgpu_bus_event{he[e].chip, he[e].interaction, (int64_t)he[e].row, he[e].multiplicity, he[e].is_send};
    *n_events = fit;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t t = tuple_of[i];
        vgpu_bus_link& l = links[i];
        l.bus = key[i][0];
        for (int f = 0; f < VGPU_MAX_FIELDS; f++) l.fields[f] = bb::from_monty(key[i][1 + f]);
        l.multiplicity = mult[i];
        l.sends = sends[t]; l.receives = receives[t];
        l.n_events = count[t];
        l.first_event = t < J ? first[t] : UINT64_MAX;
    }
    return 0;
}
