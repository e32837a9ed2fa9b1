// vgpu_check_buses: every bus tuple a machine witness leaves unbalanced, with every event that sends or receives it.
// An EVENT is one row of one chip and one of its interactions whose multiplicity (the count VirtualPairCol on that row) is not
// zero: its bus, its tuple (the interaction's fields on the row, zero-padded to VGPU_MAX_FIELDS, so trailing zeros do not tell
// tuples apart, as they do not in the LogUp denominator r1^(bus+1) + sum_f r2^f field_f) and its sign (send +, receive -).  A tuple
// is unbalanced when its sends minus its receives are not 0 mod p; the LogUp sums cancel iff no tuple is (whp over the challenges).
// Three sweeps of every row of this rank's run (a chip every rank holds whole is swept by rank 0 only: vg_reports_trace), each one
// thread per row over the chip's DevChip (logup::pair_col), no per-chip template:
//   1. bucket: each event adds +-mult / (z - L) into the bucket hash(bus, tuple) mod B, with L = limb 0 of the tuple's LogUp
//      denominator and z = limb 0 of the first challenge.  The buckets (reduced to canonical words, all-gathered on a split
//      context) that do not sum to zero are the CANDIDATES, numbered in bucket order.
//   2. count: the events of each candidate (all-gathered); the longest prefix of candidates whose events fit in cap is examined.
//   3. write: the events of the examined candidates with their tuple words (all-gathered).
// The host groups the events by exact tuple, drops the balanced ones that shared a bucket with an unbalanced one, and sorts.
#include "bus_events.cuh"
#include "lists.cuh"
#include <array>
#include <map>
#include <memory>
#include <tuple>

namespace {

constexpr int BUS_LOG_BUCKETS_MIN = 10, BUS_LOG_BUCKETS_MAX = 20;   // B = 2^10 .. 2^20 buckets

__global__ void __launch_bounds__(256) bus_bucket_kernel(const __grid_constant__ BParams p) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    row_events(p, i, [&](uint32_t m, uint32_t mult, const uint32_t (&fv)[VGPU_MAX_FIELDS]) {
        const DevInteraction& it = p.chip.interactions[m];
        uint32_t l = it.alpha.c[0];                   // limb 0 of r1^(bus+1) + sum_f r2^f field_f
#pragma unroll
        for (int k = 0; k < VGPU_MAX_FIELDS; k++) l = bb::add(l, bb::mul(p.chip.betas[k].c[0], fv[k]));
        const uint32_t v = bb::mul(mult, bb::inv(bb::sub(p.z, l)));
        atomicAdd(p.acc + bucket_of(p.bus[m], fv, p.log_b), (unsigned long long)(it.is_send ? v : bb::neg(v)));
    });
}

__global__ void __launch_bounds__(256) bus_count_kernel(const __grid_constant__ BParams p) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    row_events(p, i, [&](uint32_t m, uint32_t, const uint32_t (&fv)[VGPU_MAX_FIELDS]) {
        const uint32_t c = __ldg(p.cand + bucket_of(p.bus[m], fv, p.log_b));
        if (c != BUS_NONE) atomicAdd(p.count + c, 1u);
    });
}

__global__ void __launch_bounds__(256) bus_write_kernel(const __grid_constant__ BParams p) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    row_events(p, i, [&](uint32_t m, uint32_t mult, const uint32_t (&fv)[VGPU_MAX_FIELDS]) {
        const uint32_t c = __ldg(p.cand + bucket_of(p.bus[m], fv, p.log_b));
        if (c >= p.examined) return;                  // BUS_NONE too
        BusEventRec* e = p.out + atomicAdd(p.wpos, 1ull);
        e->chip = p.chip.chip_id; e->interaction = m; e->row = p.g0 + i;
        e->multiplicity = bb::from_monty(mult); e->is_send = p.chip.interactions[m].is_send; e->bus = p.bus[m];
#pragma unroll
        for (int k = 0; k < VGPU_MAX_FIELDS; k++) e->fields[k] = bb::from_monty(fv[k]);
        e->pad = 0;
    });
}

// this rank's bucket sums, canonical
__global__ void __launch_bounds__(256) bus_reduce_kernel(const unsigned long long* acc, uint32_t nb, uint32_t* out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < nb) out[j] = (uint32_t)(acc[j] % bb::P);
}

// the buckets whose sums over the ranks ([rank][bucket]) are not zero, appended to list in any order
__global__ void __launch_bounds__(256) bus_mark_kernel(const uint32_t* sums, uint32_t nb, uint32_t nranks, uint32_t* list, uint32_t* n_list) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nb) return;
    uint32_t s = 0;
    for (uint32_t r = 0; r < nranks; r++) s = bb::add(s, __ldg(sums + (uint64_t)r * nb + j));
    if (s) list[atomicAdd(n_list, 1u)] = j;
}

// cand[sorted[t]] = t: the candidates numbered in bucket order
__global__ void __launch_bounds__(256) bus_number_kernel(const uint32_t* sorted, uint32_t k, uint32_t* cand) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < k) cand[sorted[t]] = t;
}

unsigned blocks_of(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

extern "C" int32_t vgpu_check_buses(vgpu_ctx* ctx, const vgpu_dmat* const main[VGPU_NUM_CHIPS], const vgpu_dmat* const prep[2],
                                    const uint32_t challenges[15], uint64_t cap, vgpu_bus_imbalance* tuples, uint64_t* n_tuples,
                                    vgpu_bus_event* events, uint64_t* n_events, uint64_t* unexamined) {
    if (!main || !prep || !challenges) VG_FAIL(ctx, "check_buses: null argument");
    if (!n_tuples || !n_events || !unexamined || (cap && (!tuples || !events))) VG_FAIL(ctx, "check_buses: null output");
    VG_TRY(vg_check_machine(ctx, "check_buses", main, prep));
    VG_TRY(vg_enter(ctx));
    // the plan, from global heights and the run rule alone: alike on every rank
    const bool gather = vg_sharded(ctx);
    const uint32_t N = gather ? (uint32_t)ctx->comm_size : 1, me = gather ? (uint32_t)ctx->comm_rank : 0;
    uint64_t slots = 0;                               // interactions x rows of the whole witness
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) slots += main[i]->gh * vgpu_basic_machine_chip(i)->n_interactions;
    uint32_t log_b = BUS_LOG_BUCKETS_MIN;
    while (log_b < BUS_LOG_BUCKETS_MAX && (1ull << log_b) < slots) log_b++;
    const uint32_t B = 1u << log_b;
    std::vector<std::unique_ptr<BParams>> sweeps;
    const uint32_t z = bb::to_monty(challenges[0] % bb::P);
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) {
        const vgpu_chip_desc* d = vgpu_basic_machine_chip(i);
        const vgpu_dmat *m = main[i], *pr = vg_machine_prep(prep, i);
        VgRun run;
        if (!d->n_interactions || !vg_reports_trace(ctx, m->gh, &run)) continue;
        VG_TRY(vg_dmat_materialize(ctx, m));
        VG_TRY(vg_dmat_materialize(ctx, pr));
        auto p = std::make_unique<BParams>();
        p->main = vg_run_rows(m, run); p->mcs = m->col_stride;
        p->prep = vg_run_rows(pr, run); p->pcs = pr ? pr->col_stride : 0;
        p->g0 = run.begin; p->n = run.count;
        p->z = z; p->log_b = log_b;
        for (uint32_t k = 0; k < d->n_interactions; k++) p->bus[k] = d->interactions[k].bus;
        VG_TRY(vg_build_devchip(ctx, d, challenges, &p->chip));
        if (p->n) sweeps.push_back(std::move(p));
    }
    VgBuf acc(ctx), sums(ctx), cand(ctx), list(ctx), nlist(ctx);
    VG_TRY(acc.alloc((size_t)B * 8));
    VG_TRY(sums.alloc((size_t)N * B * 4));
    VG_TRY(cand.alloc((size_t)B * 4));
    VG_TRY(list.alloc((size_t)B * 4));
    VG_TRY(nlist.alloc(4));
    VG_CUDA(ctx, cudaMemsetAsync(acc.p, 0, (size_t)B * 8, ctx->stream));
    VG_CUDA(ctx, cudaMemsetAsync(nlist.p, 0, 4, ctx->stream));
    auto launch = [&](void (*kernel)(BParams)) -> int32_t {
        for (auto& p : sweeps) {
            KScope ks(ctx, KC_CHECK, 4.0 * (double)p->n * (double)(p->chip.width + p->chip.prep_width));
            kernel<<<blocks_of(p->n, 256), 256, 0, ctx->stream>>>(*p);
            VG_LAUNCH_CHECK(ctx);
        }
        return 0;
    };
    for (auto& p : sweeps) p->acc = acc.as<unsigned long long>();
    VG_TRY(launch(bus_bucket_kernel));
    {
        KScope ks(ctx, KC_CHECK, 12.0 * B);
        bus_reduce_kernel<<<blocks_of(B, 256), 256, 0, ctx->stream>>>(acc.as<unsigned long long>(), B, sums.as<uint32_t>() + (uint64_t)me * B);
        VG_LAUNCH_CHECK(ctx);
    }
    if (gather) VG_TRY(vg_comm_allgather_inplace(ctx, sums.as<uint32_t>(), B));
    {
        KScope ks(ctx, KC_CHECK, 4.0 * N * B);
        bus_mark_kernel<<<blocks_of(B, 256), 256, 0, ctx->stream>>>(sums.as<uint32_t>(), B, N, list.as<uint32_t>(), nlist.as<uint32_t>());
        VG_LAUNCH_CHECK(ctx);
    }
    uint32_t K = 0;
    VG_CUDA(ctx, cudaMemcpyAsync(&K, nlist.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *n_tuples = 0; *n_events = 0; *unexamined = 0;
    if (!K) return 0;
    // the candidates in bucket order: every rank numbers them alike
    std::vector<uint32_t> cands(K);
    VG_CUDA(ctx, cudaMemcpyAsync(cands.data(), list.p, (size_t)K * 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::sort(cands.begin(), cands.end());
    VG_CUDA(ctx, cudaMemcpyAsync(list.p, cands.data(), (size_t)K * 4, cudaMemcpyHostToDevice, ctx->stream));
    VG_CUDA(ctx, cudaMemsetAsync(cand.p, 0xff, (size_t)B * 4, ctx->stream));
    VgBuf counts(ctx);
    VG_TRY(counts.alloc((size_t)N * K * 4));
    uint32_t* mine = counts.as<uint32_t>() + (uint64_t)me * K;
    VG_CUDA(ctx, cudaMemsetAsync(mine, 0, (size_t)K * 4, ctx->stream));
    {
        KScope ks(ctx, KC_CHECK, 8.0 * K);
        bus_number_kernel<<<blocks_of(K, 256), 256, 0, ctx->stream>>>(list.as<uint32_t>(), K, cand.as<uint32_t>());
        VG_LAUNCH_CHECK(ctx);
    }
    for (auto& p : sweeps) { p->cand = cand.as<uint32_t>(); p->count = mine; }
    VG_TRY(launch(bus_count_kernel));
    if (gather) VG_TRY(vg_comm_allgather_inplace(ctx, counts.as<uint32_t>(), K));
    std::vector<uint32_t> hc((size_t)N * K);
    VG_CUDA(ctx, cudaMemcpyAsync(hc.data(), counts.p, hc.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // the longest prefix of candidates whose events (all ranks) fit in cap
    uint32_t J = 0;
    uint64_t fit = 0;
    for (; J < K; J++) {
        uint64_t t = 0;
        for (uint32_t r = 0; r < N; r++) t += hc[(size_t)r * K + J];
        if (fit + t > cap) break;
        fit += t;
    }
    *unexamined = K - J;
    if (!J) return 0;
    std::vector<uint64_t> per(N, 0);
    for (uint32_t r = 0; r < N; r++)
        for (uint32_t c = 0; c < J; c++) per[r] += hc[(size_t)r * K + c];
    std::vector<BusEventRec> he(fit);
    uint64_t gathered = 0;
    VG_TRY(vg_gather_lists(ctx, gather, per, cap, [&](BusEventRec* slot) -> int32_t {
        VgBuf wpos(ctx);
        VG_TRY(wpos.alloc(8));
        VG_CUDA(ctx, cudaMemsetAsync(wpos.p, 0, 8, ctx->stream));
        for (auto& p : sweeps) { p->examined = J; p->wpos = wpos.as<unsigned long long>(); p->out = slot; }
        return launch(bus_write_kernel);
    }, he.data(), fit, &gathered));
    // group by exact tuple (bus, fields): ascending, as the map orders its keys
    std::map<std::array<uint32_t, 1 + VGPU_MAX_FIELDS>, std::vector<const BusEventRec*>> groups;
    for (const BusEventRec& x : he) {
        std::array<uint32_t, 1 + VGPU_MAX_FIELDS> key;
        key[0] = x.bus;
        std::copy(x.fields, x.fields + VGPU_MAX_FIELDS, key.begin() + 1);
        groups[key].push_back(&x);
    }
    uint64_t nt = 0, ne = 0;
    for (auto& [key, evs] : groups) {
        uint32_t net = 0;
        for (const BusEventRec* e : evs) net = e->is_send ? bb::add(net, e->multiplicity) : bb::sub(net, e->multiplicity);
        if (!net) continue;
        std::sort(evs.begin(), evs.end(), [](const BusEventRec* a, const BusEventRec* b) {
            return std::tie(a->chip, a->row, a->interaction) < std::tie(b->chip, b->row, b->interaction);
        });
        vgpu_bus_imbalance& t = tuples[nt++];
        t.bus = key[0];
        std::copy(key.begin() + 1, key.end(), t.fields);
        t.net = net;
        t.first_event = ne; t.n_events = evs.size();
        for (const BusEventRec* e : evs) events[ne++] = vgpu_bus_event{e->chip, e->interaction, (int64_t)e->row, e->multiplicity, e->is_send};
    }
    *n_tuples = nt; *n_events = ne;
    return 0;
}
