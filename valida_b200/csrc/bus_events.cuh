// The bus events of a machine witness, as the reports over them read them: vgpu_check_buses (buses.cu) and vgpu_bus_links (links.cu).
// An EVENT is one row of one chip and one of its interactions whose multiplicity (the count VirtualPairCol on that row) is not zero;
// its tuple is (bus, the interaction's fields on the row, zero-padded to VGPU_MAX_FIELDS).
//   - BParams: one chip's sweep of this rank's run of rows (one thread per row), with check_buses' bucket, count and write state;
//   - bucket_of: the fixed hash of a tuple (Montgomery words), alike on every rank and on the host;
//   - row_events: every event of one row.
#pragma once
#include "ctx.h"
#include "devchip.h"
#include "logup.cuh"

namespace {

constexpr uint32_t BUS_NONE = 0xffffffffu;

// one event as check_buses' write pass leaves it, canonical words (22 words: all-gathered as such)
struct BusEventRec {
    uint32_t chip, interaction;
    uint64_t row;
    uint32_t multiplicity, is_send, bus, fields[VGPU_MAX_FIELDS], pad;
};
static_assert(sizeof(BusEventRec) == 88, "BusEventRec is 22 words");

struct BParams {
    const uint32_t* main; uint64_t mcs;            // at local row 0 of the rows swept
    const uint32_t* prep; uint64_t pcs;            // null without a preprocessed trace
    uint64_t g0, n;                                // global row of local row 0; rows swept
    uint32_t z;                                    // the weights' pole (Montgomery)
    uint32_t log_b;
    uint32_t bus[VGPU_MAX_INTERACTIONS];
    unsigned long long* acc;                       // bucket pass: B sums of +-mult * weight, each term < p
    const uint32_t* cand;                          // count / write passes: candidate number of each bucket, BUS_NONE if none
    uint32_t* count;                               // count pass: events per candidate
    uint32_t examined;                             // write pass: the events of candidates below it are written ...
    unsigned long long* wpos; BusEventRec* out;    // ... at out[atomicAdd(wpos, 1)]
    DevChip chip;
};

// the bucket of a tuple: a fixed 64-bit mix of the bus and the 14 padded field words (Montgomery), alike on every rank
__host__ __device__ __forceinline__ uint32_t bucket_of(uint32_t bus, const uint32_t (&f)[VGPU_MAX_FIELDS], uint32_t log_b) {
    uint64_t x = 0x9e3779b97f4a7c15ull * (bus + 1);
#pragma unroll
    for (int k = 0; k < VGPU_MAX_FIELDS; k++) {
        x = (x ^ f[k]) * 0xff51afd7ed558ccdull;
        x ^= x >> 32;
    }
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return (uint32_t)(x >> (64 - log_b));
}

// Calls f(m, mult, fields) for every event of local row i (interaction m, Montgomery words).
template <class F>
__device__ __forceinline__ void row_events(const BParams& p, uint64_t i, F&& f) {
    const uint32_t* ml = p.main + i;
    const uint32_t* pl = p.prep ? p.prep + i : nullptr;
    for (uint32_t m = 0; m < p.chip.n_interactions; m++) {
        const DevInteraction& it = p.chip.interactions[m];
        const uint32_t mult = logup::pair_col(it.count, ml, p.mcs, pl, p.pcs);
        if (!mult) continue;
        uint32_t fv[VGPU_MAX_FIELDS];
#pragma unroll
        for (int k = 0; k < VGPU_MAX_FIELDS; k++) fv[k] = (uint32_t)k < it.n_fields ? logup::pair_col(it.fields[k], ml, p.mcs, pl, p.pcs) : 0u;
        f(m, mult, fv);
    }
}

}  // namespace
