// C1 — the two transposing exchanges of a split commit (SURVEY.md §8(e), option B), written as kernels that STORE
// THROUGH PEER POINTERS: the data moves over NVLink while the kernel runs, no staging buffer and no collective call.
//   rows -> columns : a rank holds a contiguous run of rows of a trace (what it uploaded, or what its LogUp / quotient
//                     sweep produced); every column goes to the rank that extends that column (coset LDE);
//   columns -> rows : the extended columns are cut into the ranks' runs (ctx.h) of the committed (bit-reversed) row
//                     order and every run goes to the rank that owns those rows from then on (leaf hashing, sub-tree,
//                     quotient sweep, openings, FRI) — the ONE bulk exchange of a commit.
// Both are followed by vg_comm_barrier() (stream-ordered) before anybody reads what it received.
// No reference counterpart: the reference is single-process rayon (derive/src/lib.rs:302,316,341).
#include "ctx.h"

namespace {

constexpr int MAX_RANKS = 16;

struct R2CParams {
    const uint32_t* src; uint64_t scs, hl;      // local rows: hl x w, column stride scs
    uint64_t gh, row0;                          // logical height and the first local row
    uint32_t* dst[MAX_RANKS];                   // peer d's column buffer (columns [c0[d], c0[d+1]) at stride gh)
    uint32_t c0[MAX_RANKS + 1];
    uint32_t nranks;
};
// grid: x = 16-byte chunks of the local rows, y = column
__global__ void __launch_bounds__(256) rows_to_cols_kernel(const __grid_constant__ R2CParams p) {
    const uint32_t c = blockIdx.y;
    uint32_t d = 0;
    while (d + 1 < p.nranks && c >= p.c0[d + 1]) d++;
    const uint64_t n4 = p.hl >> 2;
    const uint4* s = reinterpret_cast<const uint4*>(p.src + (uint64_t)c * p.scs);
    uint4* o = reinterpret_cast<uint4*>(p.dst[d] + (uint64_t)(c - p.c0[d]) * p.gh + p.row0);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (uint64_t)gridDim.x * blockDim.x) o[i] = __ldg(s + i);
}
// The same hand-over from a row shard whose columns are not 16-byte aligned (a borrowed caller buffer: 4-byte alignment, any column
// stride): four 32-bit loads per 16-byte chunk of a column, one 16-byte store into the peer's column buffer, which is aligned (a
// symmetric-heap allocation, gh and row0 multiples of 4).
__global__ void __launch_bounds__(256) rows_to_cols_scalar_kernel(const __grid_constant__ R2CParams p) {
    const uint32_t c = blockIdx.y;
    uint32_t d = 0;
    while (d + 1 < p.nranks && c >= p.c0[d + 1]) d++;
    const uint64_t n4 = p.hl >> 2;
    const uint32_t* s = p.src + (uint64_t)c * p.scs;
    uint4* o = reinterpret_cast<uint4*>(p.dst[d] + (uint64_t)(c - p.c0[d]) * p.gh + p.row0);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (uint64_t)gridDim.x * blockDim.x)
        o[i] = make_uint4(__ldg(s + 4 * i), __ldg(s + 4 * i + 1), __ldg(s + 4 * i + 2), __ldg(s + 4 * i + 3));
}

struct C2RParams {
    const uint32_t* src; uint64_t H, cs;        // local columns [c0, c1) at stride H; cs: the shards' column stride (the same on every rank)
    uint32_t* dst[MAX_RANKS];                   // peer d's shard matrix (rows [rb[d], rb[d + 1]) x w, stride cs)
    uint64_t rb[MAX_RANKS + 1];                 // the run table: rank d holds committed rows [rb[d], rb[d + 1])
    uint32_t c0, nranks;
};
// grid: x = 16-byte chunks of a shard column, y = local column, z = destination rank
__global__ void __launch_bounds__(256) cols_to_rows_kernel(const __grid_constant__ C2RParams p) {
    const uint32_t lc = blockIdx.y, d = blockIdx.z;
    const uint64_t n4 = (p.rb[d + 1] - p.rb[d]) >> 2;
    const uint4* s = reinterpret_cast<const uint4*>(p.src + (uint64_t)lc * p.H + p.rb[d]);
    uint4* o = reinterpret_cast<uint4*>(p.dst[d] + (uint64_t)(p.c0 + lc) * p.cs);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (uint64_t)gridDim.x * blockDim.x) o[i] = __ldg(s + i);
}

}  // namespace

// rows: this rank's row shard (VG_ROWS) of a gh x gw matrix.  cols_symm: a symmetric-heap buffer (the same size on every rank, room
// for the widest share); after the barrier that follows, it holds this rank's columns [col_begin[rank], col_begin[rank + 1]) at stride gh.
// A shard the library allocated has 16-byte aligned columns and is read with vector loads; a borrowed one may have any column stride
// and a 4-byte aligned base, and is read a word at a time.
int32_t vg_exchange_rows_to_cols(vgpu_ctx* ctx, const vgpu_dmat* rows, uint32_t* cols_symm, const uint32_t* col_begin /* comm_size + 1 */) {
    const int G = ctx->comm_size;
    if (rows->dist != VG_ROWS || (rows->h & 3) || (rows->row0 & 3)) VG_FAIL(ctx, "exchange: row shard of %llu rows at %llu is not 16-byte aligned", (unsigned long long)rows->h, (unsigned long long)rows->row0);
    const bool vec = ((uintptr_t)rows->d & 15) == 0 && (rows->col_stride & 3) == 0;
    R2CParams p{};
    p.src = rows->d; p.scs = rows->col_stride; p.hl = rows->h; p.gh = rows->gh; p.row0 = rows->row0; p.nranks = (uint32_t)G;
    for (int d = 0; d <= G; d++) p.c0[d] = col_begin[d];
    for (int d = 0; d < G; d++) p.dst[d] = vg_peer_ptr(ctx, cols_symm, d);
    const uint64_t n4 = rows->h >> 2;
    unsigned gx = (unsigned)((n4 + 255) / 256);
    if (gx > 64) gx = 64;
    KScope ks(ctx, KC_EXCHANGE, 8.0 * (double)rows->h * (double)rows->gw);
    if (vec) rows_to_cols_kernel<<<dim3(gx, (unsigned)rows->gw), 256, 0, ctx->stream>>>(p);
    else rows_to_cols_scalar_kernel<<<dim3(gx, (unsigned)rows->gw), 256, 0, ctx->stream>>>(p);
    VG_LAUNCH_CHECK(ctx);
    ctx->stat_exchange.calls++; ctx->stat_exchange.bytes += 4.0 * (double)rows->h * (double)rows->gw * (G - 1) / G;
    return 0;
}

// lde_cols: this rank's extended columns [c0, c1) of a matrix of H rows (stride H, committed row order).  shard: the VG_ROWS
// matrix (this rank's run of the H rows x gw, symmetric heap) that receives, on every rank, that rank's run of rows of ALL columns.
int32_t vg_exchange_cols_to_rows(vgpu_ctx* ctx, const uint32_t* lde_cols, uint64_t H, uint64_t c0, uint64_t c1, vgpu_dmat* shard, cudaStream_t on) {
    const cudaStream_t st = on ? on : ctx->stream;
    const int G = ctx->comm_size;
    if (c1 <= c0) return 0;
    if (shard->dist != VG_ROWS || !shard->symm || shard->gh != H || shard->col_stride != vg_run_max(H, G) || (shard->h & 3))
        VG_FAIL(ctx, "exchange: shard matrix does not match the extended columns");
    C2RParams p{};
    p.src = lde_cols; p.H = H; p.cs = shard->col_stride; p.c0 = (uint32_t)c0; p.nranks = (uint32_t)G;
    for (int d = 0; d <= G; d++) p.rb[d] = vg_run_bound(H, G, d);
    for (int d = 0; d < G; d++) p.dst[d] = vg_peer_ptr(ctx, shard->d, d);
    const uint64_t n4 = shard->col_stride >> 2;
    unsigned gx = (unsigned)((n4 + 255) / 256);
    if (gx > 64) gx = 64;
    KScope ks(ctx, KC_EXCHANGE, 8.0 * (double)H * (double)(c1 - c0));
    cols_to_rows_kernel<<<dim3(gx, (unsigned)(c1 - c0), (unsigned)G), 256, 0, st>>>(p);
    VG_LAUNCH_CHECK(ctx);
    ctx->stat_exchange.calls++; ctx->stat_exchange.bytes += 4.0 * (double)(H - shard->h) * (double)(c1 - c0);
    return 0;
}
