// K3/K4 — Keccak-256 Merkle commitment over mixed-height column-major LDE matrices (sm_90a).
// Replaces FieldMerkleTreeMmcs<BabyBear, SerializingHasher32<Keccak256Hash>,
// CompressionFunctionFromHasher<_,_,2,8>, 8>::commit (basic/src/bin/valida.rs:367-374) as reached
// from TwoAdicFriPcs::commit_shifted_batches (derive/src/lib.rs:309,330,355,372).
//  * leaf kernel: one thread per LDE row; the row of every matrix of that height is streamed from
//    the column-major store (coalesced across the warp), converted Montgomery -> canonical, absorbed
//    little-endian into a register-resident 1600-bit state; digest words are reduced mod p;
//  * node kernel: one thread per parent, 64-byte compression (one permutation), with the
//    "inject shorter matrices" rule: node = compress(compress(l, r), hash(rows at that height)).
//  * short layers (<= 2^15 nodes): tree_tail_kernel reduces a sub-tree per CTA in shared memory, a thread per node while a level is
//    wide, a warp per node (the Keccak state spread over 25 lanes) on the last levels, where only the dependent chain is left.
//  * query_path_kernel: a query's path below the kept layers (merkle.h), rebuilt from the leaves by one CTA per path.
// With VGPU_MERKLE_POSEIDON16 the p16_* kernels take the place of each of these, with the same plan, layout and launches.
// Digests are stored canonical, 8 words (32 B) per node.  Every layer is computed, but only layers VG_TREE_DROP and up are kept for
// the opening phase; the lower ones live in a transient block freed when the build returns.  Split proof (merkle.h): a rank
// computes and keeps its run of every layer — the sub-tree over its rows — and only the last split layer (merkle.h) is all-gathered.
#include "ctx.h"
#include "keccak.cuh"
#include "merkle.h"
#include "poseidon.cuh"
#include <algorithm>
#include <cstring>
#include <numeric>

namespace {

constexpr int RATE_WORDS = 34;   // 136-byte rate

// Sponge over `nwords` canonical words fetched by `fetch(i)`; Keccak pad 0x01 .. 0x80.
template <bool SHORT = false, class Fetch>
__device__ __forceinline__ void keccak256_words(const uint32_t nwords, Fetch fetch, uint32_t out[8]) {
    uint2 A[25];
#pragma unroll
    for (int i = 0; i < 25; i++) A[i] = make_uint2(0, 0);
    uint32_t nblocks = nwords / RATE_WORDS + 1;
    if (SHORT) {   // a single block whose length the compiler sees (64-byte compression, FRI leaf): zero lanes fold away in round 0
#pragma unroll
        for (int i = 0; i < RATE_WORDS / 2; i++) {
            const uint32_t g0 = 2 * i, g1 = g0 + 1;
            uint32_t w0 = g0 < nwords ? fetch(g0) : (g0 == nwords ? 1u : 0u);
            uint32_t w1 = g1 < nwords ? fetch(g1) : (g1 == nwords ? 1u : 0u);
            if (i == RATE_WORDS / 2 - 1) w1 ^= 0x80000000u;
            A[i] = make_uint2(w0, w1);
        }
        kk::keccak_f_peeled<true, true>(A);
        out[0] = A[0].x; out[1] = A[0].y; out[2] = A[1].x; out[3] = A[1].y;
        out[4] = A[2].x; out[5] = A[2].y; out[6] = A[3].x; out[7] = A[3].y;
        return;
    }
    for (uint32_t b = 0; b < nblocks; b++) {
        uint32_t base = b * RATE_WORDS;
#pragma unroll
        for (int i = 0; i < RATE_WORDS / 2; i++) {
            uint32_t g0 = base + 2 * i, g1 = g0 + 1;
            uint32_t w0 = g0 < nwords ? fetch(g0) : (g0 == nwords ? 1u : 0u);
            uint32_t w1 = g1 < nwords ? fetch(g1) : (g1 == nwords ? 1u : 0u);
            if (i == RATE_WORDS / 2 - 1 && b == nblocks - 1) w1 ^= 0x80000000u;
            A[i].x ^= w0; A[i].y ^= w1;
        }
        if (b == nblocks - 1) kk::keccak_f_peeled<false, true>(A); else kk::keccak_f(A);
    }
    out[0] = A[0].x; out[1] = A[0].y; out[2] = A[1].x; out[3] = A[1].y;
    out[4] = A[2].x; out[5] = A[2].y; out[6] = A[3].x; out[7] = A[3].y;
}

__device__ __forceinline__ uint32_t wrap_mod_p(uint32_t w) {   // F::from_wrapped_u32
    w = bb::umin32(w, w - bb::P);
    return bb::umin32(w, w - bb::P);
}

// colptr[i] = device pointer to column i of the concatenated row (all matrices of this height).
// rows [row0, row0 + nrows) of the layer (a rank's share when the tree is split across GPUs)
__global__ void __launch_bounds__(128) leaf_hash_kernel(const uint32_t* const* __restrict__ colptr, uint32_t nwords, uint64_t row0, uint64_t nrows, uint32_t* __restrict__ digests) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    r += row0;
    uint32_t d[8];
    keccak256_words(nwords, [&](uint32_t i) { return bb::from_monty(__ldg(colptr[i] + r)); }, d);
    uint4* o = reinterpret_cast<uint4*>(digests + r * 8);
    o[0] = make_uint4(wrap_mod_p(d[0]), wrap_mod_p(d[1]), wrap_mod_p(d[2]), wrap_mod_p(d[3]));
    o[1] = make_uint4(wrap_mod_p(d[4]), wrap_mod_p(d[5]), wrap_mod_p(d[6]), wrap_mod_p(d[7]));
}

// Rows of at most LEAF_NB_MAX sponge blocks (nwords / RATE_WORDS + 1 blocks with the padding: up to 67 words) take
// leaf_hash_kernel_blocks<NB>, whose absorption is unrolled for exactly NB blocks: the slots of every block but the last are all
// row words, the first block runs the round-0-peeled permutation (its capacity lanes are zero) and the last the round-23-peeled
// one, and the column pointers come from the kernel's parameter space rather than a table in global memory.
constexpr int LEAF_NB_MAX = 2;
struct LeafCols { const uint32_t* col[LEAF_NB_MAX * RATE_WORDS]; };
template <int NB>
__global__ void __launch_bounds__(128) leaf_hash_kernel_blocks(const __grid_constant__ LeafCols c, uint32_t nwords, uint64_t row0, uint64_t nrows, uint32_t* __restrict__ digests) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    r += row0;
    uint2 A[25];
#pragma unroll
    for (int i = 0; i < 25; i++) A[i] = make_uint2(0, 0);
#pragma unroll
    for (int b = 0; b < NB; b++) {
#pragma unroll
        for (int i = 0; i < RATE_WORDS; i++) {
            const uint32_t g = b * RATE_WORDS + i;
            uint32_t w = (b < NB - 1 || g < nwords) ? bb::from_monty(__ldg(c.col[g] + r)) : (g == nwords ? 1u : 0u);
            if (b == NB - 1 && i == RATE_WORDS - 1) w ^= 0x80000000u;
            if (i & 1) A[i / 2].y ^= w; else A[i / 2].x ^= w;
        }
        if (b == 0) kk::keccak_f_peeled<true, NB == 1>(A); else kk::keccak_f_peeled<false, true>(A);
    }
    uint4* o = reinterpret_cast<uint4*>(digests + r * 8);
    o[0] = make_uint4(wrap_mod_p(A[0].x), wrap_mod_p(A[0].y), wrap_mod_p(A[1].x), wrap_mod_p(A[1].y));
    o[1] = make_uint4(wrap_mod_p(A[2].x), wrap_mod_p(A[2].y), wrap_mod_p(A[3].x), wrap_mod_p(A[3].y));
}

__device__ __forceinline__ void compress_pair(const uint32_t l[8], const uint32_t r[8], uint32_t out[8]) {
    uint32_t d[8];
    keccak256_words<true>(16, [&](uint32_t i) { return i < 8 ? l[i] : r[i - 8]; }, d);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = wrap_mod_p(d[i]);
}

// next[i] = compress(prev[2i], prev[2i+1]) ; if inject != null: next[i] = compress(next[i], inject[i])
// parents [i0, i0 + n_next) of the layer
__global__ void __launch_bounds__(128) compress_layer_kernel(const uint32_t* __restrict__ prev, const uint32_t* __restrict__ inject, uint64_t i0, uint64_t n_next, uint32_t* __restrict__ next) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_next) return;
    i += i0;
    uint32_t l[8], r[8], o[8];
    const uint4* p = reinterpret_cast<const uint4*>(prev + i * 16);
    uint4 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
    l[0] = a.x; l[1] = a.y; l[2] = a.z; l[3] = a.w; l[4] = b.x; l[5] = b.y; l[6] = b.z; l[7] = b.w;
    r[0] = c.x; r[1] = c.y; r[2] = c.z; r[3] = c.w; r[4] = d.x; r[5] = d.y; r[6] = d.z; r[7] = d.w;
    compress_pair(l, r, o);
    if (inject) {
        const uint4* q = reinterpret_cast<const uint4*>(inject + i * 8);
        uint4 e = __ldg(q), f = __ldg(q + 1);
        uint32_t t[8] = {e.x, e.y, e.z, e.w, f.x, f.y, f.z, f.w};
        uint32_t o2[8];
        compress_pair(o, t, o2);
#pragma unroll
        for (int k = 0; k < 8; k++) o[k] = o2[k];
    }
    uint4* w = reinterpret_cast<uint4*>(next + i * 8);
    w[0] = make_uint4(o[0], o[1], o[2], o[3]);
    w[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

// ---- Keccak-f[1600] spread over the lanes of a warp ------------------------------------------------------------------------------
// For the last few layers of a tree there is nothing to run in parallel: a layer of n <= 32 nodes is n chains of 24 dependent rounds,
// and a lone thread needs ~5.5 us for one (4166 instructions, one warp per scheduler).  Here lane t = x + 5y of a warp holds lane
// A[x, y] of ONE state: a round is 18 shuffles and ~25 ALU instructions per lane (theta: column parity by four shuffles, D by two;
// rho: a per-lane rotation amount; pi: one shuffle; chi: two), ~140 cycles of latency — about a third of the lone thread's chain.
__constant__ uint8_t WK_ROT[25] = {0, 1, 62, 28, 27, 36, 44, 6, 55, 20, 3, 10, 43, 25, 39, 41, 45, 15, 21, 8, 18, 2, 61, 56, 14};   // r[x + 5y]
struct WarpKeccak {
    uint32_t rot, col[4], dm, dp, pi, c1, c2, lane;
    __device__ __forceinline__ void init(uint32_t lane_) {
        lane = lane_;
        const uint32_t t = lane < 25 ? lane : 0, x = t % 5, y = t / 5;
        rot = WK_ROT[t];
#pragma unroll
        for (int k = 0; k < 4; k++) col[k] = (t + 5 * (k + 1)) % 25;
        dm = (x + 4) % 5 + 5 * y; dp = (x + 1) % 5 + 5 * y;
        pi = (x + 3 * y) % 5 + 5 * x;                 // B[x, y] comes from A[(x + 3y) mod 5, x]
        c1 = (x + 1) % 5 + 5 * y; c2 = (x + 2) % 5 + 5 * y;
    }
    static __device__ __forceinline__ uint2 sh(uint2 v, uint32_t src) { return make_uint2(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src)); }
    __device__ __forceinline__ void permute(uint2& a) const {
#pragma unroll 1
        for (int round = 0; round < 24; round++) {
            uint2 p = a;
#pragma unroll
            for (int k = 0; k < 4; k++) { const uint2 o = sh(a, col[k]); p.x ^= o.x; p.y ^= o.y; }
            const uint2 pm = sh(p, dm), pp = sh(p, dp);
            a.x ^= pm.x ^ __funnelshift_l(pp.y, pp.x, 1); a.y ^= pm.y ^ __funnelshift_l(pp.x, pp.y, 1);
            uint32_t lo = a.x, hi = a.y;
            if (rot & 32) { const uint32_t tmp = lo; lo = hi; hi = tmp; }
            uint2 b = make_uint2(__funnelshift_l(hi, lo, rot & 31), __funnelshift_l(lo, hi, rot & 31));
            b = sh(b, pi);
            const uint2 b1 = sh(b, c1), b2 = sh(b, c2);
            a.x = b.x ^ (~b1.x & b2.x); a.y = b.y ^ (~b1.y & b2.y);
            if (lane == 0) { const uint2 rc = kk::RC[round]; a.x ^= rc.x; a.y ^= rc.y; }
            if (lane >= 25) a = make_uint2(0, 0);
        }
    }
    // 64-byte compression: lanes 0..7 hold the sixteen input words (2 each); on return lanes 0..3 hold the digest words, reduced mod p
    __device__ __forceinline__ uint2 compress(uint2 words) const {
        uint2 a = lane < 8 ? words : lane == 8 ? make_uint2(1u, 0u) : lane == 16 ? make_uint2(0u, 0x80000000u) : make_uint2(0u, 0u);
        permute(a);
        return make_uint2(wrap_mod_p(a.x), wrap_mod_p(a.y));
    }
};

// The short layers of a tree in ONE launch: a CTA owns `sub` consecutive nodes of the first fused layer and reduces that sub-tree
// level by level in shared memory (each level is written to its place in global memory as well), so the 10 - 16 launches of a tree's
// tail — each a handful of warps waiting on a single Keccak-f — become one or two.  Levels of more than 32 nodes take a thread per
// node; the narrower ones a WARP per node (WarpKeccak), which shortens the dependent chain that is all that is left there.
// Bases are virtual (+ global node index), as in compress_layer_kernel; inj_v[k] = digests of the rows a shorter matrix group
// contributes at fused level k, or null.
constexpr int TAIL_SUB = 256, TAIL_THREADS = 512, TAIL_MAX_LEVELS = 9, TAIL_WARP_NODES = 32;
struct TailParams {
    const uint32_t* prev_v;
    uint32_t* next_v[TAIL_MAX_LEVELS];
    const uint32_t* inj_v[TAIL_MAX_LEVELS];
    uint64_t first_begin;     // first node of the first fused layer computed by this launch
    uint32_t sub;             // nodes of the first fused layer per CTA (power of two <= TAIL_SUB)
    uint32_t levels;          // fused levels: level k has sub >> k nodes per CTA
};
// at most 80 registers (launched with TAIL_THREADS threads): left to itself ptxas takes 89 on sm_90a
__global__ void __maxnreg__(80) tree_tail_kernel(const __grid_constant__ TailParams p) {
    __shared__ uint4 buf_a[2 * TAIL_SUB * 2];     // children of the current level: 2 * sub digests (two uint4 each)
    __shared__ uint4 buf_b[TAIL_SUB * 2];
    const uint64_t node0 = p.first_begin + (uint64_t)blockIdx.x * p.sub;
    {
        const uint4* src = reinterpret_cast<const uint4*>(p.prev_v + 2 * node0 * 8);
        for (uint32_t i = threadIdx.x; i < 4 * p.sub; i += TAIL_THREADS) buf_a[i] = __ldg(src + i);
    }
    __syncthreads();
    uint4* cur = buf_a; uint4* nxt = buf_b;
    // n halves every level, so the wide levels all come first.  Two loops rather than one branch: the WarpKeccak set-up is then
    // not live across the thread-per-node rounds, which fit in 80 registers only without it.
    uint32_t k = 0;
    for (; k < p.levels && (p.sub >> k) > TAIL_WARP_NODES; k++) {      // a thread per node
        const uint32_t n = p.sub >> k;
        const uint64_t base = node0 >> k;
        for (uint32_t t = threadIdx.x; t < n; t += TAIL_THREADS) {
            const uint4 a = cur[4 * t], b = cur[4 * t + 1], c = cur[4 * t + 2], d = cur[4 * t + 3];
            uint32_t l[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}, r[8] = {c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w}, o[8];
            compress_pair(l, r, o);
            if (p.inj_v[k]) {
                const uint4* q = reinterpret_cast<const uint4*>(p.inj_v[k] + (base + t) * 8);
                const uint4 e = __ldg(q), f = __ldg(q + 1);
                uint32_t tt[8] = {e.x, e.y, e.z, e.w, f.x, f.y, f.z, f.w}, o2[8];
                compress_pair(o, tt, o2);
#pragma unroll
                for (int i = 0; i < 8; i++) o[i] = o2[i];
            }
            const uint4 w0 = make_uint4(o[0], o[1], o[2], o[3]), w1 = make_uint4(o[4], o[5], o[6], o[7]);
            nxt[2 * t] = w0; nxt[2 * t + 1] = w1;
            uint4* g = reinterpret_cast<uint4*>(p.next_v[k] + (base + t) * 8);
            g[0] = w0; g[1] = w1;
        }
        __syncthreads();
        uint4* tmp = cur; cur = nxt; nxt = tmp;
    }
    if (k == p.levels) return;
    const uint32_t lane = threadIdx.x & 31;
    WarpKeccak wk;
    wk.init(lane);
    for (; k < p.levels; k++) {      // a warp per node
        const uint32_t n = p.sub >> k;
        const uint64_t base = node0 >> k;
        for (uint32_t t = threadIdx.x >> 5; t < n; t += TAIL_THREADS / 32) {
            const uint2* in = reinterpret_cast<const uint2*>(cur + 4 * t);         // 16 words = 8 uint2
            uint2 dg = wk.compress(lane < 8 ? in[lane] : make_uint2(0, 0));        // lanes 0..3: the digest
            if (p.inj_v[k]) {
                const uint2* q = reinterpret_cast<const uint2*>(p.inj_v[k] + (base + t) * 8);
                const uint2 w = lane < 4 ? dg : (lane < 8 ? __ldg(q + (lane - 4)) : make_uint2(0, 0));
                dg = wk.compress(w);
            }
            if (lane < 4) {
                reinterpret_cast<uint2*>(nxt + 2 * t)[lane] = dg;
                reinterpret_cast<uint2*>(p.next_v[k] + (base + t) * 8)[lane] = dg;
            }
        }
        __syncthreads();
        uint4* tmp = cur; cur = nxt; nxt = tmp;
    }
}

// FRI commit-phase leaf: the pair (v[2i], v[2i+1]) of ext5 values flattened to 10 base words
// (ExtensionMmcs over a width-2 matrix); v is limb-major: limb l of element e at v[l * cs + e].
__global__ void __launch_bounds__(128) fri_leaf_hash_kernel(const uint32_t* __restrict__ v, uint64_t cs, uint64_t i0, uint64_t npairs, uint32_t* __restrict__ digests) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    i += i0;
    uint32_t w[10];
#pragma unroll
    for (int l = 0; l < 5; l++) {
        uint2 t = __ldg(reinterpret_cast<const uint2*>(v + (uint64_t)l * cs + 2 * i));
        w[l] = bb::from_monty(t.x); w[5 + l] = bb::from_monty(t.y);
    }
    uint32_t d[8];
    keccak256_words<true>(10, [&](uint32_t k) { return w[k]; }, d);
    uint4* o = reinterpret_cast<uint4*>(digests + i * 8);
    o[0] = make_uint4(wrap_mod_p(d[0]), wrap_mod_p(d[1]), wrap_mod_p(d[2]), wrap_mod_p(d[3]));
    o[1] = make_uint4(wrap_mod_p(d[4]), wrap_mod_p(d[5]), wrap_mod_p(d[6]), wrap_mod_p(d[7]));
}

// One tree whose lower paths query_path_kernel rebuilds (merkle.h, VgPathTree).  Input tree: cols[col_at[j] .. col_at[j + 1]) are
// the columns (virtual row bases, as in hash_rows) of the rows hashed at level j — the leaves at j = 0, the rows injected above.
struct PathTree {
    const uint32_t* const* cols;        // null for a FRI tree
    const uint32_t* fri_v;              // FRI tree: the layer's values, limb stride fri_cs
    uint64_t fri_cs;
    uint32_t col_at[VG_TREE_DROP + 1];
    uint32_t levels;                    // rebuilt levels s: the sub-tree has 2^s leaves
};
constexpr int PATH_THREADS = 1 << VG_TREE_DROP;    // a thread per leaf of the largest sub-tree

// A CTA per request: recomputes the 2^s-leaf sub-tree holding the leaf, level by level in shared memory, with the build's sponge
// and compression, and writes the sibling of the leaf's path at every level below s.
__global__ void __launch_bounds__(PATH_THREADS) query_path_kernel(const PathTree* __restrict__ trees, const VgPathReq* __restrict__ reqs, uint32_t* __restrict__ out) {
    __shared__ uint4 buf[2][2 * PATH_THREADS];      // one level's digests (two uint4 each); levels alternate between the halves
    const VgPathReq q = reqs[blockIdx.x];
    const PathTree& T = trees[q.tree];
    const uint32_t s = T.levels, t = threadIdx.x;
    const uint64_t base = q.leaf >> s << s;         // first leaf of the sub-tree
    const uint32_t* const* cols = T.cols;
    if (t < (1u << s)) {
        uint32_t d[8];
        if (cols) {
            const uint64_t r = base + t;
            keccak256_words(T.col_at[1], [&](uint32_t i) { return bb::from_monty(__ldg(cols[i] + r)); }, d);
        } else {   // fri_leaf_hash_kernel's leaf: the pair (v[2i], v[2i+1]) flattened to 10 words
            const uint64_t i = base + t;
            uint32_t w[10];
#pragma unroll
            for (int l = 0; l < 5; l++) {
                const uint2 v = __ldg(reinterpret_cast<const uint2*>(T.fri_v + (uint64_t)l * T.fri_cs + 2 * i));
                w[l] = bb::from_monty(v.x); w[5 + l] = bb::from_monty(v.y);
            }
            keccak256_words<true>(10, [&](uint32_t k) { return w[k]; }, d);
        }
        buf[0][2 * t] = make_uint4(wrap_mod_p(d[0]), wrap_mod_p(d[1]), wrap_mod_p(d[2]), wrap_mod_p(d[3]));
        buf[0][2 * t + 1] = make_uint4(wrap_mod_p(d[4]), wrap_mod_p(d[5]), wrap_mod_p(d[6]), wrap_mod_p(d[7]));
    }
    __syncthreads();
    uint32_t cur = 0;
    for (uint32_t j = 0; j < s; j++) {
        const uint32_t sib = (uint32_t)(((q.leaf >> j) ^ 1) - (base >> j));
        if (t < 2) reinterpret_cast<uint4*>(out + ((uint64_t)q.slot * VG_TREE_DROP + j) * 8)[t] = buf[cur][2 * sib + t];
        if (j + 1 == s) break;
        if (t < (1u << (s - j - 1))) {       // node t of level j + 1
            const uint4 a = buf[cur][4 * t], b = buf[cur][4 * t + 1], c = buf[cur][4 * t + 2], e = buf[cur][4 * t + 3];
            uint32_t l[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}, r[8] = {c.x, c.y, c.z, c.w, e.x, e.y, e.z, e.w}, o[8];
            compress_pair(l, r, o);
            const uint32_t c0 = cols ? T.col_at[j + 1] : 0, nw = cols ? T.col_at[j + 2] - c0 : 0;
            if (nw) {   // node = compress(compress(l, r), hash(rows of the matrices of this level's height))
                const uint64_t row = (base >> (j + 1)) + t;
                uint32_t h[8], o2[8];
                keccak256_words(nw, [&](uint32_t i) { return bb::from_monty(__ldg(cols[c0 + i] + row)); }, h);
#pragma unroll
                for (int k = 0; k < 8; k++) h[k] = wrap_mod_p(h[k]);
                compress_pair(o, h, o2);
#pragma unroll
                for (int k = 0; k < 8; k++) o[k] = o2[k];
            }
            buf[cur ^ 1][2 * t] = make_uint4(o[0], o[1], o[2], o[3]);
            buf[cur ^ 1][2 * t + 1] = make_uint4(o[4], o[5], o[6], o[7]);
        }
        __syncthreads();
        cur ^= 1;
    }
}

// ---- Poseidon-16 MMCS (VGPU_MERKLE_POSEIDON16) --------------------------------------------------------------------------------
// The same trees with FieldMerkleTreeMmcs<_, PaddingFreeSponge<Perm16, 16, 8, 8>, TruncatedPermutation<Perm16, 2, 8, 16>, 8> over
// the challenger's permutation (poseidon.cuh).  Each kernel below mirrors the Keccak kernel above it in indexing, virtual bases,
// shard runs and injection; the permutation runs on Montgomery words, so the leaves absorb the LDE words as stored and only the
// eight digest words are converted to canonical.  Every CTA first copies the 736 constants to shared memory.

// PaddingFreeSponge: state zero; each chunk of 8 words overwrites state[0 .. len) and is followed by one permutation (ceil(n / 8)
// in all, none extra when 8 divides n); the digest is state[0 .. 8)
template <class Fetch>
__device__ __forceinline__ void p16_sponge(const uint32_t nwords, Fetch fetch, const uint32_t* sc, uint32_t out[8]) {
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 16; i++) s[i] = 0;
    for (uint32_t b = 0; b < nwords; b += 8) {
#pragma unroll
        for (int i = 0; i < 8; i++) if (b + i < nwords) s[i] = fetch(b + i);
        p16::permute(s, sc, sc + p16::RC_WORDS);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = bb::from_monty(s[i]);
}
// TruncatedPermutation: permute(l || r)[0 .. 8); digests are canonical in and out
__device__ __forceinline__ void p16_compress(const uint32_t l[8], const uint32_t r[8], const uint32_t* sc, uint32_t out[8]) {
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = bb::to_monty(l[i]); s[8 + i] = bb::to_monty(r[i]); }
    p16::permute(s, sc, sc + p16::RC_WORDS);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = bb::from_monty(s[i]);
}
__device__ __forceinline__ void store_digest(uint32_t* at, const uint32_t d[8]) {
    uint4* o = reinterpret_cast<uint4*>(at);
    o[0] = make_uint4(d[0], d[1], d[2], d[3]);
    o[1] = make_uint4(d[4], d[5], d[6], d[7]);
}
__device__ __forceinline__ void load_digest(const uint32_t* at, uint32_t d[8]) {
    const uint4* q = reinterpret_cast<const uint4*>(at);
    const uint4 e = __ldg(q), f = __ldg(q + 1);
    d[0] = e.x; d[1] = e.y; d[2] = e.z; d[3] = e.w; d[4] = f.x; d[5] = f.y; d[6] = f.z; d[7] = f.w;
}

// word k of FRI leaf i: limb k % 5 of element 2i + k / 5 (v limb-major, limb stride cs)
__device__ __forceinline__ uint32_t fri_word(const uint32_t* __restrict__ v, uint64_t cs, uint64_t i, uint32_t k) {
    return __ldg(v + (uint64_t)(k % 5) * cs + 2 * i + k / 5);
}

// leaf_hash_kernel: a thread per row of [row0, row0 + nrows), the concatenated row read through the column table
__global__ void __launch_bounds__(128) p16_leaf_kernel(const uint32_t* const* __restrict__ colptr, uint32_t nwords, uint64_t row0, uint64_t nrows,
                                                      uint32_t* __restrict__ digests, const uint32_t* __restrict__ consts) {
    __shared__ uint32_t sc[p16::CONST_WORDS];
    p16::load_consts(sc, consts);
    __syncthreads();
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    r += row0;
    uint32_t d[8];
    p16_sponge(nwords, [&](uint32_t i) { return __ldg(colptr[i] + r); }, sc, d);
    store_digest(digests + r * 8, d);
}

// compress_layer_kernel: next[i] = compress(prev[2i], prev[2i+1]), then compress(next[i], inject[i]) when a shorter group joins
__global__ void __launch_bounds__(128) p16_layer_kernel(const uint32_t* __restrict__ prev, const uint32_t* __restrict__ inject, uint64_t i0, uint64_t n_next,
                                                       uint32_t* __restrict__ next, const uint32_t* __restrict__ consts) {
    __shared__ uint32_t sc[p16::CONST_WORDS];
    p16::load_consts(sc, consts);
    __syncthreads();
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_next) return;
    i += i0;
    uint32_t l[8], r[8], o[8];
    load_digest(prev + i * 16, l);
    load_digest(prev + i * 16 + 8, r);
    p16_compress(l, r, sc, o);
    if (inject) {
        load_digest(inject + i * 8, r);
        p16_compress(o, r, sc, l);
#pragma unroll
        for (int k = 0; k < 8; k++) o[k] = l[k];
    }
    store_digest(next + i * 8, o);
}

// tree_tail_kernel's fused short layers (same TailParams, same launch shape), a thread per node on every level
__global__ void __launch_bounds__(TAIL_THREADS) p16_tail_kernel(const __grid_constant__ TailParams p, const uint32_t* __restrict__ consts) {
    __shared__ uint4 buf_a[2 * TAIL_SUB * 2];
    __shared__ uint4 buf_b[TAIL_SUB * 2];
    __shared__ uint32_t sc[p16::CONST_WORDS];
    p16::load_consts(sc, consts);
    const uint64_t node0 = p.first_begin + (uint64_t)blockIdx.x * p.sub;
    {
        const uint4* src = reinterpret_cast<const uint4*>(p.prev_v + 2 * node0 * 8);
        for (uint32_t i = threadIdx.x; i < 4 * p.sub; i += TAIL_THREADS) buf_a[i] = __ldg(src + i);
    }
    __syncthreads();
    uint4* cur = buf_a; uint4* nxt = buf_b;
    for (uint32_t k = 0; k < p.levels; k++) {
        const uint32_t n = p.sub >> k;
        const uint64_t base = node0 >> k;
        for (uint32_t t = threadIdx.x; t < n; t += TAIL_THREADS) {
            const uint4 a = cur[4 * t], b = cur[4 * t + 1], c = cur[4 * t + 2], d = cur[4 * t + 3];
            uint32_t l[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}, r[8] = {c.x, c.y, c.z, c.w, d.x, d.y, d.z, d.w}, o[8];
            p16_compress(l, r, sc, o);
            if (p.inj_v[k]) {
                load_digest(p.inj_v[k] + (base + t) * 8, r);
                p16_compress(o, r, sc, l);
#pragma unroll
                for (int i = 0; i < 8; i++) o[i] = l[i];
            }
            const uint4 w0 = make_uint4(o[0], o[1], o[2], o[3]), w1 = make_uint4(o[4], o[5], o[6], o[7]);
            nxt[2 * t] = w0; nxt[2 * t + 1] = w1;
            uint4* g = reinterpret_cast<uint4*>(p.next_v[k] + (base + t) * 8);
            g[0] = w0; g[1] = w1;
        }
        __syncthreads();
        uint4* tmp = cur; cur = nxt; nxt = tmp;
    }
}

// fri_leaf_hash_kernel: the pair (v[2i], v[2i+1]) of ext5 values flattened to 10 base words, two permutations
__global__ void __launch_bounds__(128) p16_fri_leaf_kernel(const uint32_t* __restrict__ v, uint64_t cs, uint64_t i0, uint64_t npairs, uint32_t* __restrict__ digests,
                                                          const uint32_t* __restrict__ consts) {
    __shared__ uint32_t sc[p16::CONST_WORDS];
    p16::load_consts(sc, consts);
    __syncthreads();
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    i += i0;
    uint32_t d[8];
    p16_sponge(10, [&](uint32_t k) { return fri_word(v, cs, i, k); }, sc, d);
    store_digest(digests + i * 8, d);
}

// query_path_kernel with the Poseidon-16 sponge and compression: a CTA per request rebuilds the 2^s-leaf sub-tree holding the leaf.
// A node of a level is one to ceil(nw / 8) + 2 permutations (compression; the sponge of the injected row and the second compression)
// run by ONE loop around ONE inlined permutation: each inlined copy costs ~2k instructions of registers and code.
__global__ void __launch_bounds__(PATH_THREADS) p16_path_kernel(const PathTree* __restrict__ trees, const VgPathReq* __restrict__ reqs, uint32_t* __restrict__ out,
                                                               const uint32_t* __restrict__ consts) {
    __shared__ uint4 buf[2][2 * PATH_THREADS];
    __shared__ uint32_t sc[p16::CONST_WORDS];
    p16::load_consts(sc, consts);
    const VgPathReq q = reqs[blockIdx.x];
    const PathTree& T = trees[q.tree];
    const uint32_t s = T.levels, t = threadIdx.x;
    const uint64_t base = q.leaf >> s << s;
    const uint32_t* const* cols = T.cols;
    __syncthreads();
    if (t < (1u << s)) {
        uint32_t d[8];
        if (cols) {
            const uint64_t r = base + t;
            p16_sponge(T.col_at[1], [&](uint32_t i) { return __ldg(cols[i] + r); }, sc, d);
        } else {   // p16_fri_leaf_kernel's leaf
            p16_sponge(10, [&](uint32_t k) { return fri_word(T.fri_v, T.fri_cs, base + t, k); }, sc, d);
        }
        buf[0][2 * t] = make_uint4(d[0], d[1], d[2], d[3]);
        buf[0][2 * t + 1] = make_uint4(d[4], d[5], d[6], d[7]);
    }
    __syncthreads();
    uint32_t cur = 0;
    for (uint32_t j = 0; j < s; j++) {
        const uint32_t sib = (uint32_t)(((q.leaf >> j) ^ 1) - (base >> j));
        if (t < 2) reinterpret_cast<uint4*>(out + ((uint64_t)q.slot * VG_TREE_DROP + j) * 8)[t] = buf[cur][2 * sib + t];
        if (j + 1 == s) break;
        if (t < (1u << (s - j - 1))) {       // node t of level j + 1
            const uint32_t c0 = cols ? T.col_at[j + 1] : 0, nw = cols ? T.col_at[j + 2] - c0 : 0;
            const uint64_t row = (base >> (j + 1)) + t;
            const uint32_t chunks = (nw + 7) / 8, steps = nw ? chunks + 2 : 1;
            const uint32_t* kids = reinterpret_cast<const uint32_t*>(&buf[cur][4 * t]);
            uint32_t st[16], o[8];       // o: the first compression's output (Montgomery)
            for (uint32_t k = 0; k < steps; k++) {
                if (k == 0) {                        // compress(left, right)
#pragma unroll
                    for (int i = 0; i < 16; i++) st[i] = bb::to_monty(kids[i]);
                } else if (k <= chunks) {            // sponge of the rows injected at this level
                    if (k == 1) {
#pragma unroll
                        for (int i = 0; i < 16; i++) st[i] = 0;
                    }
                    const uint32_t w0 = (k - 1) * 8;
#pragma unroll
                    for (int i = 0; i < 8; i++) if (w0 + i < nw) st[i] = __ldg(cols[c0 + w0 + i] + row);
                } else {                             // compress(node, row digest)
#pragma unroll
                    for (int i = 0; i < 8; i++) { st[8 + i] = st[i]; st[i] = o[i]; }
                }
                p16::permute(st, sc, sc + p16::RC_WORDS);
                if (k == 0) {
#pragma unroll
                    for (int i = 0; i < 8; i++) o[i] = st[i];
                }
            }
#pragma unroll
            for (int i = 0; i < 8; i++) o[i] = bb::from_monty(st[i]);
            buf[cur ^ 1][2 * t] = make_uint4(o[0], o[1], o[2], o[3]);
            buf[cur ^ 1][2 * t + 1] = make_uint4(o[4], o[5], o[6], o[7]);
        }
        __syncthreads();
        cur ^= 1;
    }
}

}  // namespace

// ---- host side: layer plan, launches --------------------------------------------------------------------------
// Layer plan of a tree over `leaves` leaves (merkle.h): which run of every layer this rank computes and which it keeps.
struct LayerPlan { uint64_t len, cbegin, ccount, sbegin, scount; bool gather; };
static std::vector<LayerPlan> plan_tree(const vgpu_ctx* ctx, uint64_t leaves, bool split) {
    const int G = split ? ctx->comm_size : 1, r = split ? ctx->comm_rank : 0;
    std::vector<LayerPlan> plan;
    for (uint64_t len = leaves; len >= 1; len >>= 1) {
        const VgRun run = vg_layer_run(len, G, r);
        LayerPlan p{};
        p.len = len; p.cbegin = run.begin; p.ccount = run.count;
        // the last split layer (the sub-roots at a power of two G, the V-node layer otherwise), completed by the all-gather
        p.gather = run.split && (len == 1 || !vg_layer_split(len / 2, G));
        if (run.split && !p.gather) { p.sbegin = p.cbegin; p.scount = p.ccount; } else { p.sbegin = 0; p.scount = len; }
        plan.push_back(p);
        if (len == 1) break;
    }
    return plan;
}
// The layers below VG_TREE_DROP (all but the root of a shorter tree) of a tree being built: a transient block, handed back to the
// context's cache when the build returns (the kernels writing and reading it are already enqueued on the context's stream), and
// the tree's pointers into it cleared.
struct LowerLayers {
    VgTree* t; VgBuf d; size_t n = 0;
    ~LowerLayers() { for (size_t i = 0; i < n; i++) t->layer_ptr[i] = nullptr; }
};
static int32_t alloc_tree(vgpu_ctx* ctx, const std::vector<LayerPlan>& plan, VgTree* t, LowerLayers* low) {
    const size_t keep = std::min(plan.size() - 1, VG_TREE_DROP);     // first kept layer
    uint64_t kept = 0, dropped = 0;
    for (size_t i = 0; i < plan.size(); i++) (i < keep ? dropped : kept) += plan[i].scount;
    t->digests = VgBuf(ctx);
    VG_TRY(t->digests.alloc(kept * 32));
    if (dropped) VG_TRY(low->d.alloc(dropped * 32));
    t->layer_ptr.clear(); t->layer_len.clear(); t->layer_begin.clear(); t->layer_count.clear();
    uint32_t* at[2] = {low->d.as<uint32_t>(), t->digests.as<uint32_t>()};
    for (size_t i = 0; i < plan.size(); i++) {
        const LayerPlan& p = plan[i];
        uint32_t*& a = at[i >= keep];
        t->layer_ptr.push_back(a); t->layer_len.push_back(p.len); t->layer_begin.push_back(p.sbegin); t->layer_count.push_back(p.scount);
        a += p.scount * 8;
    }
    low->n = keep;
    return 0;
}

// digest of rows [row0, row0 + nrows) of the concatenated matrices, written to digests_v[row * 8] (digests_v is a VIRTUAL
// base: the stored run starts at its first row).  A row shard contributes its local rows through a base shifted likewise.
// p16: Poseidon-16 sponge (always through a column table in global memory), else Keccak-256.
static int32_t hash_rows(vgpu_ctx* ctx, bool p16, const std::vector<const vgpu_dmat*>& mats, uint64_t row0, uint64_t nrows, uint32_t* digests_v) {
    std::vector<const uint32_t*> cols;
    for (auto* m : mats) {
        if (m->dist == VG_ROWS && (row0 < m->row0 || row0 + nrows > m->row0 + m->h)) VG_FAIL(ctx, "commit: rows [%llu, +%llu) are not in this rank's shard", (unsigned long long)row0, (unsigned long long)nrows);
        for (uint64_t c = 0; c < m->w; c++) cols.push_back(m->d + c * m->col_stride - m->row0);
    }
    const uint32_t nwords = (uint32_t)cols.size(), nblocks = nwords / RATE_WORDS + 1, grid = (uint32_t)((nrows + 127) / 128);
    uint32_t* consts = nullptr;
    if (p16) VG_TRY(vg_poseidon_consts(ctx, &consts));
    if (!p16 && nblocks <= LEAF_NB_MAX) {
        LeafCols lc{};
        std::copy(cols.begin(), cols.end(), lc.col);
        {
            KScope ks(ctx, KC_LEAF_HASH, (double)nrows * (4.0 * nwords + 32.0));
            if (nblocks == 1) leaf_hash_kernel_blocks<1><<<grid, 128, 0, ctx->stream>>>(lc, nwords, row0, nrows, digests_v);
            else leaf_hash_kernel_blocks<2><<<grid, 128, 0, ctx->stream>>>(lc, nwords, row0, nrows, digests_v);
        }
        VG_LAUNCH_CHECK(ctx);
        return 0;
    }
    VgBuf dcols(ctx);
    VG_TRY(dcols.upload(cols.data(), cols.size()));
    {
        KScope ks(ctx, p16 ? KC_P16_LEAF : KC_LEAF_HASH, (double)nrows * (4.0 * nwords + 32.0));
        if (p16) p16_leaf_kernel<<<grid, 128, 0, ctx->stream>>>(dcols.as<const uint32_t*>(), nwords, row0, nrows, digests_v, consts);
        else leaf_hash_kernel<<<grid, 128, 0, ctx->stream>>>(dcols.as<const uint32_t*>(), nwords, row0, nrows, digests_v);
    }
    VG_LAUNCH_CHECK(ctx);
    return 0;
}

// layers 1.. of a planned tree whose leaf layer is already hashed; inject(lvl, plan, inj_v, &have) fills the digests of the rows a
// shorter matrix group contributes at layer lvl.  Long layers take one launch each; from the first layer of at most TAIL_FUSE nodes
// (computed here) on, runs of up to 9 layers go into ONE launch of tree_tail_kernel; a run ends at the sub-root layer of a split tree
// (its all-gather comes next) and at the root.
constexpr uint64_t TAIL_FUSE = 1u << 15;
template <class Inject>
static int32_t build_upper_layers(vgpu_ctx* ctx, const std::vector<LayerPlan>& plan, VgTree* t, uint32_t* inject_buf, Inject inject) {
    const bool p16 = t->hash == VGPU_MERKLE_POSEIDON16;
    uint32_t* consts = nullptr;
    if (p16) VG_TRY(vg_poseidon_consts(ctx, &consts));
    if (plan[0].gather) VG_TRY(vg_comm_allgather_runs(ctx, t->layer_ptr[0], plan[0].len, 8));
    size_t lvl = 1;
    while (lvl < plan.size()) {
        const LayerPlan& p = plan[lvl];
        const uint32_t* prev_v = t->layer_ptr[lvl - 1] - plan[lvl - 1].sbegin * 8;
        if (p.ccount <= TAIL_FUSE) {
            // one launch: levels lvl .. lvl + n - 1, each half the one below; stop after a gather layer and at the root
            TailParams tp{};
            tp.prev_v = prev_v; tp.first_begin = p.cbegin;
            // a CTA's sub-tree starts on a multiple of `sub` nodes: a power of two dividing both ends of the run (an uneven run of
            // units need not start on a multiple of its length)
            tp.sub = (uint32_t)std::min<uint64_t>(TAIL_SUB, (p.cbegin | p.ccount) & (~(p.cbegin | p.ccount) + 1));
            uint32_t n = 0;
            uint32_t* inj_at = inject_buf;
            double bytes = 0;
            while (n < TAIL_MAX_LEVELS && lvl + n < plan.size() && (tp.sub >> n) >= 1) {
                const LayerPlan& q = plan[lvl + n];
                if (q.ccount != (p.ccount >> n) || q.cbegin != (p.cbegin >> n)) break;      // the run of halving layers ends (past a gather layer)
                tp.next_v[n] = t->layer_ptr[lvl + n] - q.sbegin * 8;
                tp.inj_v[n] = nullptr;
                if (inject_buf) {
                    uint32_t* buf_v = inj_at - q.cbegin * 8;
                    bool have = false;
                    VG_TRY(inject(lvl + n, q, buf_v, &have));
                    if (have) { tp.inj_v[n] = buf_v; inj_at += q.ccount * 8; }
                }
                bytes += (double)q.ccount * (tp.inj_v[n] ? 128.0 : 96.0);
                n++;
                if (q.gather) break;
            }
            tp.levels = n;
            {
                KScope ks(ctx, p16 ? KC_P16_COMPRESS : KC_COMPRESS, bytes);
                if (p16) p16_tail_kernel<<<(unsigned)(p.ccount / tp.sub), TAIL_THREADS, 0, ctx->stream>>>(tp, consts);
                else tree_tail_kernel<<<(unsigned)(p.ccount / tp.sub), TAIL_THREADS, 0, ctx->stream>>>(tp);
            }
            VG_LAUNCH_CHECK(ctx);
            lvl += n;
            if (plan[lvl - 1].gather) VG_TRY(vg_comm_allgather_runs(ctx, t->layer_ptr[lvl - 1], plan[lvl - 1].len, 8));
            continue;
        }
        uint32_t* next_v = t->layer_ptr[lvl] - p.sbegin * 8;
        const uint32_t* inj_v = nullptr;
        if (inject_buf) {
            uint32_t* buf_v = inject_buf - p.cbegin * 8;
            bool have = false;
            VG_TRY(inject(lvl, p, buf_v, &have));
            if (have) inj_v = buf_v;
        }
        {
            KScope ks(ctx, p16 ? KC_P16_COMPRESS : KC_COMPRESS, (double)p.ccount * (inj_v ? 128.0 : 96.0));
            if (p16) p16_layer_kernel<<<(unsigned)((p.ccount + 127) / 128), 128, 0, ctx->stream>>>(prev_v, inj_v, p.cbegin, p.ccount, next_v, consts);
            else compress_layer_kernel<<<(unsigned)((p.ccount + 127) / 128), 128, 0, ctx->stream>>>(prev_v, inj_v, p.cbegin, p.ccount, next_v);
        }
        VG_LAUNCH_CHECK(ctx);
        if (p.gather) VG_TRY(vg_comm_allgather_runs(ctx, t->layer_ptr[lvl], p.len, 8));
        lvl++;
    }
    return 0;
}

// Single-matrix tree over ext5 pairs (p3-fri commit phase).
int32_t vg_fri_layer_commit(vgpu_ctx* ctx, const uint32_t* v, uint64_t cs, uint64_t npairs, bool v_is_shard, VgTree* tree, uint32_t root_out[8]) {
    const std::vector<LayerPlan> plan = plan_tree(ctx, npairs, v_is_shard);
    LowerLayers low{tree, VgBuf(ctx)};
    VG_TRY(alloc_tree(ctx, plan, tree, &low));
    tree->hash = ctx->merkle_hash;
    const bool p16 = tree->hash == VGPU_MERKLE_POSEIDON16;
    uint32_t* consts = nullptr;
    if (p16) VG_TRY(vg_poseidon_consts(ctx, &consts));
    const LayerPlan& l0 = plan[0];
    {
        // v holds the pairs of this rank's run when it is a shard (the run IS the computed run), all pairs otherwise
        const uint32_t* v_v = v_is_shard ? v - 2 * l0.cbegin : v;
        KScope ks(ctx, p16 ? KC_P16_FRI_LEAF : KC_FRI_LEAF, (double)l0.ccount * 72.0);
        const unsigned grid = (unsigned)((l0.ccount + 127) / 128);
        if (p16) p16_fri_leaf_kernel<<<grid, 128, 0, ctx->stream>>>(v_v, cs, l0.cbegin, l0.ccount, tree->layer_ptr[0] - l0.sbegin * 8, consts);
        else fri_leaf_hash_kernel<<<grid, 128, 0, ctx->stream>>>(v_v, cs, l0.cbegin, l0.ccount, tree->layer_ptr[0] - l0.sbegin * 8);
    }
    VG_LAUNCH_CHECK(ctx);
    VG_TRY(build_upper_layers(ctx, plan, tree, nullptr, [](size_t, const LayerPlan&, uint32_t*, bool*) { return 0; }));
    VG_CUDA(ctx, cudaMemcpyAsync(root_out, tree->layer_ptr.back(), 32, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

// Build the mixed-height tree over the bit-reversed LDE matrices of `pd` (see merkle.h for `need`).
int32_t vg_merkle_build(vgpu_ctx* ctx, vgpu_prover_data* pd, const std::vector<uint64_t>& heights,
                        const std::function<int32_t(const std::vector<size_t>&)>& need) {
    size_t n = heights.size();
    if (!n) VG_FAIL(ctx, "commit: no matrices");
    std::vector<size_t> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return heights[a] > heights[b]; });
    uint64_t max_h = heights[order[0]];
    if (max_h & (max_h - 1)) VG_FAIL(ctx, "commit: heights must be powers of two");
    pd->max_height = max_h;
    const std::vector<LayerPlan> plan = plan_tree(ctx, max_h, vg_row_run(ctx, max_h).split);
    LowerLayers low{&pd->tree, VgBuf(ctx)};
    VG_TRY(alloc_tree(ctx, plan, &pd->tree, &low));
    pd->tree.hash = ctx->merkle_hash;
    const bool p16 = pd->tree.hash == VGPU_MERKLE_POSEIDON16;
    size_t pos = 0;
    std::vector<size_t> idx;
    std::vector<const vgpu_dmat*> group;
    auto take = [&](uint64_t height) -> int32_t {   // the matrices of that height, extended on demand
        idx.clear(); group.clear();
        while (pos < n && heights[order[pos]] == height) idx.push_back(order[pos++]);
        if (idx.empty()) return 0;
        if (need) VG_TRY(need(idx));
        for (size_t i : idx) {
            if (!pd->ldes[i] || pd->ldes[i]->gh != height) VG_FAIL(ctx, "commit: matrix %zu was not extended to height %llu", i, (unsigned long long)height);
            group.push_back(pd->ldes[i]);
        }
        return 0;
    };
    VG_TRY(take(max_h));
    VG_TRY(hash_rows(ctx, p16, group, plan[0].cbegin, plan[0].ccount, pd->tree.layer_ptr[0] - plan[0].sbegin * 8));
    VgBuf inject_buf(ctx);
    if (pos < n) {
        // one layer's row digests at a time — except inside a fused run of short layers, where the digests of every injecting
        // layer of the run (at most 2 * TAIL_FUSE in all) must coexist
        const uint64_t c1 = plan.size() > 1 ? plan[1].ccount : 1;
        VG_TRY(inject_buf.alloc((c1 <= 2 * TAIL_FUSE ? 2 * c1 : c1) * 32));
    }
    VG_TRY(build_upper_layers(ctx, plan, &pd->tree, inject_buf.as<uint32_t>(), [&](size_t, const LayerPlan& p, uint32_t* buf_v, bool* have) -> int32_t {
        VG_TRY(take(p.len));
        *have = !group.empty();
        if (*have) VG_TRY(hash_rows(ctx, p16, group, p.cbegin, p.ccount, buf_v));
        return 0;
    }));
    inject_buf.reset();
    if (pos != n) VG_FAIL(ctx, "commit: a matrix height does not match any tree layer");
    VG_CUDA(ctx, cudaMemcpyAsync(pd->root, pd->tree.layer_ptr.back(), 32, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

// The lower levels of the requested paths (merkle.h): one upload of the tree table, the column pointers and the requests, one launch.
int32_t vg_tree_paths(vgpu_ctx* ctx, const std::vector<VgPathTree>& trees, const std::vector<VgPathReq>& reqs, size_t slots, VgBuf* out) {
    *out = VgBuf(ctx);
    VG_TRY(out->alloc(slots * VG_TREE_DROP * 32));
    if (reqs.empty()) return 0;
    const bool p16 = trees[0].tree->hash == VGPU_MERKLE_POSEIDON16;
    for (const VgPathTree& t : trees)
        if (t.tree->hash != trees[0].tree->hash) VG_FAIL(ctx, "tree paths: the trees of one request were built with different hashes");
    uint32_t* consts = nullptr;
    if (p16) VG_TRY(vg_poseidon_consts(ctx, &consts));
    std::vector<PathTree> pt(trees.size());
    std::vector<const uint32_t*> cols;
    std::vector<size_t> col_first(trees.size());  // input tree: its first entry of the column table
    std::vector<double> bytes(trees.size());      // per request: the sub-tree's rows read, and the sibling digests written
    for (size_t k = 0; k < trees.size(); k++) {
        const VgPathTree& src = trees[k];
        PathTree& p = pt[k];
        p.levels = (uint32_t)src.tree->rebuilt();
        bytes[k] = 32.0 * p.levels;
        if (!src.pd) {
            p.fri_v = src.fri_v; p.fri_cs = src.fri_cs;
            bytes[k] += 40.0 * (1u << p.levels);
            continue;
        }
        // the columns of level j in the build's order: the matrices of height max_h >> j, in the caller's order
        col_first[k] = cols.size();
        for (uint32_t j = 0; j < p.levels; j++) {
            p.col_at[j] = (uint32_t)(cols.size() - col_first[k]);
            for (const vgpu_dmat* m : src.pd->ldes) {
                if (m->gh != src.pd->max_height >> j) continue;
                for (uint64_t c = 0; c < m->w; c++) cols.push_back(m->d + c * m->col_stride - m->row0);
                bytes[k] += 4.0 * m->w * (double)(1u << (p.levels - j));
            }
        }
        p.col_at[p.levels] = (uint32_t)(cols.size() - col_first[k]);
    }
    // one device block: [trees][requests][column table]
    const size_t tree_b = pt.size() * sizeof(PathTree), req_b = reqs.size() * sizeof(VgPathReq), col_b = cols.size() * sizeof(void*);
    VgBuf blk(ctx);
    VG_TRY(blk.alloc(tree_b + req_b + col_b));
    const uint32_t* const* dcols = reinterpret_cast<const uint32_t* const*>(blk.as<uint8_t>() + tree_b + req_b);
    for (size_t k = 0; k < pt.size(); k++)
        if (trees[k].pd) pt[k].cols = dcols + col_first[k];
    std::vector<uint8_t> host(tree_b + req_b + col_b);
    std::memcpy(host.data(), pt.data(), tree_b);
    std::memcpy(host.data() + tree_b, reqs.data(), req_b);
    std::memcpy(host.data() + tree_b + req_b, cols.data(), col_b);
    // cudaMemcpyAsync from pageable memory stages synchronously: `host` may go once the call returns
    VG_CUDA(ctx, cudaMemcpyAsync(blk.p, host.data(), host.size(), cudaMemcpyHostToDevice, ctx->stream));
    double total = 0;
    for (const VgPathReq& r : reqs) total += bytes[r.tree];
    {
        KScope ks(ctx, p16 ? KC_P16_PATH : KC_TREE_PATH, total);
        const PathTree* dt = blk.as<const PathTree>();
        const VgPathReq* dr = reinterpret_cast<const VgPathReq*>(blk.as<uint8_t>() + tree_b);
        if (p16) p16_path_kernel<<<(unsigned)reqs.size(), PATH_THREADS, 0, ctx->stream>>>(dt, dr, out->as<uint32_t>(), consts);
        else query_path_kernel<<<(unsigned)reqs.size(), PATH_THREADS, 0, ctx->stream>>>(dt, dr, out->as<uint32_t>());
    }
    VG_LAUNCH_CHECK(ctx);
    return 0;
}
