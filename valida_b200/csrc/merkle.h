// <ValMmcs as Mmcs>::ProverData, device resident: committed (bit-reversed) LDE matrices in the
// caller's order + the digest layers (canonical words, 8 per node).
// Split proof: a layer is cut into the ranks' runs of the row rule (ctx.h) while every run is a whole number of nodes, and a rank
// computes and KEEPS only its run (its sub-tree); the last such layer is all-gathered (the only collective of a tree) and the layers
// above it are computed by every rank.  That is the layer of comm_size sub-roots at a power-of-two comm_size, and the layer of
// V = 8 P nodes, a run of whole units per rank, otherwise.
// A tree keeps only its layers VG_TREE_DROP and up (only the root for a tree of depth VG_TREE_DROP or less): a query's path below
// them is rebuilt from the leaves by vg_tree_paths.  The lower layers are the bulk of a tree (2^-VG_TREE_DROP of it is kept), and
// a proof reads 40 paths from them.
#pragma once
#include "ctx.h"
#include <algorithm>
#include <functional>

// 8: the kept layers are 1/256 of a tree, and a rebuilt path recomputes a 256-leaf sub-tree, one CTA of 256 threads with a thread per
// leaf.  It must not exceed 8: a unit of a split tree's leaves has at least 256 leaves (a FRI layer of 512 values per unit, in pairs),
// so every dropped node lies inside one rank's run, and the layer that is all-gathered is never dropped.
constexpr size_t VG_TREE_DROP = 8;

struct VgTree {
    int32_t hash = VGPU_MERKLE_KECCAK256;  // the hash it was built with (vgpu_ctx_set_merkle_hash)
    VgBuf digests;                         // the stored parts of the kept layers
    std::vector<uint32_t*> layer_ptr;      // layer_ptr[i] -> node layer_begin[i] of layer i; null for a dropped layer
    std::vector<uint64_t> layer_len;       // nodes of the whole layer
    std::vector<uint64_t> layer_begin, layer_count;   // the run of nodes computed on this rank (and stored, if the layer is kept)
    size_t depth() const { return layer_len.size() - 1; }
    // the levels of an authentication path that are not stored: vg_tree_paths rebuilds them
    size_t rebuilt() const { return std::min(depth(), VG_TREE_DROP); }
    // whether THIS rank is the one that reports node `j` of layer `lvl` in a query answer (the owner of a split layer's run;
    // vg_reports_replicated for the layers every rank holds)
    bool reports(const vgpu_ctx* ctx, size_t lvl, uint64_t j) const {
        if (layer_count[lvl] == layer_len[lvl]) return vg_reports_replicated(ctx);
        return j >= layer_begin[lvl] && j < layer_begin[lvl] + layer_count[lvl];
    }
    // address of node `j` of a kept layer `lvl` if this rank reports it, else null
    const uint32_t* node(const vgpu_ctx* ctx, size_t lvl, uint64_t j) const {
        return reports(ctx, lvl, j) ? layer_ptr[lvl] + (j - layer_begin[lvl]) * 8 : nullptr;
    }
};

struct vgpu_prover_data {
    vgpu_ctx* ctx = nullptr;
    std::vector<vgpu_dmat*> ldes;          // owned; VG_ROWS shards for the tall matrices of a split proof
    VgTree tree;
    uint64_t max_height = 0;
    uint32_t root[8] = {0};
};

// heights[i] = height of committed matrix i.  `need(group)` is called with the indices of one height group right before
// its rows are hashed and must fill pd->ldes[i] (the commit extends a matrix only when the tree reaches its height, so
// that uploads of shorter matrices and hashing of taller ones overlap); null = every pd->ldes[i] is already there.
int32_t vg_merkle_build(vgpu_ctx* ctx, vgpu_prover_data* pd, const std::vector<uint64_t>& heights,
                        const std::function<int32_t(const std::vector<size_t>&)>& need);
// Tree over the sibling pairs of an ext5 vector (p3-fri commit phase).  v: limb-major, limb stride cs, holding pairs
// [pair0, pair0 + local_pairs) of the npairs of the layer (all of them, or this rank's run).  The root arrives in root_out
// once the context's stream has been synchronised (the caller needs it for the transcript anyway).
int32_t vg_fri_layer_commit(vgpu_ctx* ctx, const uint32_t* v, uint64_t cs, uint64_t npairs, bool v_is_shard, VgTree* tree, uint32_t root_out[8]);

// The leaves of a tree whose lower paths vg_tree_paths rebuilds: the rows of pd->ldes (an input tree, pd->tree), or the ext5
// pairs of a FRI layer's values (fri_v: limb-major, limb stride fri_cs, addressed by the layer's global element index).
struct VgPathTree { const VgTree* tree; const vgpu_prover_data* pd; const uint32_t* fri_v; uint64_t fri_cs; };
struct VgPathReq { uint32_t tree, slot; uint64_t leaf; };
// Enqueues ONE launch that writes, for every request, the sibling digests of levels 0 .. rebuilt() - 1 of leaf `leaf`'s path to
// out[(slot * VG_TREE_DROP + lvl) * 8 ..]; out receives a block of `slots` * VG_TREE_DROP digests.  Every requested leaf must be
// one this rank reports (VgTree::reports at layer 0).
int32_t vg_tree_paths(vgpu_ctx* ctx, const std::vector<VgPathTree>& trees, const std::vector<VgPathReq>& reqs, size_t slots, VgBuf* out);
