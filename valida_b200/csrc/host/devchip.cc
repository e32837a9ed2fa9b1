#include "../devchip.h"
#include <cstring>

static DevPairCol conv(const vgpu_pair_col& p) {
    DevPairCol d{};
    d.constant = bb::to_monty(p.constant % bb::P);
    d.n_terms = p.n_terms;
    for (uint32_t t = 0; t < p.n_terms && t < VGPU_MAX_TERMS; t++) {
        d.is_prep[t] = p.terms[t].is_preprocessed; d.column[t] = p.terms[t].column; d.weight[t] = bb::to_monty(p.terms[t].weight % bb::P);
    }
    return d;
}

int32_t vg_build_devchip(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const uint32_t ch[15], DevChip* out) {
    if (chip->n_interactions > VGPU_MAX_INTERACTIONS) VG_FAIL(ctx, "chip has too many interactions");
    std::memset(out, 0, sizeof *out);
    out->chip_id = chip->chip_id; out->width = chip->width; out->prep_width = chip->preprocessed_width; out->n_interactions = chip->n_interactions;
    bb::E5 r1, r2;
    for (int i = 0; i < 5; i++) { r1.c[i] = bb::to_monty(ch[5 + i] % bb::P); r2.c[i] = bb::to_monty(ch[10 + i] % bb::P); }
    bb::E5 b = bb::e5_one();
    for (int j = 0; j < VGPU_MAX_FIELDS; j++) { out->betas[j] = b; b = bb::e5_mul(b, r2); }
    for (uint32_t m = 0; m < chip->n_interactions; m++) {
        const vgpu_interaction& it = chip->interactions[m];
        if (it.n_fields > VGPU_MAX_FIELDS) VG_FAIL(ctx, "interaction has too many fields");
        DevInteraction& d = out->interactions[m];
        d.n_fields = it.n_fields;
        for (uint32_t j = 0; j < it.n_fields; j++) d.fields[j] = conv(it.fields[j]);
        d.count = conv(it.count);
        d.is_send = it.is_send;
        d.alpha = bb::e5_pow(r1, it.bus + 1);
    }
    return 0;
}
