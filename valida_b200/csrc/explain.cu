// What a failed constraint reads.  The catalogue of each chip's constraints (vgpu_chip_constraint_cells) comes from the same AIR
// text the kernels evaluate: air::eval_chip runs once per chip on the host with DepBuilder, whose value is the set of main-trace
// cells an expression reads (local and next row, one 128-bit mask each: no chip is wider than 79 columns); operators take the union,
// constants and selectors are empty.  The LogUp constraints' cells follow logup::eval_constraints from the chip description.  So the
// numbering is the one of check_kernel, quotient_kernel and vgpu_check_failures, and cannot drift from it.
// vgpu_explain_failures then reads those cells on given rows: each cell is reported by the rank that holds its row (rank 0 of a
// whole matrix on a split context) and one vg_gather_words (one all-gather, summed) gives every rank the same words.
#include "ctx.h"
#include "devchip.h"
#include "airs.cuh"
#include "open.h"
#include <mutex>
#include <set>
#include <tuple>

namespace {

// the main-trace columns an expression reads on the local row (l) and the next row (n): column c is bit c % 64 of word c / 64
struct Cells {
    uint64_t l[2], n[2];
};
BB_HD Cells operator|(const Cells& a, const Cells& b) { return Cells{{a.l[0] | b.l[0], a.l[1] | b.l[1]}, {a.n[0] | b.n[0], a.n[1] | b.n[1]}}; }
BB_HD Cells operator+(const Cells& a, const Cells& b) { return a | b; }
BB_HD Cells operator-(const Cells& a, const Cells& b) { return a | b; }
BB_HD Cells operator*(const Cells& a, const Cells& b) { return a | b; }

}  // namespace

namespace air {
template <> struct Lift<Cells> { static BB_HD Cells from_monty_word(uint32_t) { return Cells{}; } };
}  // namespace air

namespace {

constexpr uint32_t MAX_WIDTH = 128;

struct AirEntry { const char* section; Cells cells; };

struct DepBuilder {
    using V = Cells;
    V first{}, last{}, trans{};
    const char* sec = "";
    std::vector<AirEntry>* out;
    static V cell(int c, bool next) {
        V v{};
        (next ? v.n : v.l)[c >> 6] |= 1ull << (c & 63);
        return v;
    }
    V L(int c) const { return cell(c, false); }
    V N(int c) const { return cell(c, true); }
    void z(const V& x) { out->push_back({sec, x}); }
    void section(const char* s) { sec = s; }
};

// the assertions of chip i's Air::eval in eval order, each with its section and the cells it reads
const std::vector<AirEntry>& air_entries(uint32_t chip_id) {
    static std::vector<AirEntry> table[VGPU_NUM_CHIPS];
    static std::once_flag once;
    std::call_once(once, [] {
        for (uint32_t i = 0; i < VGPU_NUM_CHIPS; i++) {
            DepBuilder b;
            b.out = &table[i];
            air::with_chip(i, [&](auto c) { air::eval_chip<decltype(c)::value>(b); });
        }
    });
    return table[chip_id];
}

// ---- column names: the layout airs.cuh's comments state, named after the reference's column structs -----------------------------
struct Names {
    std::vector<std::string> v;
    Names& one(const char* n) { v.emplace_back(n); return *this; }
    Names& arr(const char* n, int k) { for (int i = 0; i < k; i++) v.push_back(std::string(n) + "[" + std::to_string(i) + "]"); return *this; }
    Names& arr2(const char* n, int k, int m) {
        for (int i = 0; i < k; i++)
            for (int j = 0; j < m; j++) v.push_back(std::string(n) + "[" + std::to_string(i) + "][" + std::to_string(j) + "]");
        return *this;
    }
};

struct NameTable {
    std::vector<std::string> main[VGPU_NUM_CHIPS], prep[VGPU_NUM_CHIPS];
    std::string perm[VGPU_MAX_INTERACTIONS + 1][5];   // [m][limb]: interaction m's reciprocal; [k][limb] is named at lookup
    std::string running_sum[5];
};

const NameTable& names() {
    static NameTable t;
    static std::once_flag once;
    std::call_once(once, [] {
        auto operands = [](Names& n, const char* pre) {
            for (const char* o : {"a", "b", "c", "d", "e"}) n.v.push_back(std::string(pre) + "operands." + o);
        };
        {   // 0 cpu
            Names n;
            n.one("clk").one("pc").one("fp").one("instruction.opcode");
            operands(n, "instruction.");
            for (const char* f : {"is_bus_op", "is_bus_op_with_mem", "is_imm_op", "is_left_imm_op", "is_load", "is_load_u8", "is_load_s8",
                                  "is_store", "is_store_u8", "is_beq", "is_bne", "is_jal", "is_jalv", "is_imm32", "is_advice", "is_stop", "is_loadfp"})
                n.v.push_back(std::string("opcode_flags.") + f);
            n.one("diff").one("diff_inv").one("not_equal");
            for (int c = 0; c < 3; c++) {
                const std::string ch = "mem_channels[" + std::to_string(c) + "].";
                for (const char* f : {"used", "is_read", "addr"}) n.v.push_back(ch + f);
                n.arr((ch + "value").c_str(), 4);
            }
            n.one("chip_channel.clk_or_zero");
            t.main[0] = n.v;
        }
        t.main[1] = Names().one("multiplicity").v;
        {
            Names p;
            p.one("pc").one("opcode");
            operands(p, "");
            t.prep[1] = p.v;
        }
        t.main[2] = Names().one("addr").arr("value", 4).one("clk").one("is_static_initial").one("is_read").one("is_write").one("diff")
                        .one("diff_inv").one("addr_not_equal").one("counter").one("counter_mult").v;
        t.main[3] = Names().arr("input_1", 4).arr("input_2", 4).arr("carry", 3).arr("output", 4).one("is_real").v;
        t.main[4] = Names().arr("input_1", 4).arr("input_2", 4).arr("borrow", 3).arr("output", 4).one("is_real").v;
        t.main[5] = Names().arr("input_1", 4).arr("input_2", 4).arr("output", 4).one("r").one("s").one("is_mul").one("is_mulhs").one("is_mulhu")
                        .one("counter").v;
        t.main[6] = Names().arr("input_1", 4).arr("input_2", 4).arr("output", 4).one("is_div").one("is_sdiv").v;
        t.main[7] = Names().arr("input_1", 4).arr("input_2", 4).arr("output", 4).arr("bits_2", 8).one("temp_1").arr("power_of_two", 4)
                        .one("is_shl").one("is_shr").one("is_sra").v;
        t.main[8] = Names().arr("input_1", 4).arr("input_2", 4).arr("byte_flag", 4).arr("bits", 9).one("output").one("multiplicity").one("is_lt")
                        .one("is_lte").one("is_slt").one("is_sle").one("diff_inv").arr("top_bits_1", 8).arr("top_bits_2", 8).one("different_signs").v;
        t.main[9] = Names().arr("input_1", 4).arr("input_2", 4).one("diff").one("diff_inv").one("not_equal").one("output").one("is_ne").one("is_eq").v;
        t.main[10] = Names().arr("input_1", 4).arr("input_2", 4).arr2("bits_1", 4, 8).arr2("bits_2", 4, 8).arr("output", 4).one("is_and").one("is_or")
                         .one("is_xor").v;
        t.main[11] = Names().one("clk").one("value").one("is_real").one("diff").one("counter").one("counter_mult").one("opcode").v;
        t.main[12] = Names().one("mult").one("counter").v;
        t.prep[12] = Names().one("counter").v;
        t.main[13] = Names().one("addr").arr("value", 4).one("is_real").v;
        for (int m = 0; m <= VGPU_MAX_INTERACTIONS; m++)
            for (int l = 0; l < 5; l++) t.perm[m][l] = "interactions[" + std::to_string(m) + "].reciprocal[" + std::to_string(l) + "]";
        for (int l = 0; l < 5; l++) t.running_sum[l] = "running_sum[" + std::to_string(l) + "]";
    });
    return t;
}

const char* column_name(const vgpu_chip_desc* chip, int32_t trace, uint32_t column) {
    if (!vg_chip_ok(chip)) return nullptr;
    const NameTable& t = names();
    if (trace == VGPU_TRACE_MAIN || trace == VGPU_TRACE_PREPROCESSED) {
        const std::vector<std::string>& v = trace == VGPU_TRACE_MAIN ? t.main[chip->chip_id] : t.prep[chip->chip_id];
        const uint32_t w = trace == VGPU_TRACE_MAIN ? chip->width : chip->preprocessed_width;
        return column < w && column < v.size() ? v[column].c_str() : nullptr;
    }
    if (trace == VGPU_TRACE_PERMUTATION) {
        const uint32_t k = chip->n_interactions, m = column / 5, l = column % 5;
        if (m > k) return nullptr;
        return m == k ? t.running_sum[l].c_str() : t.perm[m][l].c_str();
    }
    return nullptr;
}

// interaction labels as Python's constraint_label words them; kept for the life of the process
const char* interaction_label(uint32_t m, uint32_t bus, bool send) {
    static std::mutex mu;
    static std::set<std::string> labels;
    char b[96];
    snprintf(b, sizeof b, "interaction %u (bus %u, %s)", m, bus, send ? "send" : "receive");
    std::lock_guard<std::mutex> g(mu);
    return labels.insert(b).first->c_str();
}

void add_pair_col(const vgpu_pair_col& pc, uint32_t next, std::vector<vgpu_cell>* out) {
    for (uint32_t t = 0; t < pc.n_terms && t < VGPU_MAX_TERMS; t++)
        out->push_back({pc.terms[t].is_preprocessed ? (uint32_t)VGPU_TRACE_PREPROCESSED : (uint32_t)VGPU_TRACE_MAIN, next, pc.terms[t].column});
}
void add_element(uint32_t m, uint32_t next, std::vector<vgpu_cell>* out) {
    for (uint32_t l = 0; l < 5; l++) out->push_back({VGPU_TRACE_PERMUTATION, next, 5 * m + l});
}

// Constraint c of the chip: its label and its cells in ascending (trace, next, column) order; false when c is out of range.
bool constraint_cells(const vgpu_chip_desc* chip, uint32_t c, const char** label, std::vector<vgpu_cell>* cells) {
    cells->clear();
    const std::vector<AirEntry>& air = air_entries(chip->chip_id);
    const uint32_t k = chip->n_interactions;
    if (c < air.size()) {
        *label = air[c].section;
        const Cells& s = air[c].cells;
        for (uint32_t next = 0; next < 2; next++)
            for (uint32_t col = 0; col < MAX_WIDTH; col++)
                if (((next ? s.n : s.l)[col >> 6] >> (col & 63)) & 1) cells->push_back({VGPU_TRACE_MAIN, next, col});
    } else if (c < air.size() + k) {        // rlc * phi_m - 1: the fields on the local row, element m
        const uint32_t m = c - (uint32_t)air.size();
        const vgpu_interaction& it = chip->interactions[m];
        *label = interaction_label(m, it.bus, it.is_send != 0);
        for (uint32_t f = 0; f < it.n_fields && f < VGPU_MAX_FIELDS; f++) add_pair_col(it.fields[f], 0, cells);
        add_element(m, 0, cells);
    } else if (c < air.size() + k + 3) {
        const uint32_t which = c - (uint32_t)air.size() - k;
        static const char* const logup[3] = {"LogUp transition", "LogUp first row", "LogUp last row"};
        *label = logup[which];
        add_element(k, 0, cells);                                   // the running sum on the local row
        if (which == 0) {                                           // phi_next - phi_local - sum of +-phi_m * count on the next row
            add_element(k, 1, cells);
            for (uint32_t m = 0; m < k; m++) { add_element(m, 1, cells); add_pair_col(chip->interactions[m].count, 1, cells); }
        } else if (which == 1) {                                    // phi_local - sum of +-phi_m * count on the local row
            for (uint32_t m = 0; m < k; m++) { add_element(m, 0, cells); add_pair_col(chip->interactions[m].count, 0, cells); }
        }                                                           // last row: phi_local - the cumulative sum, the same cell
    } else {
        return false;
    }
    auto key = [](const vgpu_cell& x) { return std::make_tuple(x.trace, x.next, x.column); };
    std::sort(cells->begin(), cells->end(), [&](const vgpu_cell& a, const vgpu_cell& b) { return key(a) < key(b); });
    cells->erase(std::unique(cells->begin(), cells->end(), [&](const vgpu_cell& a, const vgpu_cell& b) { return key(a) == key(b); }), cells->end());
    return true;
}

}  // namespace

void vg_air_reads(uint32_t chip_id, uint64_t local[2], uint64_t next[2]) {
    Cells u{};
    for (const AirEntry& e : air_entries(chip_id)) u = u | e.cells;
    for (int w = 0; w < 2; w++) { local[w] = u.l[w]; next[w] = u.n[w]; }
}

extern "C" const char* vgpu_chip_column_name(const vgpu_chip_desc* chip, int32_t trace, uint32_t column) {
    return column_name(chip, trace, column);
}

extern "C" int32_t vgpu_chip_constraint_cells(const vgpu_chip_desc* chip, uint32_t constraint, const char** label, vgpu_cell* cells,
                                              uint32_t cap, uint32_t* n) {
    if (!vg_chip_ok(chip) || !label || !n || (cap && !cells)) return -1;
    std::vector<vgpu_cell> v;
    if (!constraint_cells(chip, constraint, label, &v)) return -1;
    for (uint32_t i = 0; i < v.size() && i < cap; i++) cells[i] = v[i];
    *n = (uint32_t)v.size();
    return 0;
}

extern "C" int32_t vgpu_explain_failures(vgpu_ctx* ctx, const vgpu_chip_desc* chip, const vgpu_dmat* main, const vgpu_dmat* prep_or_null,
                                         const vgpu_dmat* perm_or_null, const vgpu_check_failure* items, uint64_t n, uint64_t* first,
                                         uint32_t* values, uint64_t cap, uint64_t* n_values) {
    if (!n_values || (n && (!items || !first || !values))) VG_FAIL(ctx, "explain_failures: null output");
    if (!chip || !main) VG_FAIL(ctx, "explain_failures: null argument");
    if (chip->n_interactions > VGPU_MAX_INTERACTIONS) VG_FAIL(ctx, "explain_failures: %u interactions exceed %d", chip->n_interactions, VGPU_MAX_INTERACTIONS);
    VG_TRY(vg_check_shapes(ctx, chip, main, prep_or_null, perm_or_null, true));
    const uint64_t h = main->gh;
    const uint32_t total = vg_chip_constraints(chip);
    // every item's cells, in catalogue order; refused alike on every rank (the list and the global shapes only)
    std::vector<std::vector<vgpu_cell>> cat(total);
    std::vector<bool> have(total, false);
    uint64_t need = 0;
    for (uint64_t i = 0; i < n; i++) {
        const vgpu_check_failure& it = items[i];
        if (it.row < 0 || (uint64_t)it.row >= h)
            VG_FAIL(ctx, "explain_failures: item %llu: row %lld is outside the trace of height %llu", (unsigned long long)i, (long long)it.row,
                    (unsigned long long)h);
        if (it.constraint >= total)
            VG_FAIL(ctx, "explain_failures: item %llu: constraint %u is not below the chip's %u constraints", (unsigned long long)i, it.constraint, total);
        if (!have[it.constraint]) {
            const char* label;
            constraint_cells(chip, it.constraint, &label, &cat[it.constraint]);
            have[it.constraint] = true;
        }
        need += cat[it.constraint].size();
    }
    if (cap < need)
        VG_FAIL(ctx, "explain_failures: the items read %llu cells, more than cap = %llu", (unsigned long long)need, (unsigned long long)cap);
    if (first) first[0] = 0;
    *n_values = need;
    if (!n) return 0;
    VG_TRY(vg_enter(ctx));
    for (const vgpu_dmat* m : {main, prep_or_null, perm_or_null}) VG_TRY(vg_dmat_materialize(ctx, m));
    // the word behind each cell this rank holds (null: another rank's, or no permutation trace); slot[j]: its place in the gather
    const vgpu_dmat* mats[3] = {main, prep_or_null, perm_or_null};
    std::vector<const uint32_t*> ptrs;
    std::vector<uint64_t> slot(need);
    uint64_t j = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t row = (uint64_t)items[i].row;
        for (const vgpu_cell& c : cat[items[i].constraint]) {
            const vgpu_dmat* m = mats[c.trace];
            if (!m) { slot[j++] = ~0ull; continue; }
            slot[j++] = ptrs.size();
            ptrs.push_back(vg_reported_word(ctx, m, c.next ? (row + 1) % h : row, c.column));
        }
        first[i + 1] = j;
    }
    std::vector<uint32_t> words;
    VG_TRY(vg_gather_words(ctx, ptrs, &words));
    for (uint64_t v = 0; v < need; v++) values[v] = slot[v] == ~0ull ? VGPU_CELL_ABSENT : bb::from_monty(words[slot[v]]);
    return 0;
}
