// Device transcription of the 14 BasicMachine AIRs (Air::eval of each chip), written against a
// minimal builder concept so the same text serves the fused quotient sweep on the device and a
// host-side constraint counter:
//     B::V                   value type: F (base field, prover sweep / counting) or X (extension, verifier at zeta)
//     B::L(c) / B::N(c)      main-trace cell of the local / next row (column c)
//     b.first/last/trans     selector values (is_first_row, is_last_row, is_transition)
//     b.z(x)                 AirBuilder::assert_zero(x)
//     b.section(name)        names the block of the reference's eval that the assertions after it transcribe (a no-op for
//                            every builder but the host catalogue's, explain.cu)
// Filters (`when`, `when_ne`, `when_transition`, ...) are multiplied in explicitly, which is what
// p3-air's FilteredAirBuilder lowers to.  Constraint ORDER is part of the result (alpha-folding,
// machine/src/folding_builder.rs:62-66) and follows each eval() line by line.
// Sources: cpu/src/stark.rs:22-305, alu_u32/src/{add,sub,mul,shift,lt,com,bitwise}/stark.rs,
// output/src/stark.rs:21-39, static_data/src/stark.rs:25-37; memory/range/program/div are empty.
#pragma once
#include <type_traits>
#include "../../include/valida_b200.h"
#include "bb.cuh"

namespace air {

struct F {
    uint32_t v;   // Montgomery
};
BB_HD F operator+(F a, F b) { return F{bb::add(a.v, b.v)}; }
BB_HD F operator-(F a, F b) { return F{bb::sub(a.v, b.v)}; }
BB_HD F operator*(F a, F b) { return F{bb::mul(a.v, b.v)}; }
// extension-field value (verifier folder: every trace cell is an opened value in the degree-5 extension)
struct X {
    bb::E5 e;
};
BB_HD X operator+(const X& a, const X& b) { return X{bb::e5_add(a.e, b.e)}; }
BB_HD X operator-(const X& a, const X& b) { return X{bb::e5_sub(a.e, b.e)}; }
BB_HD X operator*(const X& a, const X& b) { return X{bb::e5_mul(a.e, b.e)}; }
// compile-time Montgomery constant
constexpr uint32_t cmont(uint64_t x) { return (uint32_t)(((x % bb::P) << 32) % bb::P); }
template <class V> struct Lift;
template <> struct Lift<F> { static BB_HD F from_monty_word(uint32_t m) { return F{m}; } };
template <> struct Lift<X> { static BB_HD X from_monty_word(uint32_t m) { return X{bb::e5_from_base(m)}; } };
template <class V, uint32_t C> BB_HD V K() { return Lift<V>::from_monty_word(cmont(C)); }
template <class V> BB_HD V ONE() { return Lift<V>::from_monty_word(bb::R1); }
template <class V> BB_HD V ZERO() { return Lift<V>::from_monty_word(0); }

// helpers shared by several chips
template <class B> BB_HD typename B::V word_be(const B& b, bool next, int c0) {
    using V = typename B::V;   // Word::reduce: sum base[i]*w[i], base = (2^24, 2^16, 2^8, 1)
    auto at = [&](int c) { return next ? b.N(c) : b.L(c); };
    return K<V, 1u << 24>() * at(c0) + K<V, 1u << 16>() * at(c0 + 1) + K<V, 1u << 8>() * at(c0 + 2) + at(c0 + 3);
}
template <class B> BB_HD typename B::V sqdiff4(const B& b, int a0, int b0) {
    using V = typename B::V;
    V s = ZERO<V>();
    for (int i = 0; i < 4; i++) { V d = b.L(a0 + i) - b.L(b0 + i); s = s + d * d; }
    return s;
}

// ---- 0: CpuChip (cpu/src/stark.rs) --------------------------------------------------------------
// columns: clk 0, pc 1, fp 2, opcode 3, operands a..e 4..8, flags 9..25 (is_bus_op 9, is_bus_op_with_mem 10,
// is_imm_op 11, is_left_imm_op 12, is_load 13, is_load_u8 14, is_load_s8 15, is_store 16, is_store_u8 17, is_beq 18,
// is_bne 19, is_jal 20, is_jalv 21, is_imm32 22, is_advice 23, is_stop 24, is_loadfp 25), diff 26, diff_inv 27,
// not_equal 28, mem channel c at 29+7c: used, is_read, addr, value[4]; chip_channel.clk_or_zero 50.
template <class B> BB_HD void eval_cpu(B& b) {
    using V = typename B::V;
    const V one = ONE<V>();
    const V bpi = K<V, 24>();
    const V clk = b.L(0), pc = b.L(1), fp = b.L(2);
    const V opa = b.L(4), opb = b.L(5), opc = b.L(6);
    const V is_bus = b.L(9), is_bus_mem = b.L(10), is_imm = b.L(11), is_limm = b.L(12), is_load = b.L(13), is_store = b.L(16);
    const V is_beq = b.L(18), is_bne = b.L(19), is_jal = b.L(20), is_jalv = b.L(21), is_imm32 = b.L(22), is_advice = b.L(23), is_stop = b.L(24), is_loadfp = b.L(25);
    const V diff = b.L(26), diff_inv = b.L(27), not_equal = b.L(28);
    const int R1V = 32, R2V = 39, WV = 46;   // value words of read-1, read-2, write channels
    const V r1_used = b.L(29), r1_addr = b.L(31), r2_used = b.L(36), r2_addr = b.L(38), w_used = b.L(43), w_addr = b.L(45);
    const V tr = b.trans;
    const V rv1 = word_be(b, false, R1V), rv2 = word_be(b, false, R2V), wv = word_be(b, false, WV);
    const V npc = b.N(1), nfp = b.N(2);

    b.section("CpuChip::eval_pc");
    const V inc_pc = pc + one;
    b.z(tr * (is_imm32 + is_loadfp + is_bus + is_advice) * (npc - inc_pc));
    const V equal = one - not_equal;
    b.z(tr * is_beq * (bpi * npc - (equal * opa + bpi * not_equal * inc_pc)));
    b.z(tr * is_bne * (bpi * npc - (bpi * equal * inc_pc + not_equal * opa)));
    b.z(tr * is_jal * (bpi * npc - opb));
    b.z(tr * is_jalv * (bpi * npc - rv1));
    b.section("CpuChip::eval_fp");
    b.z(tr * is_jal * (nfp - (fp + opc)));
    b.z(tr * is_jalv * (nfp - (fp + rv2)));
    b.z(tr * (one - is_jal - is_jalv) * (nfp - fp));
    b.section("CpuChip::eval_equality");
    b.z(diff - sqdiff4(b, R1V, R2V));
    b.z(not_equal * (not_equal - one));
    b.z(not_equal - diff * diff_inv);
    b.z((one - not_equal) * diff);
    b.section("CpuChip::eval_memory_channels");
    b.z(is_load * (is_load - one)); b.z(is_store * (is_store - one)); b.z(is_jal * (is_jal - one)); b.z(is_jalv * (is_jalv - one));
    b.z(is_beq * (is_beq - one)); b.z(is_bne * (is_bne - one)); b.z(is_imm32 * (is_imm32 - one)); b.z(is_loadfp * (is_loadfp - one));
    b.z(is_imm * (is_imm - one)); b.z(is_limm * (is_limm - one)); b.z(is_bus * (is_bus - one));
    const V addr_a = fp + opa, addr_b = fp + opb, addr_c = fp + opc;
    b.z(b.L(30) - one);
    b.z(b.L(37) - one);
    b.z(b.L(44));
    // read (1)
    b.z((is_jalv + is_beq + is_bne + is_bus * (one - is_limm)) * (r1_addr - addr_b));
    b.z((is_load + is_store) * (r1_addr - addr_c));
    b.z((is_load + is_store + is_jalv + is_beq + is_bne + (one - is_limm) * is_bus) * (r1_used - one));
    b.z((is_jal + is_limm + is_loadfp + is_imm32) * r1_used);
    // read (2)
    b.z(is_load * (r2_addr - rv1));
    b.z(is_store * (r2_addr - addr_b));
    b.z((is_jalv + (one - is_imm) * is_bus) * (r2_addr - addr_c));
    b.z((is_load + is_store + is_jalv + (one - is_imm) * (is_beq + is_bne + is_bus)) * (r2_used - one));
    b.z((is_jal + is_imm * (is_beq + is_bne + is_bus) + is_loadfp + is_imm32) * r2_used);
    // write
    b.z((is_load + is_jal + is_jalv + is_imm32 + is_bus + is_loadfp) * (w_addr - addr_a));
    b.z(is_store * (w_addr - rv2));
    b.z(is_store * sqdiff4(b, R1V, WV));
    b.z(is_load * sqdiff4(b, R2V, WV));
    b.z(tr * (is_jal + is_jalv) * (bpi * (pc + one) - wv));
    b.z(is_imm32 * sqdiff4(b, WV, 5));      // write value vs operands.imm32() = (b, c, d, e)
    b.z(is_loadfp * (addr_b - wv));
    b.z((is_store + is_load + is_jal + is_jalv + is_imm32 + is_loadfp + is_bus) * (w_used - one));
    b.z((is_beq + is_bne) * w_used);
    b.section("CpuChip::eval clock");
    b.z(b.first * clk);
    b.z(tr * (clk + one - b.N(0)));
    b.z(is_bus_mem * (clk - b.L(50)));
    b.z((one - is_bus_mem) * b.L(50));
    b.section("CpuChip::eval immediates");
    b.z((is_imm + is_limm) * (is_imm + is_limm - one));
    b.z(is_imm * (opc - rv2));
    b.z(is_limm * (opb - rv1));
    b.section("CpuChip::eval stop");
    b.z(tr * is_stop * (npc - pc));
    b.z(b.last * (is_stop - one));
}

// ---- 3: Add32Chip — input_1 0..3, input_2 4..7, carry 8..10, output 11..14, is_real 15 -------------
template <class B> BB_HD void eval_add(B& b) {
    using V = typename B::V;
    const V one = ONE<V>(), base = K<V, 256>();
    const V c1 = b.L(8), c2 = b.L(9), c3 = b.L(10);
    const V o0 = b.L(3) + b.L(7) - b.L(14);
    const V o1 = b.L(2) + b.L(6) - b.L(13) + c1;
    const V o2 = b.L(1) + b.L(5) - b.L(12) + c2;
    const V o3 = b.L(0) + b.L(4) - b.L(11) + c3;
    b.section("Add32Chip::eval limbs");
    b.z(o0 * (o0 - base)); b.z(o1 * (o1 - base)); b.z(o2 * (o2 - base)); b.z(o3 * (o3 - base));
    b.section("Add32Chip::eval carries");
    b.z(o0 * (c1 - one) + (o0 - base) * c1);
    b.z(o1 * (c2 - one) + (o1 - base) * c2);
    b.z(o2 * (c3 - one) + (o2 - base) * c3);
    b.z(c1 * (c1 - one)); b.z(c2 * (c2 - one)); b.z(c3 * (c3 - one));
}

// ---- 4: Sub32Chip — same layout with borrow 8..10 --------------------------------------------------
template <class B> BB_HD void eval_sub(B& b) {
    using V = typename B::V;
    const V one = ONE<V>(), base = K<V, 256>();
    const V w1 = b.L(8), w2 = b.L(9), w3 = b.L(10);
    b.section("Sub32Chip::eval");
    b.z(b.L(14) - (base * w1 + b.L(3) - b.L(7)));
    b.z(b.L(13) - (base * w2 + b.L(2) - b.L(6) - w1));
    b.z(b.L(12) - (base * w3 + b.L(1) - b.L(5) - w2));
    b.z(b.L(11) - (b.L(0) - b.L(4) - w3));
    b.z(w1 * (w1 - one)); b.z(w2 * (w2 - one)); b.z(w3 * (w3 - one));
}

// ---- 5: Mul32Chip — input_1 0..3, input_2 4..7, output 8..11, r 12, s 13, flags 14..16, counter 17 ---
template <class B> BB_HD void eval_mul(B& b) {
    using V = typename B::V;
    const V wgt[4] = {ONE<V>(), K<V, 1u << 8>(), K<V, 1u << 16>(), K<V, 1u << 24>()};
    V pi4 = ZERO<V>(), pi2 = ZERO<V>(), sg4 = ZERO<V>(), sg2 = ZERO<V>();
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            if (i + j < 4) pi4 = pi4 + wgt[i + j] * b.L(3 - i) * b.L(7 - j);
            if (i < 2 && j < 2 && i + j < 2) pi2 = pi2 + wgt[i + j] * b.L(3 - i) * b.L(7 - j);
        }
    for (int i = 0; i < 4; i++) { sg4 = sg4 + wgt[i] * b.L(11 - i); if (i < 2) sg2 = sg2 + wgt[i] * b.L(11 - i); }
    b.section("Mul32Chip::eval congruences");
    b.z(pi4 - sg4 - b.L(12) * K<V, 2>());
    b.z(pi2 - sg2 - b.L(13) * wgt[2]);
    b.section("Mul32Chip::eval counter");
    b.z(b.first * (b.L(17) - ONE<V>()));
    const V cd = b.N(17) - b.L(17);
    b.z(b.trans * (cd * (cd - ONE<V>())));
    b.z(b.last * (b.L(17) - K<V, 1024>()));
}

// ---- 7: Shift32Chip — input_1 0..3, input_2 4..7, output 8..11, bits_2 12..19, temp_1 20, power_of_two 21..24, is_shl 25, is_shr 26, is_sra 27
template <class B> BB_HD void eval_shift(B& b) {
    using V = typename B::V;
    const V one = ONE<V>();
    V byte2 = ZERO<V>();
    const V p2[8] = {K<V, 1>(), K<V, 2>(), K<V, 4>(), K<V, 8>(), K<V, 16>(), K<V, 32>(), K<V, 64>(), K<V, 128>()};
    for (int i = 0; i < 8; i++) byte2 = byte2 + b.L(12 + i) * p2[i];
    b.section("Shift32Chip::eval bits_2");
    b.z(b.L(7) - byte2);
    for (int i = 0; i < 8; i++) { V t = b.L(12 + i); b.z(t * (t - one)); }
    b.section("Shift32Chip::eval power_of_two");
    const V t1 = (b.L(12) * K<V, 2>()) * (b.L(13) * K<V, 4>()) * (b.L(14) * K<V, 16>());
    b.z(b.L(20) - t1);
    const V b3 = b.L(15), b4 = b.L(16), tmp = b.L(20);
    b.z(b.L(21) - tmp * (one - b3) * (one - b4));
    b.z(b.L(22) - tmp * b3 * (one - b4));
    b.z(b.L(23) - tmp * (one - b3) * b4);
    b.z(b.L(24) - tmp * b3 * b4);
    const V shl = b.L(25), shr = b.L(26), sra = b.L(27);
    b.section("Shift32Chip::eval opcode flags");
    b.z(shl * (shl - one)); b.z(shr * (shr - one)); b.z(sra * (sra - one));
    const V s = shl + shr + sra;
    b.z(s * (s - one));
}

// ---- 8: Lt32Chip — input_1 0..3, input_2 4..7, byte_flag 8..11, bits 12..20, output 21, multiplicity 22,
//         is_lt 23, is_lte 24, is_slt 25, is_sle 26, diff_inv 27, top_bits_1 28..35, top_bits_2 36..43, different_signs 44
template <class B> BB_HD void eval_lt(B& b) {
    using V = typename B::V;
    const V one = ONE<V>();
    const V p2[9] = {K<V, 1>(), K<V, 2>(), K<V, 4>(), K<V, 8>(), K<V, 16>(), K<V, 32>(), K<V, 64>(), K<V, 128>(), K<V, 256>()};
    V bit_comp = ZERO<V>();
    for (int i = 0; i < 9; i++) bit_comp = bit_comp + b.L(12 + i) * p2[i];
    const V f0 = b.L(8), f1 = b.L(9), f2 = b.L(10), f3 = b.L(11);
    const V flag_sum = f0 + f1 + f2 + f3;
    b.section("Lt32Chip::eval byte_flag");
    b.z(flag_sum * (flag_sum - one));
    b.z((f0 - one) * (b.L(0) - b.L(4)));
    b.z((f0 + f1 - one) * (b.L(1) - b.L(5)));
    b.z((f0 + f1 + f2 - one) * (b.L(2) - b.L(6)));
    b.z((flag_sum - one) * (b.L(3) - b.L(7)));
    b.z((flag_sum - one) * bit_comp);
    for (int i = 0; i < 4; i++) {
        const V fl = b.L(8 + i);
        b.z(fl * (K<V, 256>() + b.L(i) - b.L(4 + i) - bit_comp));
        b.z(fl * ((b.L(i) - b.L(4 + i)) * b.L(27) - one));
        b.z(fl * (fl - one));
    }
    V top1 = ZERO<V>(), top2 = ZERO<V>();
    b.section("Lt32Chip::eval top bits");
    for (int i = 0; i < 8; i++) { top1 = top1 + b.L(28 + i) * p2[i]; top2 = top2 + b.L(36 + i) * p2[i]; }
    b.z(top1 - b.L(0));
    b.z(top2 - b.L(4));
    const V is_lt = b.L(23), is_lte = b.L(24), is_slt = b.L(25), is_sle = b.L(26), ds = b.L(44), out = b.L(21), bit8 = b.L(20);
    const V is_signed = is_slt + is_sle, is_unsigned = one - is_signed, same_sign = one - ds, are_equal = one - flag_sum;
    b.section("Lt32Chip::eval different_signs");
    b.z(is_unsigned * ds);
    b.z(is_signed * (b.L(35) - b.L(43)) * (ds - one));
    b.z(ds * (f0 - one));
    b.z(ds * (b.L(35) + b.L(43) - one));
    b.section("Lt32Chip::eval opcode flags");
    b.z(is_lt * (is_lt - one)); b.z(is_lte * (is_lte - one)); b.z(is_slt * (is_slt - one)); b.z(is_sle * (is_sle - one));
    const V opsum = is_lt + is_lte + is_slt + is_sle;
    b.z(opsum * (opsum - one));
    b.section("Lt32Chip::eval output");
    b.z(bit8 * (is_unsigned + same_sign) * out);
    b.z(bit8 * ds * (out - one));
    b.z((bit8 + are_equal - one) * (is_unsigned + same_sign) * (out - one));
    b.z((bit8 + are_equal - one) * ds * out);
    b.z(are_equal * (is_lte + is_sle) * (out - one));
    b.z(are_equal * (is_lt + is_slt) * out);
    b.section("Lt32Chip::eval bits booleans");
    for (int i = 0; i < 9; i++) { V t = b.L(12 + i); b.z(t * (t - one)); }
    for (int i = 0; i < 8; i++) { V t = b.L(28 + i); b.z(t * (t - one)); }
    for (int i = 0; i < 8; i++) { V t = b.L(36 + i); b.z(t * (t - one)); }
}

// ---- 9: Com32Chip — input_1 0..3, input_2 4..7, diff 8, diff_inv 9, not_equal 10, output 11, is_ne 12, is_eq 13
template <class B> BB_HD void eval_com(B& b) {
    using V = typename B::V;
    const V one = ONE<V>();
    const V ne = b.L(10), is_ne = b.L(12), is_eq = b.L(13);
    b.section("Com32Chip::eval");
    b.z(b.L(8) - sqdiff4(b, 0, 4));
    b.z(ne * (ne - one));
    b.z(ne - b.L(8) * b.L(9));
    b.z((one - ne) * b.L(8));
    b.z(is_ne * (is_ne - one)); b.z(is_eq * (is_eq - one));
    b.z((is_ne + is_eq) * (is_ne + is_eq - one));
    b.z(b.L(11) - (is_ne * ne + is_eq * (one - ne)));
}

// ---- 10: Bitwise32Chip — input_1 0..3, input_2 4..7, bits_1 8..39, bits_2 40..71, output 72..75, is_and 76, is_or 77, is_xor 78
template <class B> BB_HD void eval_bitwise(B& b) {
    using V = typename B::V;
    const V one = ONE<V>();
    const V p2[8] = {K<V, 1>(), K<V, 2>(), K<V, 4>(), K<V, 8>(), K<V, 16>(), K<V, 32>(), K<V, 64>(), K<V, 128>()};
    const V is_and = b.L(76), is_or = b.L(77), is_xor = b.L(78);
    b.section("Bitwise32Chip::eval bytes");
    for (int i = 0; i < 4; i++) {
        V byte1 = ZERO<V>(), byte2 = ZERO<V>(), band = ZERO<V>();
        for (int k = 0; k < 8; k++) {
            const V x = b.L(8 + 8 * i + k), y = b.L(40 + 8 * i + k);
            byte1 = byte1 + x * p2[k]; byte2 = byte2 + y * p2[k]; band = band + x * y * p2[k];
        }
        b.z(b.L(i) - byte1);
        b.z(b.L(4 + i) - byte2);
        const V outb = b.L(72 + i);
        b.z(is_and * (band - outb));
        b.z(is_or * (byte1 + byte2 - band - outb));
        b.z(is_xor * (byte1 + byte2 - K<V, 2>() * band - outb));
        for (int k = 0; k < 8; k++) { V t = b.L(8 + 8 * i + k); b.z(t * (t - one)); }
        for (int k = 0; k < 8; k++) { V t = b.L(40 + 8 * i + k); b.z(t * (t - one)); }
    }
    b.section("Bitwise32Chip::eval opcode flags");
    b.z(is_and * (is_and - one)); b.z(is_or * (is_or - one)); b.z(is_xor * (is_xor - one));
    const V s = is_and + is_or + is_xor;
    b.z(s * (s - one));
}

// ---- 11: OutputChip — clk 0, value 1, is_real 2, diff 3, counter 4, counter_mult 5, opcode 6 -----------
template <class B> BB_HD void eval_output(B& b) {
    using V = typename B::V;
    b.section("OutputChip::eval range check");
    b.z(b.trans * (b.L(3) - (b.N(0) - b.L(0))));
    b.z(b.trans * (b.N(4) - (b.L(4) + ONE<V>())));
    b.section("OutputChip::eval bus opcode");
    b.z(b.L(2) * (b.L(6) - K<V, 300>()));
}

// ---- 13: StaticDataChip — addr 0, value 1..4, is_real 5 ---------------------------------------------------
template <class B> BB_HD void eval_static_data(B& b) {
    using V = typename B::V;
    b.section("StaticDataChip::eval_main");
    b.z(b.trans * (b.L(5) * b.N(5)) * (b.N(0) - (b.L(0) + ONE<V>() + ONE<V>() + ONE<V>() + ONE<V>())));
}

template <int CHIP, class B> BB_HD void eval_chip(B& b) {
    if (CHIP == 0) eval_cpu(b);
    else if (CHIP == 3) eval_add(b);
    else if (CHIP == 4) eval_sub(b);
    else if (CHIP == 5) eval_mul(b);
    else if (CHIP == 7) eval_shift(b);
    else if (CHIP == 8) eval_lt(b);
    else if (CHIP == 9) eval_com(b);
    else if (CHIP == 10) eval_bitwise(b);
    else if (CHIP == 11) eval_output(b);
    else if (CHIP == 13) eval_static_data(b);
    // 1 program, 2 memory, 6 div, 12 range: empty eval
}

// f(std::integral_constant<int, CHIP>{}) for CHIP == chip_id: the per-chip instantiation behind a run-time chip id
// (ids >= VGPU_NUM_CHIPS call nothing)
template <int CHIP = 0, class Fn> void with_chip(uint32_t chip_id, Fn&& f) {
    if constexpr (CHIP < VGPU_NUM_CHIPS) {
        if (chip_id == CHIP) f(std::integral_constant<int, CHIP>{});
        else with_chip<CHIP + 1>(chip_id, f);
    }
}

}  // namespace air
