// CBOR codec of the proof (proof.h).  The shape is written once, as a walk over the proof types that an Encoder and a Decoder
// both instantiate: the Encoder emits exactly what serde/ciborium emits, the Decoder accepts that and refuses everything
// the walk does not describe.
#include "proof.h"
#include <algorithm>
#include <cstring>

namespace vgh {
namespace {

struct Encoder {
    // append-only byte buffer with a raw cursor: the ~150 k field elements of a proof are 12-byte stores, not push_backs
    std::vector<uint8_t> b; size_t n = 0;
    uint8_t* room(size_t k) { if (n + k > b.size()) b.resize(std::max(2 * b.size(), n + k + (1u << 20))); return b.data() + n; }
    void head(uint8_t major, uint64_t v) {
        uint8_t* o = room(9);
        const uint8_t m = (uint8_t)(major << 5);
        if (v < 24) { o[0] = m | (uint8_t)v; n += 1; }
        else if (v <= 0xff) { o[0] = m | 24; o[1] = (uint8_t)v; n += 2; }
        else if (v <= 0xffff) { o[0] = m | 25; o[1] = (uint8_t)(v >> 8); o[2] = (uint8_t)v; n += 3; }
        else if (v <= 0xffffffffull) { o[0] = m | 26; for (int i = 0; i < 4; i++) o[1 + i] = (uint8_t)(v >> (24 - 8 * i)); n += 5; }
        else { o[0] = m | 27; for (int i = 0; i < 8; i++) o[1 + i] = (uint8_t)(v >> (56 - 8 * i)); n += 9; }
    }
    void key(const char* s) { size_t k = std::strlen(s); head(3, k); std::memcpy(room(k), s, k); n += k; }
    void map(uint64_t k) { head(5, k); }
    void len(uint64_t k) { head(4, k); }
    template <class T, class F> void seq(std::vector<T>& v, F&& f) { head(4, v.size()); for (T& x : v) f(x); }
    void u32(uint32_t v) { head(0, v); }
    // BabyBear { value } holds the Montgomery word: {"value": u32}
    void felt(uint32_t v) {
        static const uint8_t pre[7] = {0xa1, 0x65, 'v', 'a', 'l', 'u', 'e'};
        uint8_t* o = room(12);
        std::memcpy(o, pre, 7);
        if (v < 24) { o[7] = (uint8_t)v; n += 8; }
        else if (v <= 0xff) { o[7] = 24; o[8] = (uint8_t)v; n += 9; }
        else if (v <= 0xffff) { o[7] = 25; o[8] = (uint8_t)(v >> 8); o[9] = (uint8_t)v; n += 10; }
        else { o[7] = 26; o[8] = (uint8_t)(v >> 24); o[9] = (uint8_t)(v >> 16); o[10] = (uint8_t)(v >> 8); o[11] = (uint8_t)v; n += 12; }
    }
    void felt_canonical(uint32_t c) { felt(bb::to_monty(c)); }
};

// Every method is a no-op once ok is false, so a walk runs to its end on any input.
struct Decoder {
    const uint8_t* p; const uint8_t* end; bool ok = true;
    uint64_t head(int major) {
        if (!ok || p >= end) { ok = false; return 0; }
        uint8_t b = *p++;
        if ((b >> 5) != major) { ok = false; return 0; }
        uint8_t info = b & 31;
        if (info < 24) return info;
        int n = info == 24 ? 1 : info == 25 ? 2 : info == 26 ? 4 : info == 27 ? 8 : -1;
        if (n < 0 || end - p < n) { ok = false; return 0; }
        uint64_t v = 0;
        for (int i = 0; i < n; i++) v = (v << 8) | *p++;
        return v;
    }
    void key(const char* s) {
        uint64_t n = head(3), want = std::strlen(s);
        if (!ok || n != want || (uint64_t)(end - p) < n || std::memcmp(p, s, n) != 0) { ok = false; return; }
        p += n;
    }
    void map(uint64_t n) { if (head(5) != n) ok = false; }
    // bounded array length: every element costs at least one byte, so a hostile length cannot make us allocate
    uint64_t arr() { uint64_t n = head(4); if (n > (uint64_t)(end - p)) { ok = false; return 0; } return n; }
    void len(uint64_t n) { if (arr() != n) ok = false; }
    template <class T, class F> void seq(std::vector<T>& v, F&& f) {
        v.clear();
        for (uint64_t i = 0, n = arr(); i < n && ok; i++) { v.emplace_back(); f(v.back()); }
    }
    void u32(uint32_t& v) { v = (uint32_t)head(0); }
    void felt(uint32_t& v) {
        map(1); key("value");
        const uint64_t x = head(0);
        if (x >= bb::P) ok = false;
        v = (uint32_t)x;
    }
    void felt_canonical(uint32_t& c) { felt(c); c = bb::from_monty(c); }
};

// ---- the shape (machine/src/proof.rs:13-44; p3-fri TwoAdicFriPcsProof, FriProof, QueryProof, CommitPhaseProofStep) ----
template <class IO> void ext(IO& s, bb::E5& e) { s.map(1); s.key("value"); s.len(5); for (uint32_t& x : e.c) s.felt(x); }
template <class IO> void exts(IO& s, std::vector<bb::E5>& v) { s.seq(v, [&](bb::E5& e) { ext(s, e); }); }
template <class IO> void digest(IO& s, Digest& d) { s.len(8); for (uint32_t& x : d) s.felt_canonical(x); }
template <class IO> void digests(IO& s, std::vector<Digest>& v) { s.seq(v, [&](Digest& d) { digest(s, d); }); }

// (encoding the per-query parts on several host threads into buffers of their own was measured: 0.88 ms against 0.64 ms serial)
template <class IO> void io(IO& s, PcsProof& p) {
    s.map(2);
    s.key("fri_proof"); s.map(4);
    s.key("commit_phase_commits"); digests(s, p.commit_phase_commits);
    s.key("query_proofs");
    s.seq(p.query_proofs, [&](std::vector<CommitPhaseStep>& q) {
        s.map(1); s.key("commit_phase_openings");
        s.seq(q, [&](CommitPhaseStep& st) { s.map(2); s.key("sibling_value"); ext(s, st.sibling_value); s.key("opening_proof"); digests(s, st.opening_proof); });
    });
    s.key("final_poly"); ext(s, p.final_poly);
    s.key("pow_witness"); s.felt(p.pow_witness);
    s.key("query_openings");
    s.seq(p.query_openings, [&](std::vector<BatchOpening>& q) {
        s.seq(q, [&](BatchOpening& bo) {
            s.map(2);
            s.key("opened_values"); s.seq(bo.opened_values, [&](std::vector<uint32_t>& row) { s.seq(row, [&](uint32_t& x) { s.felt(x); }); });
            s.key("opening_proof"); digests(s, bo.opening_proof);
        });
    });
}

template <class IO> void io(IO& s, MachineProof& p) {
    s.map(3);
    s.key("commitments"); s.map(3);
    s.key("main_trace"); digest(s, p.main_trace);
    s.key("perm_trace"); digest(s, p.perm_trace);
    s.key("quotient_chunks"); digest(s, p.quotient_chunks);
    s.key("opening_proof"); io(s, p.opening_proof);
    s.key("chip_proofs");
    s.seq(p.chip_proofs, [&](ChipProof& c) {
        s.map(3);
        s.key("log_degree"); s.u32(c.log_degree);
        s.key("opened_values"); s.map(7);
        s.key("preprocessed_local"); exts(s, c.preprocessed_local);
        s.key("preprocessed_next"); exts(s, c.preprocessed_next);
        s.key("trace_local"); exts(s, c.trace_local);
        s.key("trace_next"); exts(s, c.trace_next);
        s.key("permutation_local"); exts(s, c.permutation_local);
        s.key("permutation_next"); exts(s, c.permutation_next);
        s.key("quotient_chunks"); exts(s, c.quotient_chunks);
        s.key("cumulative_sum"); ext(s, c.cumulative_sum);
    });
}

// (opened_values, proof): a two-element array
template <class IO> void io(IO& s, OpenedValues& v, PcsProof& p) {
    s.len(2);
    s.seq(v, [&](auto& round) { s.seq(round, [&](auto& mat) { s.seq(mat, [&](std::vector<bb::E5>& at_point) { exts(s, at_point); }); }); });
    io(s, p);
}

}  // namespace

// The walk takes mutable references so that the Decoder can fill them; the Encoder only reads.
template <class... Parts> std::vector<uint8_t> write(size_t reserve, const Parts&... parts) {
    Encoder w;
    w.b.resize(reserve);
    io(w, const_cast<Parts&>(parts)...);
    w.b.resize(w.n);
    return std::move(w.b);
}
template <class... Parts> bool read(const uint8_t* data, uint64_t len, Parts*... parts) {
    Decoder r{data, data + len};
    io(r, *parts...);
    return r.ok && r.p == r.end;
}

std::vector<uint8_t> encode(const MachineProof& proof) { return write(4u << 20, proof); }
std::vector<uint8_t> encode_opening(const OpenedValues& values, const PcsProof& proof) { return write(0, values, proof); }
bool decode(const uint8_t* data, uint64_t len, MachineProof* out) { return read(data, len, out); }
bool decode_opening(const uint8_t* data, uint64_t len, OpenedValues* values, PcsProof* proof) { return read(data, len, values, proof); }

}  // namespace vgh
