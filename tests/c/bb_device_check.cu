// Device instantiation of the product's field arithmetic (valida_b200/csrc/bb.cuh): the __CUDA_ARCH__ branches — __umulhi in
// mul / monty_reduce64, __brev, the lazy 64-bit accumulators bb::Lazy5 / madw / lazy_fold and the e5_mul built on them.  Reads
// the line protocol of bb_host_check.cc from stdin (operands as decimal Montgomery words), runs every line as one thread of one
// kernel and prints the results in input order.  One more operation exercises Lazy5 at its bound:
//     lazy T NBASE NEXT V   all five limbs preset to lazy_fold(T); NBASE x fma_base(x, V); NEXT x fma_ext(x, x, 2x); value()
// with x = (V, V, V, V, V).  Built with nvcc for sm_90a by tests/test_gpu_bb_device_arith.py, which checks every answer against
// Python integers.
#include <cstdio>
#include <cstring>
#include <vector>
#include "bb.cuh"

enum Kind { MUL, ADD, SUB, NEG, INV, TO_MONTY, FROM_MONTY, REDUCE64, POW, REVBITS, GEN, E5MUL, E5ADD, E5SUB, E5INV, E5FROB, LAZY };

struct Op {
    int kind;
    unsigned long long x[10];
};

__global__ void run_ops(const Op* ops, int n, uint32_t* out /* [n][5] */, int* nout) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Op& o = ops[i];
    uint32_t* r = out + 5 * (size_t)i;
    const uint32_t a = (uint32_t)o.x[0], b = (uint32_t)o.x[1];
    bb::E5 ea, eb;
    for (int l = 0; l < 5; l++) { ea.c[l] = (uint32_t)o.x[l]; eb.c[l] = (uint32_t)o.x[5 + l]; }
    int k = 1;
    switch (o.kind) {
        case MUL: r[0] = bb::mul(a, b); break;
        case ADD: r[0] = bb::add(a, b); break;
        case SUB: r[0] = bb::sub(a, b); break;
        case NEG: r[0] = bb::neg(a); break;
        case INV: r[0] = bb::inv(a); break;
        case TO_MONTY: r[0] = bb::to_monty(a); break;
        case FROM_MONTY: r[0] = bb::from_monty(a); break;
        case REDUCE64: r[0] = bb::monty_reduce64(o.x[0]); break;
        case POW: r[0] = bb::pow(a, o.x[1]); break;
        case REVBITS: r[0] = bb::reverse_bits(a, (int)o.x[1]); break;
        case GEN: r[0] = bb::two_adic_generator_monty((int)o.x[0]); break;
        case E5MUL: case E5ADD: case E5SUB: case E5INV: case E5FROB: {
            bb::E5 e;
            if (o.kind == E5MUL) e = bb::e5_mul(ea, eb);
            else if (o.kind == E5ADD) e = bb::e5_add(ea, eb);
            else if (o.kind == E5SUB) e = bb::e5_sub(ea, eb);
            else if (o.kind == E5INV) e = bb::e5_inv(ea);
            else { uint32_t z[5]; bb::e5_frob_consts(z); e = bb::e5_frobenius(ea, z); }
            for (int l = 0; l < 5; l++) r[l] = e.c[l];
            k = 5;
            break;
        }
        case LAZY: {
            bb::Lazy5 s;
            s.init();
            for (int l = 0; l < 5; l++) s.a[l] = bb::lazy_fold(o.x[0]);
            bb::E5 x;
            for (int l = 0; l < 5; l++) x.c[l] = (uint32_t)o.x[3];
            for (unsigned long long j = 0; j < o.x[1]; j++) s.fma_base(x, (uint32_t)o.x[3]);
            const bb::E5 x2 = bb::e5_dbl(x);
            for (unsigned long long j = 0; j < o.x[2]; j++) s.fma_ext(x, x, x2);
            const bb::E5 e = s.value();
            for (int l = 0; l < 5; l++) r[l] = e.c[l];
            k = 5;
            break;
        }
    }
    nout[i] = k;
}

static int nargs(int kind) {
    switch (kind) {
        case NEG: case INV: case TO_MONTY: case FROM_MONTY: case REDUCE64: case GEN: return 1;
        case MUL: case ADD: case SUB: case POW: case REVBITS: return 2;
        case E5INV: case E5FROB: return 5;
        case E5MUL: case E5ADD: case E5SUB: return 10;
        case LAZY: return 4;
    }
    return -1;
}

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 3; } } while (0)

int main() {
    static const char* names[] = {"mul", "add", "sub", "neg", "inv", "to_monty", "from_monty", "reduce64", "pow", "revbits", "gen",
                                  "e5mul", "e5add", "e5sub", "e5inv", "e5frob", "lazy"};
    std::vector<Op> ops;
    char name[32];
    while (scanf("%31s", name) == 1) {
        Op o{};
        o.kind = -1;
        for (int k = 0; k <= LAZY; k++) if (!strcmp(name, names[k])) o.kind = k;
        if (o.kind < 0) return 2;
        for (int j = 0; j < nargs(o.kind); j++) if (scanf("%llu", &o.x[j]) != 1) return 1;
        ops.push_back(o);
    }
    const int n = (int)ops.size();
    if (!n) return 0;
    Op* d_ops; uint32_t* d_out; int* d_nout;
    CK(cudaMalloc(&d_ops, n * sizeof(Op)));
    CK(cudaMalloc(&d_out, (size_t)n * 5 * 4));
    CK(cudaMalloc(&d_nout, (size_t)n * 4));
    CK(cudaMemcpy(d_ops, ops.data(), n * sizeof(Op), cudaMemcpyHostToDevice));
    run_ops<<<(n + 127) / 128, 128>>>(d_ops, n, d_out, d_nout);
    CK(cudaGetLastError());
    std::vector<uint32_t> out((size_t)n * 5);
    std::vector<int> nout(n);
    CK(cudaMemcpy(out.data(), d_out, out.size() * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(nout.data(), d_nout, nout.size() * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; i++) {
        for (int l = 0; l < nout[i]; l++) printf(l ? " %u" : "%u", out[5 * (size_t)i + l]);
        printf("\n");
    }
    CK(cudaFree(d_ops)); CK(cudaFree(d_out)); CK(cudaFree(d_nout));
    return 0;
}
