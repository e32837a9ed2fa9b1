// The product's proof codec (valida_b200/csrc/host/proof.cc) on its own, driven from stdin: a first line naming the kind
// ("proof" or "opening"), then the CBOR bytes.  Writes the re-encoding of what it decoded to stdout and exits 0, or exits 3
// when the decoder rejects the bytes.  Built with g++ and the address / undefined-behaviour sanitizers by
// tests/test_proof_codec.py.  No GPU, no CUDA runtime call.
#include <cstdio>
#include <iostream>
#include <iterator>
#include <string>
#include "host/proof.h"

int main() {
    std::string kind;
    if (!std::getline(std::cin, kind)) return 2;
    const std::vector<uint8_t> in((std::istreambuf_iterator<char>(std::cin)), std::istreambuf_iterator<char>());
    std::vector<uint8_t> out;
    if (kind == "proof") {
        vgh::MachineProof p;
        if (!vgh::decode(in.data(), in.size(), &p)) return 3;
        out = vgh::encode(p);
    } else if (kind == "opening") {
        vgh::OpenedValues v;
        vgh::PcsProof p;
        if (!vgh::decode_opening(in.data(), in.size(), &v, &p)) return 3;
        out = vgh::encode_opening(v, p);
    } else {
        return 2;
    }
    return std::fwrite(out.data(), 1, out.size(), stdout) == out.size() ? 0 : 1;
}
