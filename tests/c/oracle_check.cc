// Test helper: the oracle's check_constraints (oracle/machine.h, the reference's debug-build check) on a GIVEN permutation
// trace, so that a tampered permutation trace can be checked too.  Built by tests/check_support.py into a temporary directory
// from the header-only oracle; test infrastructure only.
#include "machine.h"

extern "C" {

// main: h x width row-major; prep_or_null: h x preprocessed_width; perm_flat: h x 5(k+1) row-major (flatten_to_base);
// challenges15: the three LogUp challenges.  Returns row * 4096 + constraint of the first failure, or -1.
int64_t orc_check_constraints(uint32_t chip, const uint32_t* main, uint64_t h, const uint32_t* prep_or_null, const uint32_t* perm_flat,
                              const uint32_t* challenges15) {
    const orc::ChipDef& cd = orc::chips()[chip];
    orc::Matrix m(std::vector<uint32_t>(main, main + h * cd.width), cd.width);
    orc::Matrix pm;
    if (prep_or_null) pm = orc::Matrix(std::vector<uint32_t>(prep_or_null, prep_or_null + h * cd.prep_width), cd.prep_width);
    orc::ExtMatrix perm;
    perm.width = cd.interactions.size() + 1;
    perm.v.resize(h * perm.width);
    for (size_t i = 0; i < perm.v.size(); i++) std::memcpy(perm.v[i].c, perm_flat + 5 * i, 20);
    orc::Ext5 rnd[3];
    for (int i = 0; i < 3; i++) std::memcpy(rnd[i].c, challenges15 + 5 * i, 20);
    return orc::check_constraints(cd, m, prep_or_null ? &pm : nullptr, perm, rnd);
}

}  // extern "C"
