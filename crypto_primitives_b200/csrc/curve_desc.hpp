// curve_desc.hpp -- the twisted-Edwards curves of the C-ABI (cpb_curve, include/cpb200.h), described once for the host code
// that builds Pedersen contexts, serialises points and builds signature contexts.  a = -1 on both curves.
#pragma once
#include "hostfp.hpp"

namespace cpb {
namespace host {

struct CurveDesc {
    int field_id;          // base field (cpb_field id)
    int scalar_field_id;   // field of the prime-order subgroup's order r (cpb_field id)
    bool d_is_ratio;       // d = -(num/den) when true, else d = num
    u64 num, den;
    const u64* order() const { return element_field_modulus(scalar_field_id); }
    Fe d(const Field& F) const { return d_is_ratio ? F.neg(F.mul(F.from_u64(num), F.inv(F.from_u64(den)))) : F.from_u64(num); }
};

inline bool curve_desc(int curve_id, CurveDesc& c) {
    switch (curve_id) {
        case 0: c = {0, 2, true, 10240, 10241}; return true;   // CPB_JUBJUB: ark-ed-on-bls12-381, d = -(10240/10241)
        case 1: c = {3, 4, false, 3021, 1}; return true;       // CPB_ED_ON_BLS12_377: ark-ed-on-bls12-377, d = 3021
    }
    return false;
}

}  // namespace host
}  // namespace cpb
