// The device round schedule as host::derive_schedule (crypto_primitives_b200/csrc/poseidon_host.hpp) lays it out, for tests
// that check its layout directly.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
using namespace cpb;

// offs[12] <- t, sparse, off_c, off_m, off_mpre, off_cp0, off_pc, off_sp, off_arkp, off_mod, off_sc0, n_elems.
// consts (4 x u64 Montgomery limbs per element) is written when it has room for n_elems.  Returns n_elems, -1 on a bad field.
extern "C" long host_poseidon_schedule(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                       const uint64_t* mds, int allow_sparse, int* offs, uint64_t* consts, long max_elems) {
    const uint64_t* mod = host::field_modulus(field);
    if (!mod) return -1;
    host::Field F(mod);
    host::PoseidonParams P;
    P.rate = rate; P.capacity = cap; P.full_rounds = rf; P.partial_rounds = rp; P.alpha = alpha;
    const int t = rate + cap;
    P.ark.resize((size_t)(rf + rp) * t);
    P.mds.resize((size_t)t * t);
    memcpy(P.ark.data(), ark, P.ark.size() * 32);
    memcpy(P.mds.data(), mds, P.mds.size() * 32);
    const host::PoseidonSchedule S = host::derive_schedule(F, P, allow_sparse != 0);
    const int o[12] = {S.t, S.sparse, S.off_c, S.off_m, S.off_mpre, S.off_cp0, S.off_pc, S.off_sp, S.off_arkp, S.off_mod, S.off_sc0, S.n_elems};
    memcpy(offs, o, sizeof(o));
    if (S.n_elems <= max_elems) memcpy(consts, S.consts.data(), S.consts.size() * 8);
    return S.n_elems;
}
