// CPU build of the host side of the tensor-core full rounds (crypto_primitives_b200/csrc/poseidon_host.hpp: tc_full_tables; the
// row-table word map of poseidon_tc.cuh), for tests/test_poseidon_tc_full.py.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
using namespace cpb;

// The BN254 Fr t = 3 schedule's full-round row tables (u32 words) when out has room for them; returns their word count, -1 when
// the shape is not t = 3 or the schedule is dense.
extern "C" long host_tc_full_tables(int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                    const uint64_t* mds, uint32_t* out, long max_words) {
    if (rate + cap != 3) return -1;
    host::Field F(host::field_modulus(Bn254_Fr::ID));
    host::PoseidonParams P;
    P.rate = rate; P.capacity = cap; P.full_rounds = rf; P.partial_rounds = rp; P.alpha = alpha;
    P.ark.resize((size_t)(rf + rp) * 3);
    P.mds.resize(9);
    memcpy(P.ark.data(), ark, P.ark.size() * 32);
    memcpy(P.mds.data(), mds, P.mds.size() * 32);
    const host::PoseidonSchedule S = host::derive_schedule(F, P, true);
    if (!S.sparse) return -1;
    const std::vector<u32> t = host::tc_full_tables(F, S);
    if (out && (long)t.size() <= max_words) memcpy(out, t.data(), t.size() * 4);
    return (long)t.size();
}

// tc_tab_word(nt, kc, lane, r, 3) for nt, kc, lane, r in that order: where tc_output reads a row table.
extern "C" void host_tc_row_words(int* out) {
    for (int nt = 0; nt < 4; nt++)
        for (int kc = 0; kc < 3; kc++)
            for (int lane = 0; lane < 32; lane++)
                for (int r = 0; r < 2; r++) *out++ = tc_tab_word(nt, kc, lane, r, 3);
}

// The split form's matrix index of full round fr (pos_full_index: 0 M, 1 Mpre, 2 Mpost).
extern "C" int host_pos_full_index(int rf, int fr) {
    PoseidonDev P{};
    P.rf = rf;
    return pos_full_index(P, fr);
}
