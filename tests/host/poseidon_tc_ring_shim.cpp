// CPU build of the host side of the tensor-core hash kernel's staged constants and partial-round table ring
// (crypto_primitives_b200/csrc/poseidon_host.hpp: tc_const_image; poseidon_tc.cuh: tc_ring_slot, tc_ring_parity, tc_ring_next),
// for tests/test_poseidon_tc_ring.py.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
using namespace cpb;

// The compact constant image of the BN254 Fr t = 3 sparse schedule: offs[6] <- off_c, off_cp0, off_pc, off_mod, off_sc0, n_elems;
// the image (4 x u64 per element) is written when it has room.  Returns n_elems, -1 when the shape has no image.
extern "C" long host_tc_const_image(int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                    const uint64_t* mds, int* offs, uint64_t* image, long max_elems) {
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
    const host::TcConstImage I = host::tc_const_image(S);
    const int o[6] = {I.off_c, I.off_cp0, I.off_pc, I.off_mod, I.off_sc0, I.n_elems};
    memcpy(offs, o, sizeof(o));
    if (image && I.n_elems <= max_elems) memcpy(image, I.consts.data(), I.consts.size() * 8);
    return I.n_elems;
}

// Slot, phase parity and refill source of ring round g (counted over the kernel's batches), for n rounds g = 0 .. n-1 of a
// schedule with rp partial rounds: out[3 g .. 3 g + 2] <- tc_ring_slot(g), tc_ring_parity(g), tc_ring_next(g mod rp, rp).
extern "C" int host_tc_ring_map(int n, int rp, int* out) {
    for (int g = 0; g < n; g++) {
        out[3 * g] = tc_ring_slot((unsigned)g);
        out[3 * g + 1] = (int)tc_ring_parity((unsigned)g);
        out[3 * g + 2] = tc_ring_next(g % rp, rp);
    }
    return kTcRingSlots;
}
