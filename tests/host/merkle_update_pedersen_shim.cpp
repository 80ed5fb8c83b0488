// CPU build of the pieces of the Pedersen-node Merkle update (crypto_primitives_b200/csrc/cpb_merkle_update_pedersen.cu) that are
// CPB_HD, for tests/test_merkle_update_pedersen_host.py: the TwoToOneCRH row of one node (te_node_row) and where a candidate slot's
// children are read from (upd_site / upd_kids / upd_child_at at 16-word digests), and one node hash of the narrow-level warp kernel
// (k_ped_upd_top) emulated for 32 lanes: the lane split of the lookups (te_lane_sum, te_lookup_value) and the shuffle reduction.
// Not part of the product.
#include "../../crypto_primitives_b200/csrc/merkle_update.cuh"
#include "../../crypto_primitives_b200/csrc/te_ops.cuh"

#include <cstdint>
#include <vector>
using namespace cpb;

// field 0: BLS12-381 Fr (Jubjub's base field), 1: BLS12-377 Fr (ed-on-BLS12-377's).  left / right: affine (x, y), Montgomery form.
extern "C" void host_ped_node_row(int field, const uint32_t* left, const uint32_t* right, uint32_t* row) {
    if (field == 0) te_node_row<Bls12_381_Fr>(row, left, right);
    else te_node_row<Bls12_377_Fr>(row, left, right);
}

// Candidate `cand` of level l of the plan over the sorted distinct indexes U[0..m) (k pairs given, n = 2^h leaves).  Returns
// whether the candidate is touched; then src[2 b] / src[2 b + 1] = (array, element) of child b: array 0 the scratch, 1 the leaf
// array, 2 the heap-ordered inner nodes.
extern "C" int host_ped_child_src(const uint64_t* U, uint64_t m, uint64_t k, int h, int l, uint64_t cand, uint64_t* src) {
    UpdPlan X;
    X.h = h;
    X.k = k;
    upd_offsets(h, k, X.off);
    const UpdSite S = upd_site(U, m, h, l, k, cand);
    if (!S.touched) return 0;
    const UpdKids K = upd_kids(U, m, h, l, k, S);
    const u64 n = 1ull << h;
    std::vector<u32> scratch(16 * X.off[h + 1]), leaves(16 * n), nodes(16 * (n - 1));
    const u32* at[2] = {upd_child_at<16>(X, l, K.lt, K.lslot, 2 * S.node, scratch.data(), leaves.data(), nodes.data()),
                        upd_child_at<16>(X, l, K.rt, K.rslot, 2 * S.node + 1, scratch.data(), leaves.data(), nodes.data())};
    for (int b = 0; b < 2; b++) {
        const u32* p = at[b];
        const std::vector<u32>* arrs[3] = {&scratch, &leaves, &nodes};
        for (int a = 0; a < 3; a++) {
            const u32* base = arrs[a]->data();
            if (p >= base && p < base + arrs[a]->size()) {
                src[2 * b] = a;
                src[2 * b + 1] = (u64)(p - base) / 16;
                if ((u64)(p - base) % 16) src[2 * b] = 99;          // not element-aligned
            }
        }
    }
    return 1;
}

// k_ped_upd_top's hash of one row over Jubjub (BLS12-381 Fr), emulated lane by lane.  Table entries are computed on the fly from
// the generators (gens_xy: n_gens affine points, Montgomery), as the context's table holds them: entry (c, v) = the sum of
// generators c cb + j over the set bits j of v.  values[c] receives lookup c's table index (lane c % 32 handles it).  The
// reduction is __shfl_down_sync with te_add: in round `off`, lane i adds lane i + off's sum (its own when i + off > 31).
extern "C" void host_ped_warp_hash(const uint32_t* gens_xy, int n_gens, const uint32_t* d2, const uint8_t* row, long len, int cb,
                                   int n_chunks, uint32_t* values, uint32_t* out_xy) {
    using F = Bls12_381_Fr;
    u32 pm[8];
    fp_modulus<F>(pm);
    auto entry = [&](int c, u32 v, u32* yp, u32* ym, u32* t2d) {
        values[c] = v;
        TePoint s;
        te_identity<F>(s);
        for (int j = 0; j < cb; j++) {
            const int g = c * cb + j;
            if (!((v >> j) & 1u) || g >= n_gens) continue;
            TePoint q;
            te_from_affine<F>(q, gens_xy + 16 * g, gens_xy + 16 * g + 8, pm);
            te_add<F>(s, q, d2, pm);
        }
        u32 x[8], y[8];
        te_to_affine<F>(x, y, s, pm);
        te_niels<F>(yp, ym, t2d, x, y, d2, pm);
    };
    std::vector<TePoint> acc(32), snap(32);
    for (int lane = 0; lane < 32; lane++) te_lane_sum<F>(acc[lane], row, len, cb, n_chunks, lane, 32, entry, pm);
    for (int off = 16; off > 0; off >>= 1) {
        snap = acc;
        for (int lane = 0; lane < 32; lane++) te_add<F>(acc[lane], snap[lane + off < 32 ? lane + off : lane], d2, pm);
    }
    te_to_affine<F>(out_xy, out_xy + 8, acc[0], pm);
}
