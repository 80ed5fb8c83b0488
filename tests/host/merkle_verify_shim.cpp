// CPU build of the per-level operand choice of the Pedersen-leaf path verification (crypto_primitives_b200/csrc/merkle_verify_pedersen.cuh)
// for tests/test_merkle_verify_pedersen_host.py: which sibling and which side level j of proof i takes (verify_step), and the
// TwoToOneCRH row the byte tree's row kernel writes from them (ped_verify_row).  Not part of the product.
#include "../../crypto_primitives_b200/csrc/merkle_verify_pedersen.cuh"

#include <cstdint>
using namespace cpb;

// out[0] = 1 when the sibling comes from the auth-path array (0: the leaf sibling array), out[1] = its element, out[2] = 1 when the
// computed node is the right child.
extern "C" void host_verify_step(uint64_t i, int plen, int j, uint64_t index, uint64_t* out) {
    const VerifyStep s = verify_step(i, plen, j, index);
    out[0] = s.from_path ? 1 : 0;
    out[1] = s.elem;
    out[2] = s.right ? 1 : 0;
}

// field 0: BLS12-381 Fr (Jubjub's base field), 1: BLS12-377 Fr (ed-on-BLS12-377's).  cur: proof i's current digest; leaf_sibs / paths:
// the whole arrays (16 words per digest, Montgomery form); row: 32 words.
extern "C" void host_ped_verify_row(int field, const uint32_t* cur, const uint32_t* leaf_sibs, const uint32_t* paths, uint64_t i, int plen,
                                    int j, uint64_t index, uint32_t* row) {
    if (field == 0) ped_verify_row<Bls12_381_Fr>(row, cur, leaf_sibs, paths, i, plen, j, index);
    else ped_verify_row<Bls12_377_Fr>(row, cur, leaf_sibs, paths, i, plen, j, index);
}
