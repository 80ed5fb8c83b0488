// merkle_verify_pedersen.cuh -- the per-level operand choice of Path::verify (R/merkle_tree/mod.rs:172-212) for the byte tree of
// cpb_merkle_pedersen_build, shared by the row kernel of cpb_merkle_verify_pedersen.cu and the CPU tests' host shim.
#pragma once
#include "te_ops.cuh"

namespace cpb {

// Level j (0 .. plen) of proof i's fold, bottom-up: which sibling the computed node is paired with and on which side.  Level 0
// pairs the claimed leaf digest with leaf_sibling_hashes[i]; level j > 0 with auth_paths[i * plen + (plen - j)], since Path.auth_path
// is stored root side first.  The computed node is the right child when bit j of the index is set; bits above plen are never read.
struct VerifyStep {
    bool from_path;   // false: the leaf sibling array, true: the auth-path array
    u64 elem;         // element of that array (a digest of 16 words)
    bool right;       // the computed node is the right child
};
CPB_HD VerifyStep verify_step(u64 i, int plen, int j, u64 index) {
    VerifyStep s;
    s.from_path = j > 0;
    s.elem = j == 0 ? i : i * (u64)plen + (u64)(plen - j);
    s.right = ((index >> j) & 1ull) != 0;
    return s;
}

// The TwoToOneCRH row of level j (te_node_row: canonical x_l || y_l || x_r || y_r) from the current digest `cur` of proof i.
template <class F>
CPB_HD void ped_verify_row(u32* row, const u32* cur, const u32* leaf_sibs, const u32* paths, u64 i, int plen, int j, u64 index) {
    const VerifyStep s = verify_step(i, plen, j, index);
    const u32* sib = (s.from_path ? paths : leaf_sibs) + 16 * s.elem;
    te_node_row<F>(row, s.right ? sib : cur, s.right ? cur : sib);
}

}  // namespace cpb
