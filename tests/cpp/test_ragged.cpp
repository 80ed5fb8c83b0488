// C++ host-mirror test of the ragged Poseidon calls (include/cpb200.hpp over the C-ABI), the shape a Rust shim's
// Vec<Vec<F>> takes: CRH over inputs of different lengths, a Merkle tree over leaves of different lengths
// (MerkleTree::new hashes each leaf at its own length, R/merkle_tree/mod.rs:411-422), and its paths verified in one launch.
// Prints the tree's root for tests/test_gpu_ragged.py, which rebuilds the same tree through the Python API.
#include <cstdio>
#include <cstdlib>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    auto params = poseidon::Config::get_default_poseidon_parameters(CPB_BLS12_381_FR, 2, false);
    REQUIRE(params);
    const poseidon::Config& P = *params;

    // 16 leaves, leaf i has i % 9 elements: canonical values (31 i + 7 k + 1, k, 0, 0), element k of leaf i
    const size_t n = 16;
    std::vector<std::vector<Fe>> leaves(n);
    for (size_t i = 0; i < n; i++) {
        std::vector<Fe> canon;
        for (uint64_t k = 0; k < i % 9; k++) canon.push_back(Fe{31 * i + 7 * k + 1, k, 0, 0});
        leaves[i].resize(canon.size());
        if (!canon.empty()) check(cpb_field_to_montgomery(CPB_BLS12_381_FR, 0, canon[0].data(), leaves[i][0].data(), canon.size()));
    }

    // one ragged CRH call == one evaluate per input
    std::vector<Fe> digests = poseidon::CRH::evaluate_batch(P, leaves);
    for (size_t i = 0; i < n; i++) REQUIRE(digests[i] == poseidon::CRH::evaluate(P, leaves[i]));

    auto tree = PoseidonMerkleTree::create(P, P, leaves);
    REQUIRE(tree.leaf_nodes == digests && tree.height() == 5);
    std::vector<Fe> lvl = poseidon::TwoToOneCRH::compress_batch(P, digests);
    while (lvl.size() > 1) lvl = poseidon::TwoToOneCRH::compress_batch(P, lvl);
    REQUIRE(lvl[0] == tree.root());

    std::vector<size_t> all;
    for (size_t i = 0; i < n; i++) all.push_back(i);
    std::vector<uint8_t> ok = tree.verify_batch(P, P, tree.root(), all, leaves);
    for (uint8_t v : ok) REQUIRE(v == 1);
    std::vector<std::vector<Fe>> longer = leaves;
    longer[5].push_back(Fe{0, 0, 0, 0});                  // 5 elements -> 6: the zero stays inside the last rate-2 block, same digest
    longer[6].push_back(Fe{0, 0, 0, 0});                  // 6 elements -> 7: the zero starts a new block, another digest
    ok = tree.verify_batch(P, P, tree.root(), all, longer);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == (i == 6 ? 0 : 1));

    // equal lengths take the uniform calls and agree with them
    std::vector<std::vector<Fe>> pairs(8, std::vector<Fe>(leaves[2].begin(), leaves[2].end()));
    for (size_t i = 0; i < 8; i++) pairs[i][0] = leaves[9 + (i % 7)].empty() ? pairs[i][0] : leaves[9 + (i % 7)][0];
    std::vector<Fe> flat;
    for (auto& x : pairs) flat.insert(flat.end(), x.begin(), x.end());
    REQUIRE(poseidon::CRH::evaluate_batch(P, pairs) == poseidon::CRH::evaluate_batch(P, flat, 2));

    // the host form checks the offsets
    std::vector<uint64_t> bad = {0, 2, 1};
    std::vector<Fe> out(2);
    REQUIRE(cpb_poseidon_crh_ragged_batch(P.ctx(), leaves[2][0].data(), bad.data(), out[0].data(), 2) == CPB_BAD_LENGTH);
    bool threw = false;
    try { PoseidonMerkleTree::create(P, P, std::vector<std::vector<Fe>>(leaves.begin(), leaves.begin() + 3)); }
    catch (const Error& e) { threw = e.status == CPB_NOT_POW2; }
    REQUIRE(threw);

    const Fe r = tree.root();
    printf("ragged root = %016llx %016llx %016llx %016llx\n", (unsigned long long)r[3], (unsigned long long)r[2], (unsigned long long)r[1],
           (unsigned long long)r[0]);
    printf("cpp ragged ok\n");
    return 0;
}
