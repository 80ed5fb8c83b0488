// C++ host-mirror test of the Merkle update (include/cpb200.hpp over cpb_merkle_poseidon_update): update_batch / update /
// check_update(_batch) on a PoseidonMerkleTree equal a rebuild from the updated leaves, and a wrong root leaves the tree untouched.
#include <cstdio>
#include <cstdlib>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    auto params = poseidon::Config::get_default_poseidon_parameters(CPB_BLS12_381_FR, 2, false);
    REQUIRE(params);
    const poseidon::Config& P = *params;
    const size_t n = 1024, L = 2;
    auto element = [](uint64_t seed) {                     // canonical (seed, seed^2, 0, 0) -> Montgomery
        Fe c{seed * 2654435761ull + 1, seed * seed, 0, 0}, m;
        check(cpb_field_to_montgomery(CPB_BLS12_381_FR, 0, c.data(), m.data(), 1));
        return m;
    };
    std::vector<Fe> leaves(n * L);
    for (size_t i = 0; i < n * L; i++) leaves[i] = element(i);
    auto tree = PoseidonMerkleTree::create(P, P, leaves, L);

    // a batch with a repeated index (the last occurrence wins) and both ends of the tree
    std::vector<uint64_t> idx = {5, 1023, 0, 6, 5, 512};
    std::vector<Fe> upd(idx.size() * L);
    for (size_t i = 0; i < upd.size(); i++) upd[i] = element(100000 + i);
    tree.update_batch(P, P, idx, upd, L);
    for (size_t j = 0; j < idx.size(); j++)
        for (size_t e = 0; e < L; e++) leaves[idx[j] * L + e] = upd[j * L + e];
    auto rebuilt = PoseidonMerkleTree::create(P, P, leaves, L);
    REQUIRE(tree.leaf_nodes == rebuilt.leaf_nodes && tree.non_leaf_nodes == rebuilt.non_leaf_nodes);

    // single update
    std::vector<Fe> one = {element(7), element(8)};
    tree.update(P, P, 300, one);
    leaves[600] = one[0];
    leaves[601] = one[1];
    rebuilt = PoseidonMerkleTree::create(P, P, leaves, L);
    REQUIRE(tree.non_leaf_nodes == rebuilt.non_leaf_nodes);

    // check_update: a wrong root changes nothing, the right one applies
    std::vector<Fe> two = {element(9), element(10)};
    std::vector<Fe> after = leaves;
    after[2 * 77] = two[0];
    after[2 * 77 + 1] = two[1];
    const Fe good = PoseidonMerkleTree::create(P, P, after, L).root();
    Fe bad = good;
    bad[0] ^= 1;
    const auto before_nodes = tree.non_leaf_nodes;
    const auto before_leaves = tree.leaf_nodes;
    REQUIRE(!tree.check_update(P, P, 77, two, bad));
    REQUIRE(tree.non_leaf_nodes == before_nodes && tree.leaf_nodes == before_leaves);
    REQUIRE(tree.check_update_batch(P, P, {77}, two, L, good));
    REQUIRE(tree.root() == good);

    // host form rules: an index >= n is rejected
    bool threw = false;
    try { tree.update(P, P, n, one); }
    catch (const Error& e) { threw = e.status == CPB_BAD_PARAMS; }
    REQUIRE(threw);
    printf("cpp update ok\n");
    return 0;
}
