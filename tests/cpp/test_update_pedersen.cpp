// C++ host-mirror test of the Pedersen byte-tree update (include/cpb200.hpp over cpb_merkle_pedersen_update): update_batch / update /
// check_update(_batch) on a PedersenMerkleTree equal a rebuild from the updated leaves, and a wrong root leaves the tree untouched.
// argv[1]: the 4 x 256 Jubjub generators, affine (x, y) Montgomery limbs, 64 bytes each (written by the calling test).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

static bool same(const std::vector<Affine>& a, const std::vector<Affine>& b) {
    return a.size() == b.size() && (a.empty() || memcmp(a.data(), b.data(), a.size() * sizeof(Affine)) == 0);
}

int main(int argc, char** argv) {
    REQUIRE(argc == 2);
    std::vector<Affine> gens(1024);
    FILE* f = fopen(argv[1], "rb");
    REQUIRE(f && fread(gens.data(), sizeof(Affine), gens.size(), f) == gens.size());
    fclose(f);
    pedersen::Parameters P(CPB_JUBJUB, {4, 256}, gens);
    const size_t n = 256, L = 32;
    std::vector<uint8_t> leaves(n * L);
    for (size_t i = 0; i < leaves.size(); i++) leaves[i] = (uint8_t)(i * 2654435761u >> 13);
    auto tree = PedersenMerkleTree::create(P, P, leaves, L);
    REQUIRE(tree.height() == 9);

    // a batch with a repeated index (the last occurrence wins) and both ends of the tree
    std::vector<uint64_t> idx = {5, 255, 0, 6, 5, 128};
    std::vector<uint8_t> upd(idx.size() * L);
    for (size_t i = 0; i < upd.size(); i++) upd[i] = (uint8_t)(i * 7 + 3);
    tree.update_batch(P, P, idx, upd, L);
    for (size_t j = 0; j < idx.size(); j++) memcpy(&leaves[idx[j] * L], &upd[j * L], L);
    auto rebuilt = PedersenMerkleTree::create(P, P, leaves, L);
    REQUIRE(same(tree.leaf_nodes, rebuilt.leaf_nodes) && same(tree.non_leaf_nodes, rebuilt.non_leaf_nodes));

    // single update
    std::vector<uint8_t> one(L, 0xA5);
    tree.update(P, P, 77, one);
    memcpy(&leaves[77 * L], one.data(), L);
    rebuilt = PedersenMerkleTree::create(P, P, leaves, L);
    REQUIRE(same(tree.non_leaf_nodes, rebuilt.non_leaf_nodes));

    // check_update: a wrong root changes nothing, the right one applies
    std::vector<uint8_t> two(L, 0x3C);
    std::vector<uint8_t> after = leaves;
    memcpy(&after[200 * L], two.data(), L);
    const Affine good = PedersenMerkleTree::create(P, P, after, L).root();
    Affine bad = good;
    bad.y[0] ^= 1;
    const auto before_nodes = tree.non_leaf_nodes;
    const auto before_leaves = tree.leaf_nodes;
    REQUIRE(!tree.check_update(P, P, 200, two, bad));
    REQUIRE(same(tree.non_leaf_nodes, before_nodes) && same(tree.leaf_nodes, before_leaves));
    REQUIRE(tree.check_update_batch(P, P, {200}, two, L, good));
    const Affine r = tree.root();
    REQUIRE(memcmp(&r, &good, sizeof(Affine)) == 0);

    // host form rules: an index >= n is rejected
    bool threw = false;
    try { tree.update(P, P, n, one); }
    catch (const Error& e) { threw = e.status == CPB_BAD_PARAMS; }
    REQUIRE(threw);
    printf("cpp pedersen update ok\n");
    return 0;
}
