// C++ host-mirror test of the Pedersen byte-tree path verification (include/cpb200.hpp over cpb_merkle_pedersen_verify_batch): every
// leaf of a PedersenMerkleTree verifies against its root, a changed leaf or a changed root fails, a leaf over the window throws.
// argv[1]: the 4 x 256 Jubjub generators, affine (x, y) Montgomery limbs, 64 bytes each (written by the calling test).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

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
    const auto tree = PedersenMerkleTree::create(P, P, leaves, L);
    REQUIRE(tree.height() == 9);

    std::vector<size_t> all(n);
    for (size_t i = 0; i < n; i++) all[i] = i;
    auto ok = tree.verify_batch(P, P, tree.root(), all, leaves, L);
    REQUIRE(ok.size() == n);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == 1);

    // claimed leaves that are not the tree's: leaf 3 under index 7, and a flipped bit in leaf 200's
    std::vector<size_t> some = {7, 200, 0};
    std::vector<uint8_t> claimed(some.size() * L);
    memcpy(&claimed[0], &leaves[3 * L], L);
    memcpy(&claimed[L], &leaves[200 * L], L);
    claimed[L + 5] ^= 1;
    memcpy(&claimed[2 * L], &leaves[0], L);
    ok = tree.verify_batch(P, P, tree.root(), some, claimed, L);
    REQUIRE(ok[0] == 0 && ok[1] == 0 && ok[2] == 1);

    // another root: both coordinates are compared
    Affine bad = tree.root();
    bad.y[0] ^= 1;
    ok = tree.verify_batch(P, P, bad, all, leaves, L);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == 0);

    // a leaf longer than the 1024-bit window
    bool threw = false;
    try { tree.verify_batch(P, P, tree.root(), {0}, std::vector<uint8_t>(129), 129); }
    catch (const Error& e) { threw = e.status == CPB_BAD_LENGTH; }
    REQUIRE(threw);
    printf("cpp pedersen verify ok\n");
    return 0;
}
