// C++ host-mirror test of the batched duplex sponges (include/cpb200.hpp, poseidon::PoseidonSpongeBatch over the C-ABI): the
// reference's sponge KAT in every sponge of a batch, agreement with the one-shot sponge batch, the mode rules, broadcast byte
// strings against per-sponge copies, and the argument checks.  Prints the KAT squeeze of sponge 0 for tests/test_gpu_poseidon_duplex.py.
#include <cstdio>
#include <cstdlib>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

static std::vector<Fe> mont(const std::vector<Fe>& canon) {
    std::vector<Fe> out(canon.size());
    if (!canon.empty()) check(cpb_field_to_montgomery(CPB_BLS12_381_FR, 0, canon[0].data(), out[0].data(), canon.size()));
    return out;
}

int main() {
    auto params = poseidon::Config::get_default_poseidon_parameters(CPB_BLS12_381_FR, 2, false);
    REQUIRE(params);
    const poseidon::Config& P = *params;
    const size_t n = 7;

    // R/sponge/poseidon/mod.rs:381-404: absorb [0, 1, 2], squeeze 3 -- in every sponge
    std::vector<Fe> canon;
    for (size_t i = 0; i < n; i++)
        for (uint64_t k = 0; k < 3; k++) canon.push_back(Fe{k, 0, 0, 0});
    poseidon::PoseidonSpongeBatch b(P, n);
    b.absorb(mont(canon));
    REQUIRE(b.mode().squeezing == 0 && b.mode().index == 1);               // 3 elements at rate 2: one permutation, lane 0 of block 2
    std::vector<Fe> sq = b.squeeze_canonical(3);
    REQUIRE(b.mode().squeezing == 1 && b.mode().index == 1);
    for (size_t i = 1; i < n; i++)
        for (size_t j = 0; j < 3; j++) REQUIRE(sq[3 * i + j] == sq[j]);

    // the same sponges through the one-shot batch: new -> absorb(x_i) -> squeeze(3)
    std::vector<Fe> xs;
    for (size_t i = 0; i < n; i++)
        for (uint64_t k = 0; k < 5; k++) xs.push_back(Fe{31 * i + k + 1, 0, 0, 0});
    std::vector<Fe> xm = mont(xs), one_shot(n * 3);
    check(cpb_poseidon_sponge_batch(P.ctx(), xm[0].data(), 5, one_shot[0].data(), 3, n));
    poseidon::PoseidonSpongeBatch c(P, n);
    c.absorb(xm);
    REQUIRE(c.squeeze_native_field_elements(3) == one_shot);

    // absorb after squeeze starts at lane 0 without a permutation; squeeze(0) keeps the index
    c.absorb(std::vector<Fe>(xm.begin(), xm.begin() + n));
    REQUIRE(c.mode().squeezing == 0 && c.mode().index == 1);
    c.squeeze_native_field_elements(0);
    REQUIRE(c.mode().squeezing == 1 && c.mode().index == 0);

    // one broadcast byte string == the same string given to every sponge; the empty string absorbs its length prefix only
    std::vector<uint8_t> msg(40), copies;
    for (size_t i = 0; i < msg.size(); i++) msg[i] = (uint8_t)(7 * i + 3);
    for (size_t i = 0; i < n; i++) copies.insert(copies.end(), msg.begin(), msg.end());
    poseidon::PoseidonSpongeBatch d(P, n), e(P, n);
    d.absorb_bytes(msg, msg.size(), 0);
    e.absorb_bytes(copies, msg.size(), msg.size());
    d.absorb_bytes({}, 0, 0);
    e.absorb_bytes({}, 0, 0);
    REQUIRE(d.states() == e.states() && d.mode().index == e.mode().index);
    REQUIRE(d.squeeze_native_field_elements(4) == e.squeeze_native_field_elements(4));

    // argument checks: a mode index past the rate, a squeezing flag outside {0, 1}, a null buffer that is read
    std::vector<Fe> st(3 * n);
    cpb_sponge_mode bad{0, 3};
    REQUIRE(cpb_poseidon_duplex_absorb(P.ctx(), st[0].data(), &bad, xm[0].data(), 1, n) == CPB_BAD_PARAMS);
    bad = cpb_sponge_mode{2, 0};
    REQUIRE(cpb_poseidon_duplex_squeeze(P.ctx(), st[0].data(), &bad, st[0].data(), 1, 0, n) == CPB_BAD_PARAMS);
    cpb_sponge_mode ok{0, 0};
    REQUIRE(cpb_poseidon_duplex_absorb_bytes(P.ctx(), st[0].data(), &ok, nullptr, 4, 4, n) == CPB_NULL_POINTER);
    REQUIRE(ok.squeezing == 0 && ok.index == 0);

    printf("squeeze3[0] = %016llx%016llx%016llx%016llx\n", (unsigned long long)sq[0][3], (unsigned long long)sq[0][2],
           (unsigned long long)sq[0][1], (unsigned long long)sq[0][0]);
    printf("duplex cpp ok\n");
    return 0;
}
