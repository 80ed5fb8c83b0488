// C++ host-mirror test of the ragged duplex calls (include/cpb200.hpp, poseidon::RaggedPoseidonSpongeBatch over the C-ABI): the
// reference's sponge KAT through an n = 1 ragged batch, equal spans against the uniform batch, a mixed-length transcript from the copy
// of a uniform batch in which each sponge gives the same result when it is the only one with data, and the argument checks.  Prints the KAT squeeze for
// tests/test_gpu_poseidon_duplex_ragged.py.
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
static std::vector<uint64_t> offsets_of(const std::vector<size_t>& lens, uint64_t base = 0) {
    std::vector<uint64_t> off(1, base);
    for (size_t l : lens) off.push_back(off.back() + l);
    return off;
}

int main() {
    auto params = poseidon::Config::get_default_poseidon_parameters(CPB_BLS12_381_FR, 2, false);
    REQUIRE(params);
    const poseidon::Config& P = *params;

    // R/sponge/poseidon/mod.rs:381-404: absorb [0, 1, 2], squeeze 3, through an n = 1 ragged batch
    poseidon::RaggedPoseidonSpongeBatch k(P, 1);
    k.absorb(mont({Fe{0, 0, 0, 0}, Fe{1, 0, 0, 0}, Fe{2, 0, 0, 0}}), {0, 3});
    REQUIRE(k.modes()[0].squeezing == 0 && k.modes()[0].index == 1);
    const std::vector<Fe> sq = k.squeeze({0, 3}, true);
    REQUIRE(k.modes()[0].squeezing == 1 && k.modes()[0].index == 1);

    // equal spans: exactly the uniform batch, for every call kind
    const size_t n = 7;
    std::vector<Fe> xs;
    for (size_t i = 0; i < n; i++)
        for (uint64_t j = 0; j < 5; j++) xs.push_back(Fe{31 * i + j + 1, 0, 0, 0});
    const std::vector<Fe> xm = mont(xs);
    std::vector<uint8_t> msg(n * 40);
    for (size_t i = 0; i < msg.size(); i++) msg[i] = (uint8_t)(7 * i + 3);
    poseidon::PoseidonSpongeBatch u(P, n);
    poseidon::RaggedPoseidonSpongeBatch r(P, n);
    u.absorb(xm);
    r.absorb(xm, offsets_of(std::vector<size_t>(n, 5)));
    REQUIRE(u.squeeze_native_field_elements(3) == r.squeeze(offsets_of(std::vector<size_t>(n, 3)), false));
    u.absorb_bytes(msg, 40, 40);
    r.absorb_bytes(msg, offsets_of(std::vector<size_t>(n, 40)));
    REQUIRE(u.squeeze_canonical(2) == r.squeeze(offsets_of(std::vector<size_t>(n, 2)), true));
    REQUIRE(u.states() == r.states());
    for (const cpb_sponge_mode& m : r.modes()) REQUIRE(m.squeezing == u.mode().squeezing && m.index == u.mode().index);

    // the copy of a uniform batch continues with different lengths per sponge; sponge i gives the same result when it is the only
    // sponge with data (the others then absorb empty strings and squeeze nothing)
    poseidon::RaggedPoseidonSpongeBatch c(P, u);
    const std::vector<size_t> alen{0, 1, 2, 3, 4, 5, 2}, blen{0, 9, 31, 50, 1, 23, 70}, slen{0, 1, 2, 3, 4, 5, 1};
    std::vector<uint8_t> bytes(200);
    for (size_t i = 0; i < bytes.size(); i++) bytes[i] = (uint8_t)(i * 13 + 1);
    const std::vector<uint64_t> ao = offsets_of(alen, 2), bo = offsets_of(blen), so = offsets_of(slen);
    c.absorb_bytes(bytes, bo);
    c.absorb(xm, ao);
    const std::vector<Fe> out = c.squeeze(so, false);
    const size_t t = 3;
    for (size_t i = 0; i < n; i++) {
        poseidon::RaggedPoseidonSpongeBatch alone(P, u);
        std::vector<uint64_t> ob(n + 1, bo[i]), oa(n + 1, ao[i]), os(n + 1, so[i]);
        for (size_t j = i + 1; j <= n; j++) ob[j] = bo[i + 1], oa[j] = ao[i + 1], os[j] = so[i + 1];
        alone.absorb_bytes(bytes, ob);
        alone.absorb(xm, oa);
        const std::vector<Fe> o = alone.squeeze(os, false);
        for (size_t e = so[i]; e < so[i + 1]; e++) REQUIRE(o[e] == out[e]);
        for (size_t w = 0; w < t; w++) REQUIRE(alone.states()[i * t + w] == c.states()[i * t + w]);
        REQUIRE(alone.modes()[i].squeezing == c.modes()[i].squeezing && alone.modes()[i].index == c.modes()[i].index);
    }

    // argument checks: a mode index past the rate, a squeezing flag outside {0, 1}, decreasing offsets; a refused call changes nothing
    std::vector<Fe> st(3 * 2);
    std::vector<uint64_t> off{0, 1, 2};
    cpb_sponge_mode modes[2] = {{0, 0}, {0, 3}};
    REQUIRE(cpb_poseidon_duplex_absorb_ragged(P.ctx(), st[0].data(), modes, xm[0].data(), off.data(), 2) == CPB_BAD_PARAMS);
    modes[1] = cpb_sponge_mode{2, 0};
    REQUIRE(cpb_poseidon_duplex_squeeze_ragged(P.ctx(), st[0].data(), modes, st[0].data(), off.data(), 0, 2) == CPB_BAD_PARAMS);
    modes[1] = cpb_sponge_mode{0, 0};
    std::vector<uint64_t> dec{0, 2, 1};
    REQUIRE(cpb_poseidon_duplex_absorb_ragged(P.ctx(), st[0].data(), modes, xm[0].data(), dec.data(), 2) == CPB_BAD_LENGTH);
    REQUIRE(modes[0].index == 0 && modes[1].index == 0 && st == std::vector<Fe>(6));

    printf("squeeze3[0] = %016llx%016llx%016llx%016llx\n", (unsigned long long)sq[0][3], (unsigned long long)sq[0][2],
           (unsigned long long)sq[0][1], (unsigned long long)sq[0][0]);
    printf("duplex ragged cpp ok\n");
    return 0;
}
