// C++ host-mirror test of Schnorr and ElGamal over ed-on-BLS12-377 (include/cpb200.hpp, schnorr::Parameters and
// elgamal::Parameters with curve CPB_ED_ON_BLS12_377): the signing loop with redrawn nonces at the curve's rejection rate,
// verification of every signature and of the reference benchmark's message ([100u8; 128]), rejection of a changed message /
// signature / key / salt, randomised keys and signatures, and an ElGamal round trip.
#include <cstdio>
#include <cstdlib>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    // Schnorr.setup(SplitMix64(7), ED_ON_BLS12_377).generator, a point of the prime-order subgroup (Montgomery limbs)
    const Affine G{{0x47abd8066538be35ull, 0x19a8bb7efe973a87ull, 0xb911af69a671e707ull, 0x0f7fc427bd0258f7ull},
                   {0x1c455cccb3814955ull, 0xc033ea755a4eda2aull, 0xd723d0b194fe84ccull, 0x0283d74a686f913cull}};
    std::array<uint8_t, 32> salt;
    for (int i = 0; i < 32; i++) salt[i] = (uint8_t)(5 * i + 3);
    schnorr::Parameters P(G, salt, CPB_ED_ON_BLS12_377);
    uint64_t state = 4242;
    auto scalar = [&]() {                                   // a canonical value below 2^249 -> Fr Montgomery limbs
        Fe c, m;
        for (auto& w : c) { state = state * 6364136223846793005ull + 1442695040888963407ull; w = state; }
        c[3] >>= 7;
        check(cpb_field_to_montgomery(CPB_ED_ON_BLS12_377_FR, 0, c.data(), m.data(), 1));
        return m;
    };
    const size_t n = 1024;
    std::vector<Fe> sks(n);
    std::vector<std::vector<uint8_t>> msgs(n);
    for (size_t i = 0; i < n; i++) {
        sks[i] = scalar();
        if (i % 2) msgs[i].assign(128, 100);                // the reference benchmark's message
        else {
            msgs[i].resize(i % 97);
            for (size_t j = 0; j < msgs[i].size(); j++) msgs[i][j] = (uint8_t)(i * 31 + j);
        }
    }
    auto pks = schnorr::Schnorr::keygen_batch(P, sks);

    std::vector<schnorr::Signature> sigs(n);
    std::vector<size_t> todo(n);
    for (size_t i = 0; i < n; i++) todo[i] = i;
    size_t rejected = 0;
    for (int round = 0; !todo.empty(); round++) {
        REQUIRE(round < 40);
        std::vector<Fe> k, sk;
        std::vector<std::vector<uint8_t>> m;
        for (size_t i : todo) { k.push_back(scalar()); sk.push_back(sks[i]); m.push_back(msgs[i]); }
        std::vector<uint8_t> ok;
        auto s = schnorr::Schnorr::sign_with_nonces_batch(P, sk, k, m, ok);
        std::vector<size_t> next;
        for (size_t j = 0; j < todo.size(); j++) {
            if (ok[j]) sigs[todo[j]] = s[j];
            else next.push_back(todo[j]);
        }
        if (round == 0) rejected = next.size();
        todo = next;
    }
    REQUIRE(rejected > n / 4 && rejected < 3 * n / 5);    // about 41.7 %

    auto ok = schnorr::Schnorr::verify_batch(P, pks, msgs, sigs);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == 1);
    auto bad_msgs = msgs;
    bad_msgs[5].push_back(1);
    auto bad_sigs = sigs;
    bad_sigs[6].prover_response = sigs[7].prover_response;
    bad_sigs[8].verifier_challenge = sigs[9].verifier_challenge;
    REQUIRE(!schnorr::Schnorr::verify(P, pks[5], bad_msgs[5], sigs[5]));
    REQUIRE(!schnorr::Schnorr::verify(P, pks[6], msgs[6], bad_sigs[6]));
    REQUIRE(!schnorr::Schnorr::verify(P, pks[8], msgs[8], bad_sigs[8]));
    REQUIRE(!schnorr::Schnorr::verify(P, pks[11], msgs[10], sigs[10]));
    std::array<uint8_t, 32> other_salt = salt;
    other_salt[0] ^= 1;
    schnorr::Parameters P2(G, other_salt, CPB_ED_ON_BLS12_377);
    REQUIRE(!schnorr::Schnorr::verify(P2, pks[12], msgs[12], sigs[12]));
    // the same generator is not a Jubjub point
    bool threw = false;
    try { schnorr::Parameters PJ(G, salt); } catch (const Error&) { threw = true; }
    REQUIRE(threw);

    std::vector<uint8_t> rnd(n * 40);
    for (size_t i = 0; i < rnd.size(); i++) rnd[i] = (uint8_t)(i * 131 + 7);
    auto rpks = schnorr::Schnorr::randomize_public_key_batch(P, pks, rnd.data(), 40);
    auto rsigs = schnorr::Schnorr::randomize_signature_batch(P, sigs, rnd.data(), 40);
    ok = schnorr::Schnorr::verify_batch(P, rpks, msgs, rsigs);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == 1);

    elgamal::Parameters E(G, CPB_ED_ON_BLS12_377);
    std::vector<Fe> r(n), t(n);
    for (size_t i = 0; i < n; i++) { r[i] = scalar(); t[i] = scalar(); }
    auto m = E.mul_batch(t);
    auto cts = elgamal::ElGamal::encrypt_batch(E, pks, m, r);
    auto back = elgamal::ElGamal::decrypt_batch(E, sks, cts);
    for (size_t i = 0; i < n; i++) REQUIRE(back[i].x == m[i].x && back[i].y == m[i].y);
    auto c1 = E.mul_batch(r);
    for (size_t i = 0; i < n; i++) REQUIRE(cts[i].c1.x == c1[i].x && cts[i].c1.y == c1[i].y);
    printf("cpp signature ed377 ok: %zu signers (%zu nonces redrawn), ElGamal\n", n, rejected);
    return 0;
}
