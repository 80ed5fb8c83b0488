// C++ host-mirror test of Schnorr, ElGamal and the Blake2s commitment (include/cpb200.hpp over cpb_te_base_*, cpb_schnorr_*,
// cpb_elgamal_*, cpb_blake2s_commit_*): the signing loop with redrawn nonces, verification of every signature, rejection of a
// changed message / signature / key, randomised keys and signatures, an ElGamal round trip, and a commitment against hashlib.
#include <cstdio>
#include <cstdlib>
#include "cpb200.hpp"
using namespace cpb;

#define REQUIRE(c) do { if (!(c)) { fprintf(stderr, "FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main() {
    // Schnorr.setup(SplitMix64(7)).generator, a point of the prime-order subgroup (Montgomery limbs)
    const Affine G{{0xecf14e67d26f017aull, 0x548401714d5db025ull, 0xf33bc5cca566d965ull, 0x4f622a74b5d412f8ull},
                   {0xd809093521bd4c26ull, 0x5495e3237e0a8570ull, 0xb8671c9a523a3818ull, 0x1efe6681d8b3537eull}};
    std::array<uint8_t, 32> salt;
    for (int i = 0; i < 32; i++) salt[i] = (uint8_t)(7 * i + 1);
    schnorr::Parameters P(G, salt);
    uint64_t state = 12345;
    auto scalar = [&]() {                                   // a canonical value below 2^250 -> Fr Montgomery limbs
        Fe c, m;
        for (auto& w : c) { state = state * 6364136223846793005ull + 1442695040888963407ull; w = state; }
        c[3] >>= 6;
        check(cpb_field_to_montgomery(CPB_JUBJUB_FR, 0, c.data(), m.data(), 1));
        return m;
    };
    const size_t n = 512;
    std::vector<Fe> sks(n), nonces(n);
    std::vector<std::vector<uint8_t>> msgs(n);
    for (size_t i = 0; i < n; i++) {
        sks[i] = scalar();
        msgs[i].resize(i % 97);
        for (size_t j = 0; j < msgs[i].size(); j++) msgs[i][j] = (uint8_t)(i * 31 + j);
    }
    auto pks = schnorr::Schnorr::keygen_batch(P, sks);

    // the reference's loop, per batch: redraw the nonces whose challenge is not a field element
    std::vector<schnorr::Signature> sigs(n);
    std::vector<size_t> todo(n);
    for (size_t i = 0; i < n; i++) todo[i] = i;
    size_t rejected = 0;
    for (int round = 0; !todo.empty(); round++) {
        REQUIRE(round < 20);
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
    REQUIRE(rejected > 0 && rejected < n / 4);              // about 9.4 %

    auto ok = schnorr::Schnorr::verify_batch(P, pks, msgs, sigs);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == 1);
    // a changed message, response, challenge or key fails
    auto bad_msgs = msgs;
    bad_msgs[5].push_back(1);
    auto bad_sigs = sigs;
    bad_sigs[6].prover_response = sigs[7].prover_response;
    bad_sigs[8].verifier_challenge = sigs[9].verifier_challenge;
    auto bad_pks = pks;
    bad_pks[10] = pks[11];
    REQUIRE(!schnorr::Schnorr::verify(P, pks[5], bad_msgs[5], sigs[5]));
    REQUIRE(!schnorr::Schnorr::verify(P, pks[6], msgs[6], bad_sigs[6]));
    REQUIRE(!schnorr::Schnorr::verify(P, pks[8], msgs[8], bad_sigs[8]));
    REQUIRE(!schnorr::Schnorr::verify(P, bad_pks[10], msgs[10], sigs[10]));
    std::array<uint8_t, 32> other_salt = salt;
    other_salt[0] ^= 1;
    schnorr::Parameters P2(G, other_salt);
    REQUIRE(!schnorr::Schnorr::verify(P2, pks[12], msgs[12], sigs[12]));

    // randomised keys and signatures still verify (R/signature/mod.rs:80-105)
    std::vector<uint8_t> rnd(n * 40);
    for (size_t i = 0; i < rnd.size(); i++) rnd[i] = (uint8_t)(i * 131 + 7);
    auto rpks = schnorr::Schnorr::randomize_public_key_batch(P, pks, rnd.data(), 40);
    auto rsigs = schnorr::Schnorr::randomize_signature_batch(P, sigs, rnd.data(), 40);
    ok = schnorr::Schnorr::verify_batch(P, rpks, msgs, rsigs);
    for (size_t i = 0; i < n; i++) REQUIRE(ok[i] == 1);

    // ElGamal: decrypt(encrypt(m)) = m
    elgamal::Parameters E(G);
    std::vector<Fe> r(n), t(n);
    for (size_t i = 0; i < n; i++) { r[i] = scalar(); t[i] = scalar(); }
    auto m = E.mul_batch(t);
    auto cts = elgamal::ElGamal::encrypt_batch(E, pks, m, r);
    auto back = elgamal::ElGamal::decrypt_batch(E, sks, cts);
    for (size_t i = 0; i < n; i++) REQUIRE(back[i].x == m[i].x && back[i].y == m[i].y);
    auto c1 = E.mul_batch(r);
    for (size_t i = 0; i < n; i++) REQUIRE(cts[i].c1.x == c1[i].x && cts[i].c1.y == c1[i].y);

    // Blake2s commitment: Blake2s256("abc" || 0, 1, ..., 31)
    std::array<uint8_t, 32> r32;
    for (int i = 0; i < 32; i++) r32[i] = (uint8_t)i;
    auto cm = blake2s::Commitment::commit_batch({{'a', 'b', 'c'}, {}}, {r32, r32});
    const char* hex = "e0f7bc605522dd045ccd1954b126f0900edac1411fe3a003d999438ba30b6434";
    for (int i = 0; i < 32; i++) REQUIRE(cm[0][i] == (uint8_t)strtoul(std::string(hex + 2 * i, 2).c_str(), nullptr, 16));
    REQUIRE(cm[1] != cm[0]);
    printf("cpp signature ok: %zu signers (%zu nonces redrawn), ElGamal and Blake2s\n", n, rejected);
    return 0;
}
