// cpb200.hpp -- header-only C++ mirror of the reference's scheme interface over the C-ABI (cpb200.h).
//
// The reference is Rust; where no Rust toolchain exists this is the compiled-language host side:
// the same associated-function shape as the traits it mirrors (parameters first, stateless),
//   CRHScheme / TwoToOneCRHScheme   R/crh/mod.rs:18-51
//   CommitmentScheme                R/commitment/mod.rs:15-27
//   merkle_tree::MerkleTree         R/merkle_tree/mod.rs:381-533
// with batch entry points beside the single-shot ones (a GPU is amortised only over a batch).
// Errors: the reference's panics / Err become cpb::Error (std::runtime_error with the status).
// Elements are cpb::Fe = 4 x uint64_t Montgomery limbs (the memory image of ark-ff's Fp256).
#pragma once
#include <array>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "cpb200.h"

namespace cpb {

using Fe = std::array<uint64_t, 4>;
struct Affine { Fe x, y; };

struct Error : std::runtime_error {
    cpb_status status;
    Error(cpb_status s, const std::string& m) : std::runtime_error(m), status(s) {}
};
inline void check(cpb_status s) {
    if (s != CPB_OK) throw Error(s, std::string("cpb status ") + std::to_string((int)s) + ": " + cpb_last_error());
}

// Inputs of different lengths (Vec<Vec<F>>) as the C-ABI's ragged batch: the elements back to back plus n + 1 offsets.
inline void ragged_pack(const std::vector<std::vector<Fe>>& inputs, std::vector<Fe>& values, std::vector<uint64_t>& offsets) {
    offsets.assign(1, 0);
    values.clear();
    for (const auto& x : inputs) {
        values.insert(values.end(), x.begin(), x.end());
        offsets.push_back(values.size());
    }
}
inline bool equal_lengths(const std::vector<std::vector<Fe>>& inputs) {
    for (const auto& x : inputs)
        if (x.size() != inputs[0].size()) return false;
    return true;
}

namespace poseidon {

// PoseidonConfig<F> (R/sponge/poseidon/mod.rs:26-45) + the device context built from it.
class Config {
public:
    int field_id, full_rounds, partial_rounds, rate, capacity;
    uint64_t alpha;
    std::vector<Fe> ark, mds;   // ark[round * t + i], mds[i * t + j]

    // PoseidonConfig::new (mod.rs:189-217)
    Config(int field, int full_rounds_, int partial_rounds_, uint64_t alpha_, std::vector<Fe> mds_, std::vector<Fe> ark_, int rate_,
           int capacity_, int device = 0)
        : field_id(field), full_rounds(full_rounds_), partial_rounds(partial_rounds_), rate(rate_), capacity(capacity_), alpha(alpha_),
          ark(std::move(ark_)), mds(std::move(mds_)) {
        const size_t t = (size_t)rate + capacity;
        if (ark.size() != (size_t)(full_rounds + partial_rounds) * t || mds.size() != t * t)
            throw Error(CPB_BAD_PARAMS, "PoseidonConfig::new: ark/mds shape");
        cpb_poseidon_ctx* c = nullptr;
        check(cpb_poseidon_ctx_create(field, rate, capacity, full_rounds, partial_rounds, alpha, ark[0].data(), mds[0].data(), device, &c));
        ctx_.reset(c, cpb_poseidon_ctx_destroy);
    }
    // PoseidonDefaultConfigField::get_default_poseidon_parameters (traits.rs:59-103); nullptr where the reference returns None.
    static std::unique_ptr<Config> get_default_poseidon_parameters(int field, int rate, bool optimized_for_weights, int device = 0) {
        uint64_t alpha; int rf, rp, skip;
        if (cpb_poseidon_default_entry(field, rate, optimized_for_weights, &alpha, &rf, &rp, &skip) != CPB_OK) return nullptr;
        uint64_t mod[4];
        check(cpb_field_modulus(field, mod));
        uint64_t bits = 256;
        while (bits && !((mod[(bits - 1) / 64] >> ((bits - 1) % 64)) & 1)) bits--;
        const size_t t = (size_t)rate + 1;
        std::vector<Fe> ark((size_t)(rf + rp) * t), mds(t * t);
        check(cpb_poseidon_find_ark_and_mds(field, bits, rate, rf, rp, skip, ark[0].data(), mds[0].data()));
        return std::unique_ptr<Config>(new Config(field, rf, rp, alpha, std::move(mds), std::move(ark), rate, 1, device));
    }
    cpb_poseidon_ctx* ctx() const { return ctx_.get(); }

private:
    std::shared_ptr<cpb_poseidon_ctx> ctx_;
};

// crh::poseidon::CRH (R/crh/poseidon/mod.rs:15-41)
struct CRH {
    using Parameters = Config;
    static Fe evaluate(const Parameters& p, const std::vector<Fe>& input) {
        Fe out;
        check(cpb_poseidon_crh_batch(p.ctx(), input.empty() ? nullptr : input[0].data(), input.size(), out.data(), 1));
        return out;
    }
    // n inputs of `len` elements each, contiguous
    static std::vector<Fe> evaluate_batch(const Parameters& p, const std::vector<Fe>& inputs, size_t len) {
        const size_t n = len ? inputs.size() / len : 0;
        std::vector<Fe> out(n);
        if (n) check(cpb_poseidon_crh_batch(p.ctx(), inputs[0].data(), len, out[0].data(), n));
        return out;
    }
    // n inputs of any lengths, each hashed at its own length (one ragged call; equal lengths take the uniform call)
    static std::vector<Fe> evaluate_batch(const Parameters& p, const std::vector<std::vector<Fe>>& inputs) {
        std::vector<Fe> out(inputs.size());
        if (inputs.empty()) return out;
        std::vector<Fe> values;
        std::vector<uint64_t> offsets;
        ragged_pack(inputs, values, offsets);
        if (equal_lengths(inputs) && !inputs[0].empty())
            check(cpb_poseidon_crh_batch(p.ctx(), values[0].data(), inputs[0].size(), out[0].data(), out.size()));
        else
            check(cpb_poseidon_crh_ragged_batch(p.ctx(), values.empty() ? nullptr : values[0].data(), offsets.data(), out[0].data(), out.size()));
        return out;
    }
};

// crh::poseidon::TwoToOneCRH (mod.rs:43-80); evaluate == compress (:58-64)
struct TwoToOneCRH {
    using Parameters = Config;
    static Fe compress(const Parameters& p, const Fe& left, const Fe& right) {
        Fe pair[2] = {left, right}, out;
        check(cpb_poseidon_compress_batch(p.ctx(), pair[0].data(), out.data(), 1));
        return out;
    }
    static Fe evaluate(const Parameters& p, const Fe& left, const Fe& right) { return compress(p, left, right); }
    static std::vector<Fe> compress_batch(const Parameters& p, const std::vector<Fe>& pairs) {
        std::vector<Fe> out(pairs.size() / 2);
        if (!out.empty()) check(cpb_poseidon_compress_batch(p.ctx(), pairs[0].data(), out[0].data(), out.size()));
        return out;
    }
};

}  // namespace poseidon

namespace pedersen {

struct Window { int WINDOW_SIZE, NUM_WINDOWS; };   // R/crh/pedersen/mod.rs:23-26

// pedersen::Parameters (mod.rs:28-31) [+ randomness_generator, R/commitment/pedersen/mod.rs:17-21]
class Parameters {
public:
    Window window;
    Parameters(int curve, Window w, const std::vector<Affine>& generators, const std::vector<Affine>& randomness_generator = {}, int device = 0)
        : window(w) {
        if (generators.size() != (size_t)w.WINDOW_SIZE * w.NUM_WINDOWS) throw Error(CPB_BAD_PARAMS, "Incorrect pp size for window params");
        cpb_pedersen_ctx* c = nullptr;
        check(cpb_pedersen_ctx_create(curve, w.WINDOW_SIZE, w.NUM_WINDOWS, generators[0].x.data(), randomness_generator.size(),
                                      randomness_generator.empty() ? nullptr : randomness_generator[0].x.data(), device, &c));
        ctx_.reset(c, cpb_pedersen_ctx_destroy);
    }
    cpb_pedersen_ctx* ctx() const { return ctx_.get(); }

private:
    std::shared_ptr<cpb_pedersen_ctx> ctx_;
};

struct CRH {   // mod.rs:58-130
    static Affine evaluate(const Parameters& p, const std::vector<uint8_t>& input) {
        Affine out;
        check(cpb_pedersen_crh_batch(p.ctx(), input.data(), input.size(), input.size(), out.x.data(), 1));
        return out;
    }
    static std::vector<Affine> evaluate_batch(const Parameters& p, const uint8_t* inputs, size_t len, size_t n) {
        std::vector<Affine> out(n);
        if (n) check(cpb_pedersen_crh_batch(p.ctx(), inputs, len, len, out[0].x.data(), n));
        return out;
    }
};
struct TwoToOneCRH {   // mod.rs:132-198
    static Affine compress(const Parameters& p, const Affine& l, const Affine& r) {
        Affine kids[2] = {l, r}, out;
        check(cpb_pedersen_two_to_one_batch(p.ctx(), kids[0].x.data(), out.x.data(), 1));
        return out;
    }
};
struct Commitment {   // R/commitment/pedersen/mod.rs:38-106; randomness = 32-byte LE canonical scalar
    static Affine commit(const Parameters& p, const std::vector<uint8_t>& input, const std::array<uint8_t, 32>& randomness) {
        Affine out;
        check(cpb_pedersen_commit_batch(p.ctx(), input.data(), input.size(), input.size(), randomness.data(), out.x.data(), 1));
        return out;
    }
};

}  // namespace pedersen

// MerkleTree of JubJubMerkleTreeParams (R/merkle_tree/tests/mod.rs:19-33): byte leaves, pedersen::CRH leaf hash, ByteDigestConverter,
// pedersen::TwoToOneCRH inner nodes.  Digests are affine points.
class PedersenMerkleTree {
public:
    std::vector<Affine> leaf_nodes, non_leaf_nodes;   // the reference's two arrays (mod.rs:383-395)

    // n leaves of leaf_len bytes each, back to back
    static PedersenMerkleTree create(const pedersen::Parameters& leaf, const pedersen::Parameters& two_to_one, const std::vector<uint8_t>& leaves,
                                     size_t leaf_len) {
        PedersenMerkleTree t;
        const size_t n = leaf_len ? leaves.size() / leaf_len : 0;
        t.leaf_nodes.resize(n);
        t.non_leaf_nodes.resize(n ? n - 1 : 0);
        check(cpb_merkle_pedersen_build(leaf.ctx(), two_to_one.ctx(), leaves.empty() ? nullptr : leaves.data(), leaf_len, n,
                                        n ? t.leaf_nodes[0].x.data() : nullptr, n > 1 ? t.non_leaf_nodes[0].x.data() : nullptr));
        return t;
    }
    Affine root() const { return non_leaf_nodes.at(0); }
    size_t height() const {
        size_t h = 1, n = leaf_nodes.size();
        while (n > 1) { n >>= 1; h++; }
        return h;
    }

    // k x MerkleTree::update (mod.rs:690-701) in one call: leaf indexes[i] becomes leaves[i * leaf_len .. (i+1) * leaf_len) (bytes); a
    // repeated index takes its last leaf.  Only the touched nodes and the siblings they read cross PCIe.
    void update_batch(const pedersen::Parameters& leaf, const pedersen::Parameters& two_to_one, const std::vector<uint64_t>& indexes,
                      const std::vector<uint8_t>& leaves, size_t leaf_len) {
        update_impl(leaf, two_to_one, indexes, leaves, leaf_len, nullptr);
    }
    void update(const pedersen::Parameters& leaf, const pedersen::Parameters& two_to_one, size_t index, const std::vector<uint8_t>& new_leaf) {
        update_batch(leaf, two_to_one, {(uint64_t)index}, new_leaf, new_leaf.size());
    }
    // check_update (mod.rs:706-725) for all k at once: the tree changes only when the new root equals asserted_new_root.
    bool check_update_batch(const pedersen::Parameters& leaf, const pedersen::Parameters& two_to_one, const std::vector<uint64_t>& indexes,
                            const std::vector<uint8_t>& leaves, size_t leaf_len, const Affine& asserted_new_root) {
        return update_impl(leaf, two_to_one, indexes, leaves, leaf_len, &asserted_new_root);
    }
    bool check_update(const pedersen::Parameters& leaf, const pedersen::Parameters& two_to_one, size_t index, const std::vector<uint8_t>& new_leaf,
                      const Affine& asserted_new_root) {
        return check_update_batch(leaf, two_to_one, {(uint64_t)index}, new_leaf, new_leaf.size(), asserted_new_root);
    }

private:
    bool update_impl(const pedersen::Parameters& leaf, const pedersen::Parameters& two_to_one, const std::vector<uint64_t>& indexes,
                     const std::vector<uint8_t>& leaves, size_t leaf_len, const Affine* asserted) {
        const size_t k = indexes.size();
        if (leaves.size() != k * leaf_len) throw Error(CPB_BAD_LENGTH, "one leaf of leaf_len bytes per index");
        int applied = 0;
        check(cpb_merkle_pedersen_update(leaf.ctx(), two_to_one.ctx(), leaf_nodes.empty() ? nullptr : leaf_nodes[0].x.data(),
                                         non_leaf_nodes.empty() ? nullptr : non_leaf_nodes[0].x.data(), leaf_nodes.size(), indexes.data(),
                                         leaves.empty() ? nullptr : leaves.data(), leaf_len, k, asserted ? asserted->x.data() : nullptr, &applied));
        return applied != 0;
    }
};

// Byte strings of different lengths as the C-ABI's ragged batch: the bytes back to back plus n + 1 offsets.
inline void ragged_pack(const std::vector<std::vector<uint8_t>>& inputs, std::vector<uint8_t>& values, std::vector<uint64_t>& offsets) {
    offsets.assign(1, 0);
    values.clear();
    for (const auto& x : inputs) {
        values.insert(values.end(), x.begin(), x.end());
        offsets.push_back(values.size());
    }
    values.push_back(0);                                  // never empty, so data() is a valid pointer
}

// Parameters{generator} shared by Schnorr and ElGamal over Jubjub, with the generator's fixed-base tables on the device.
class TeBase {
public:
    Affine generator;
    explicit TeBase(const Affine& g, int curve = CPB_JUBJUB, int device = 0) : generator(g) {
        cpb_te_base_ctx* c = nullptr;
        check(cpb_te_base_ctx_create(curve, g.x.data(), device, &c));
        ctx_.reset(c, cpb_te_base_ctx_destroy);
    }
    cpb_te_base_ctx* ctx() const { return ctx_.get(); }
    // keygen of both schemes: scalars[i] * generator (Fr Montgomery limbs)
    std::vector<Affine> mul_batch(const std::vector<Fe>& scalars) const {
        std::vector<Affine> out(scalars.size());
        if (!scalars.empty()) check(cpb_te_base_mul_batch(ctx(), scalars[0].data(), out[0].x.data(), scalars.size()));
        return out;
    }

private:
    std::shared_ptr<cpb_te_base_ctx> ctx_;
};

namespace schnorr {   // Schnorr<Jubjub, Blake2s256>, R/signature/schnorr/mod.rs; SignatureScheme, R/signature/mod.rs:14-50

struct Signature { Fe prover_response, verifier_challenge; };

// schnorr::Parameters{generator, salt} (mod.rs:24-29)
struct Parameters {
    TeBase base;
    std::array<uint8_t, 32> salt;
    Parameters(const Affine& generator, const std::array<uint8_t, 32>& salt_, int device = 0) : base(generator, CPB_JUBJUB, device), salt(salt_) {}
};

struct Schnorr {
    static std::vector<Affine> keygen_batch(const Parameters& p, const std::vector<Fe>& secret_keys) { return p.base.mul_batch(secret_keys); }
    // One iteration of the signing loop (mod.rs:87-104) per item with the given nonce; signed[i] = 0 when the challenge is not
    // a field element -- draw a new nonce for that item.
    static std::vector<Signature> sign_with_nonces_batch(const Parameters& p, const std::vector<Fe>& sks, const std::vector<Fe>& nonces,
                                                         const std::vector<std::vector<uint8_t>>& messages, std::vector<uint8_t>& signed_out) {
        const size_t n = sks.size();
        if (nonces.size() != n || messages.size() != n) throw Error(CPB_BAD_LENGTH, "sign: one nonce and one message per key");
        std::vector<uint8_t> values;
        std::vector<uint64_t> offsets;
        ragged_pack(messages, values, offsets);
        std::vector<Signature> out(n);
        signed_out.assign(n, 0);
        if (n) check(cpb_schnorr_sign_batch(p.base.ctx(), p.salt.data(), sks[0].data(), nonces[0].data(), values.data(), offsets.data(),
                                            out[0].prover_response.data(), signed_out.data(), n));
        return out;
    }
    // mod.rs:117-148
    static std::vector<uint8_t> verify_batch(const Parameters& p, const std::vector<Affine>& pks, const std::vector<std::vector<uint8_t>>& messages,
                                             const std::vector<Signature>& sigs) {
        const size_t n = pks.size();
        if (messages.size() != n || sigs.size() != n) throw Error(CPB_BAD_LENGTH, "verify: one message and one signature per key");
        std::vector<uint8_t> values, ok(n);
        std::vector<uint64_t> offsets;
        ragged_pack(messages, values, offsets);
        if (n) check(cpb_schnorr_verify_batch(p.base.ctx(), p.salt.data(), pks[0].x.data(), values.data(), offsets.data(),
                                              sigs[0].prover_response.data(), ok.data(), n));
        return ok;
    }
    static bool verify(const Parameters& p, const Affine& pk, const std::vector<uint8_t>& message, const Signature& sig) {
        return verify_batch(p, {pk}, {message}, {sig})[0] != 0;
    }
    // mod.rs:150-174; randomness: n x len bytes
    static std::vector<Affine> randomize_public_key_batch(const Parameters& p, const std::vector<Affine>& pks, const uint8_t* randomness, size_t len) {
        std::vector<Affine> out(pks.size());
        if (!pks.empty())
            check(cpb_schnorr_randomize_public_key_batch(p.base.ctx(), pks[0].x.data(), randomness, len, len, out[0].x.data(), pks.size()));
        return out;
    }
    // mod.rs:176-198
    static std::vector<Signature> randomize_signature_batch(const Parameters& p, const std::vector<Signature>& sigs, const uint8_t* randomness,
                                                            size_t len) {
        std::vector<Signature> out(sigs.size());
        if (!sigs.empty())
            check(cpb_schnorr_randomize_signature_batch(p.base.ctx(), sigs[0].prover_response.data(), randomness, len, len,
                                                        out[0].prover_response.data(), sigs.size()));
        return out;
    }
};

}  // namespace schnorr

namespace elgamal {   // ElGamal<Jubjub>, R/encryption/elgamal/mod.rs; AsymmetricEncryptionScheme

struct Ciphertext { Affine c1, c2; };
using Parameters = TeBase;   // elgamal::Parameters{generator} (mod.rs:14-16)

struct ElGamal {
    // mod.rs:69-84
    static std::vector<Ciphertext> encrypt_batch(const Parameters& p, const std::vector<Affine>& pks, const std::vector<Affine>& msgs,
                                                 const std::vector<Fe>& rands) {
        const size_t n = pks.size();
        if (msgs.size() != n || rands.size() != n) throw Error(CPB_BAD_LENGTH, "encrypt: one message and one randomness per key");
        std::vector<Ciphertext> out(n);
        if (n) check(cpb_elgamal_encrypt_batch(p.ctx(), pks[0].x.data(), msgs[0].x.data(), rands[0].data(), out[0].c1.x.data(), n));
        return out;
    }
    // mod.rs:86-101
    static std::vector<Affine> decrypt_batch(const Parameters& p, const std::vector<Fe>& sks, const std::vector<Ciphertext>& cts) {
        const size_t n = sks.size();
        if (cts.size() != n) throw Error(CPB_BAD_LENGTH, "decrypt: one ciphertext per key");
        std::vector<Affine> out(n);
        if (n) check(cpb_elgamal_decrypt_batch(p.ctx(), sks[0].data(), cts[0].c1.x.data(), out[0].x.data(), n));
        return out;
    }
};

}  // namespace elgamal

namespace blake2s {   // commitment::blake2s::Commitment, R/commitment/blake2s/mod.rs:11-33

struct Commitment {
    static std::vector<std::array<uint8_t, 32>> commit_batch(const std::vector<std::vector<uint8_t>>& inputs,
                                                             const std::vector<std::array<uint8_t, 32>>& randomness, int device = 0) {
        const size_t n = inputs.size();
        if (randomness.size() != n) throw Error(CPB_BAD_LENGTH, "commit: one randomness per input");
        std::vector<uint8_t> values;
        std::vector<uint64_t> offsets;
        ragged_pack(inputs, values, offsets);
        std::vector<std::array<uint8_t, 32>> out(n);
        if (n) check(cpb_blake2s_commit_batch(device, values.data(), offsets.data(), randomness[0].data(), out[0].data(), n));
        return out;
    }
};

}  // namespace blake2s

// MerkleTree<FieldMTConfig> (R/merkle_tree/mod.rs:381-533; Config of R/merkle_tree/tests/mod.rs:198-206)
class PoseidonMerkleTree {
public:
    std::vector<Fe> leaf_nodes, non_leaf_nodes;   // the reference's two arrays (mod.rs:383-395)

    static PoseidonMerkleTree create(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const std::vector<Fe>& leaves, size_t leaf_len) {
        PoseidonMerkleTree t;
        const size_t n = leaf_len ? leaves.size() / leaf_len : 0;
        t.leaf_nodes.resize(n);
        t.non_leaf_nodes.resize(n ? n - 1 : 0);
        check(cpb_merkle_poseidon_build(leaf.ctx(), two_to_one.ctx(), leaves.empty() ? nullptr : leaves[0].data(), leaf_len, n,
                                        n ? t.leaf_nodes[0].data() : nullptr, n > 1 ? t.non_leaf_nodes[0].data() : nullptr));
        return t;
    }
    // leaves of different lengths (Config::Leaf = [F]): each leaf hashed at its own length
    static PoseidonMerkleTree create(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const std::vector<std::vector<Fe>>& leaves) {
        std::vector<Fe> values;
        std::vector<uint64_t> offsets;
        ragged_pack(leaves, values, offsets);
        if (!leaves.empty() && equal_lengths(leaves) && !leaves[0].empty()) return create(leaf, two_to_one, values, leaves[0].size());
        PoseidonMerkleTree t;
        const size_t n = leaves.size();
        t.leaf_nodes.resize(n);
        t.non_leaf_nodes.resize(n ? n - 1 : 0);
        check(cpb_merkle_poseidon_build_ragged(leaf.ctx(), two_to_one.ctx(), values.empty() ? nullptr : values[0].data(), offsets.data(), n,
                                               n ? t.leaf_nodes[0].data() : nullptr, n > 1 ? t.non_leaf_nodes[0].data() : nullptr));
        return t;
    }
    Fe root() const { return non_leaf_nodes.at(0); }
    size_t height() const {
        size_t h = 1, n = leaf_nodes.size();
        while (n > 1) { n >>= 1; h++; }
        return h;
    }
    // authentication path of leaf `index`, root side first (compute_auth_path, mod.rs:548-573)
    std::vector<Fe> auth_path(size_t index) const {
        std::vector<Fe> path;
        size_t cur = (index + leaf_nodes.size() - 1 - 1) >> 1;   // parent of the leaf's position in the full tree
        while (cur != 0) {
            path.push_back(non_leaf_nodes[(cur & 1) ? cur + 1 : cur - 1]);
            cur = (cur - 1) >> 1;
        }
        return std::vector<Fe>(path.rbegin(), path.rend());
    }
    Fe leaf_sibling_hash(size_t index) const { return leaf_nodes[index ^ 1]; }

    // n x Path::verify (mod.rs:172-212) against `root` in ONE kernel launch: proofs for leaves `indexes` of this tree
    // (generate_proof for each), `leaves` = the claimed leaves, leaf_len elements each.  ok[i] = 1 when path i recomputes the root.
    std::vector<uint8_t> verify_batch(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const Fe& root,
                                      const std::vector<size_t>& indexes, const std::vector<Fe>& leaves, size_t leaf_len) const {
        const size_t n = indexes.size(), plen = height() - 2;
        std::vector<Fe> sib, paths;
        std::vector<uint64_t> idx;
        proofs(indexes, sib, paths, idx);
        std::vector<uint8_t> ok(n, 0);
        if (n)
            check(cpb_merkle_poseidon_verify_batch(leaf.ctx(), two_to_one.ctx(), root.data(), leaves[0].data(), leaf_len, sib[0].data(),
                                                   plen ? paths[0].data() : nullptr, plen, idx.data(), ok.data(), n));
        return ok;
    }
    // the same with claimed leaves of different lengths: leaves[i] belongs to indexes[i]
    std::vector<uint8_t> verify_batch(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const Fe& root,
                                      const std::vector<size_t>& indexes, const std::vector<std::vector<Fe>>& leaves) const {
        const size_t n = indexes.size(), plen = height() - 2;
        if (leaves.size() != n) throw Error(CPB_BAD_LENGTH, "one leaf per index");
        std::vector<Fe> sib, paths, values;
        std::vector<uint64_t> idx, offsets;
        proofs(indexes, sib, paths, idx);
        ragged_pack(leaves, values, offsets);
        std::vector<uint8_t> ok(n, 0);
        if (n)
            check(cpb_merkle_poseidon_verify_ragged_batch(leaf.ctx(), two_to_one.ctx(), root.data(), values.empty() ? nullptr : values[0].data(),
                                                          offsets.data(), sib[0].data(), plen ? paths[0].data() : nullptr, plen, idx.data(),
                                                          ok.data(), n));
        return ok;
    }

    // k x MerkleTree::update (mod.rs:690-701) in one call: leaf indexes[i] becomes leaves[i * leaf_len .. (i+1) * leaf_len); a repeated
    // index takes its last leaf.  Only the touched nodes and the siblings they read cross PCIe.
    void update_batch(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const std::vector<uint64_t>& indexes,
                      const std::vector<Fe>& leaves, size_t leaf_len) {
        update_impl(leaf, two_to_one, indexes, leaves, leaf_len, nullptr);
    }
    void update(const poseidon::Config& leaf, const poseidon::Config& two_to_one, size_t index, const std::vector<Fe>& new_leaf) {
        update_batch(leaf, two_to_one, {(uint64_t)index}, new_leaf, new_leaf.size());
    }
    // check_update (mod.rs:706-725) for all k at once: the tree changes only when the new root equals asserted_new_root.
    bool check_update_batch(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const std::vector<uint64_t>& indexes,
                            const std::vector<Fe>& leaves, size_t leaf_len, const Fe& asserted_new_root) {
        return update_impl(leaf, two_to_one, indexes, leaves, leaf_len, &asserted_new_root);
    }
    bool check_update(const poseidon::Config& leaf, const poseidon::Config& two_to_one, size_t index, const std::vector<Fe>& new_leaf,
                      const Fe& asserted_new_root) {
        return check_update_batch(leaf, two_to_one, {(uint64_t)index}, new_leaf, new_leaf.size(), asserted_new_root);
    }

private:
    bool update_impl(const poseidon::Config& leaf, const poseidon::Config& two_to_one, const std::vector<uint64_t>& indexes,
                     const std::vector<Fe>& leaves, size_t leaf_len, const Fe* asserted) {
        const size_t k = indexes.size();
        if (leaves.size() != k * leaf_len) throw Error(CPB_BAD_LENGTH, "one leaf of leaf_len elements per index");
        int applied = 0;
        check(cpb_merkle_poseidon_update(leaf.ctx(), two_to_one.ctx(), leaf_nodes.empty() ? nullptr : leaf_nodes[0].data(),
                                         non_leaf_nodes.empty() ? nullptr : non_leaf_nodes[0].data(), leaf_nodes.size(), indexes.data(),
                                         leaves.empty() ? nullptr : leaves[0].data(), leaf_len, k, asserted ? asserted->data() : nullptr,
                                         &applied));
        return applied != 0;
    }
    void proofs(const std::vector<size_t>& indexes, std::vector<Fe>& sib, std::vector<Fe>& paths, std::vector<uint64_t>& idx) const {
        const size_t n = indexes.size(), plen = height() - 2;
        sib.resize(n);
        paths.resize(n * plen);
        idx.resize(n);
        for (size_t i = 0; i < n; i++) {
            sib[i] = leaf_sibling_hash(indexes[i]);
            std::vector<Fe> ap = auth_path(indexes[i]);
            for (size_t k = 0; k < plen; k++) paths[i * plen + k] = ap[k];
            idx[i] = indexes[i];
        }
    }
};

// A group of GPUs driven by this process (include/cpb200.h, "Merkle tree across several GPUs"): MerkleTree::new with the
// leaves sharded over the devices; the result is the reference's two arrays, identical to a one-GPU build.
class GpuGroup {
public:
    explicit GpuGroup(const std::vector<int>& devices) : devices_(devices) {
        cpb_multi* m = nullptr;
        check(cpb_multi_create((int)devices.size(), devices.data(), &m));
        m_.reset(m, cpb_multi_destroy);
    }
    bool uses_nccl() const { return cpb_multi_uses_nccl(m_.get()) != 0; }
    // leaf[d] / two_to_one[d]: the same parameters, created on devices()[d] (Config's `device` argument)
    PoseidonMerkleTree create(const std::vector<const poseidon::Config*>& leaf, const std::vector<const poseidon::Config*>& two_to_one,
                              const std::vector<Fe>& leaves, size_t leaf_len) const {
        if (leaf.size() != devices_.size() || two_to_one.size() != devices_.size()) throw Error(CPB_BAD_PARAMS, "one context per device");
        std::vector<cpb_poseidon_ctx*> lc, nc;
        for (auto* c : leaf) lc.push_back(c->ctx());
        for (auto* c : two_to_one) nc.push_back(c->ctx());
        PoseidonMerkleTree t;
        const size_t n = leaf_len ? leaves.size() / leaf_len : 0;
        t.leaf_nodes.resize(n);
        t.non_leaf_nodes.resize(n ? n - 1 : 0);
        check(cpb_merkle_poseidon_build_multi(m_.get(), lc.data(), nc.data(), leaves.empty() ? nullptr : leaves[0].data(), leaf_len, n,
                                              n ? t.leaf_nodes[0].data() : nullptr, n > 1 ? t.non_leaf_nodes[0].data() : nullptr));
        return t;
    }
    const std::vector<int>& devices() const { return devices_; }

private:
    std::vector<int> devices_;
    std::shared_ptr<cpb_multi> m_;
};

}  // namespace cpb
