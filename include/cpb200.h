/*
 * cpb200.h -- C ABI of libcpb200.so: H100-native (sm_90a) batched evaluation of the
 * ark-crypto-primitives hot path (Poseidon CRH / two-to-one, Pedersen CRH / commitment,
 * Merkle-tree build).  This is the drop-in boundary: plain pointers and sizes, no C++ or
 * torch types.  A Rust shim crate binds these symbols and implements the reference traits on
 * top of them (INTEGRATION.md shows the bindings).
 *
 * R below = /root/reference/crypto-primitives/src (arkworks-rs/crypto-primitives @ 6a770ebf).
 *
 * DATA LAYOUT.  A field element is 4 x uint64_t little-endian limbs in Montgomery form
 * (R = 2^256), fully reduced -- the memory image of ark-ff's Fp<MontBackend<_,4>,4>
 * (`BigInt<4>` in `.0.0`), so a `&[Fr]` can be passed without conversion.  A curve point is
 * affine (x, y): 8 x uint64_t.  Byte inputs are plain uint8_t.  All arrays are dense, C order.
 *
 * PRECONDITION.  Field elements and point coordinates passed in must be fully reduced (< p), as ark-ff guarantees for
 * every `Fp` value; this is not checked on the hot path.  Unreduced limbs yield unspecified digests -- never a memory
 * error (no address is derived from a field value).  cpb_field_to_montgomery() does check its canonical inputs.
 *
 * POINTERS.  Functions without suffix take HOST pointers and perform the H2D/D2H copies
 * themselves on the context's stream; `_dev` functions take DEVICE pointers (on the context's
 * device) plus a CUDA stream handle (`cudaStream_t` passed as void*, NULL = default stream),
 * launch asynchronously and do not synchronise.
 *
 * ERRORS.  Every function returns a cpb_status.  Nothing panics/throws across the ABI (each entry point runs under an
 * exception guard: host allocation failures and the like come back as CPB_INTERNAL_ERROR); the
 * shim maps codes back to the reference's behaviour (R/lib.rs:46-52 `Error`, and the panics at
 * R/crh/pedersen/mod.rs:82-89, R/merkle_tree/mod.rs:430-433).  cpb_last_error() returns a
 * thread-local description of the last failure.  There is NO CPU fallback: without a usable
 * sm_90 (H100) device every compute entry point fails with CPB_NO_DEVICE / CPB_CUDA_ERROR.
 *
 * THREADING.  A context is immutable after creation and may be used from several host
 * threads concurrently (reference: `Parameters: Sync`, R/crh/mod.rs:21); host-pointer calls
 * serialise on an internal mutex that guards the context's staging buffers.
 */
#ifndef CPB200_H
#define CPB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum cpb_status {
    CPB_OK = 0,
    CPB_BAD_LENGTH = 1,   /* R/crh/pedersen/mod.rs:82-89 "incorrect input length" panic; Error::IncorrectInputLength */
    CPB_BAD_PARAMS = 2,   /* PoseidonConfig::new asserts, R/sponge/poseidon/mod.rs:198-206; generator-count assert R/crh/pedersen/mod.rs:101-109 */
    CPB_NOT_POW2 = 3,     /* R/merkle_tree/mod.rs:430-433 */
    CPB_CUDA_ERROR = 4,
    CPB_NO_DEVICE = 5,
    CPB_UNSUPPORTED = 6,
    CPB_NULL_POINTER = 7,
    CPB_INTERNAL_ERROR = 8,  /* host allocation failure or any C++ exception caught at the boundary */
    CPB_NCCL_ERROR = 9       /* libnccl could not be loaded, or an NCCL call of the multi-GPU build failed */
} cpb_status;

typedef enum cpb_field {
    CPB_BLS12_381_FR = 0, /* the reference's test field, R/sponge/test.rs:5-12 */
    CPB_BN254_FR = 1,
    CPB_JUBJUB_FR = 2,    /* ark_ed_on_bls12_381::Fr, R/merkle_tree/tests/mod.rs:195 */
    CPB_BLS12_377_FR = 3, /* R/crh/poseidon/constraints.rs:133-190 */
    CPB_ED_ON_BLS12_377_FR = 4  /* ark_ed_on_bls12_377::Fr, the scalar field of CPB_ED_ON_BLS12_377 (R/benches/signature.rs:5-10).  Known
                                   to the field-level calls only (cpb_field_modulus, cpb_field_{to,from}_montgomery[_dev],
                                   cpb_field_serialized_size, cpb_field_{serialize,deserialize}); every call that takes the field of a hash
                                   (Poseidon, Merkle, path wire formats) answers CPB_BAD_PARAMS for it, as for an unknown id. */
} cpb_field;

typedef enum cpb_curve {
    CPB_JUBJUB = 0,          /* ark_ed_on_bls12_381::EdwardsProjective (a=-1, d=-10240/10241), base field BLS12-381 Fr;
                                the curve of R/merkle_tree/tests/mod.rs:8 and R/crh/pedersen/constraints.rs:168 */
    CPB_ED_ON_BLS12_377 = 1  /* ark_ed_on_bls12_377 (a=-1, d=3021), base field BLS12-377 Fr; R/benches/crh.rs:5 */
} cpb_curve;

typedef struct cpb_poseidon_ctx cpb_poseidon_ctx;
typedef struct cpb_pedersen_ctx cpb_pedersen_ctx;
typedef struct cpb_bowe_hopwood_ctx cpb_bowe_hopwood_ctx;
typedef struct cpb_exchange cpb_exchange;   /* one rank's end of the multi-GPU root exchange (one process per GPU) */
typedef struct cpb_multi cpb_multi;         /* a group of GPUs driven by one process */

const char* cpb_last_error(void);

/* ABI revision of this header: bumped when entry points or status codes are added (2 = CPB_INTERNAL_ERROR, cpb_abi_version; 3 = _dev field conversion, host pinning, launch count, multi-GPU build, CPB_NCCL_ERROR, wire formats; 4 = ragged Poseidon batches: CRH, sponge, Merkle build and path verification over inputs of different lengths; 5 = Merkle update and
 * check_update of Poseidon-node trees, in place on device arrays or over host arrays; later additions under 5 are additive: Merkle path verification of the Pedersen
 * trees, batched duplex sponges with the cpb_sponge_mode type, ragged duplex calls with a mode per sponge (a library that has
 * them exports cpb_poseidon_duplex_absorb_ragged), the field CPB_ED_ON_BLS12_377_FR with signatures and encryption over
 * CPB_ED_ON_BLS12_377 (a library that has them exports cpb_te_base_ctx_create_ex and answers CPB_OK to
 * cpb_field_modulus(CPB_ED_ON_BLS12_377_FR, ...)). */
#define CPB_ABI_VERSION 5
int cpb_abi_version(void);
int cpb_version(void);
/* Number of visible CUDA devices with compute capability 10.x (0 when none / no driver). */
int cpb_device_count(void);

/* Page-lock / unlock a caller-owned host buffer (cudaHostRegister, portable): host-pointer entry points then copy at
 * full PCIe rate and overlap copies with hashing.  A Rust `Vec<Fr>` is pageable; the shim may pin it once and reuse it. */
cpb_status cpb_host_register(void* ptr, size_t bytes);
cpb_status cpb_host_unregister(void* ptr);

/* ---- fields ----------------------------------------------------------------------------- */
/* Modulus as 4 LE limbs.  (ark-ff `F::MODULUS`.) */
cpb_status cpb_field_modulus(int field_id, uint64_t out[4]);
/* Canonical little-endian integers (< 2^256; reduced mod p) <-> Montgomery limbs, on `device`.
 * Convenience for non-Rust callers; ark-ff callers already hold Montgomery limbs. */
cpb_status cpb_field_to_montgomery(int field_id, int device, const uint64_t* in, uint64_t* out, size_t n);
cpb_status cpb_field_from_montgomery(int field_id, int device, const uint64_t* in, uint64_t* out, size_t n);
/* Same on device buffers (in-place allowed: out == in), asynchronous on `stream`. */
cpb_status cpb_field_to_montgomery_dev(int field_id, int device, const uint64_t* in, uint64_t* out, size_t n, void* stream);
cpb_status cpb_field_from_montgomery_dev(int field_id, int device, const uint64_t* in, uint64_t* out, size_t n, void* stream);

/* ---- Poseidon --------------------------------------------------------------------------- */
/* find_poseidon_ark_and_mds, R/sponge/poseidon/traits.rs:105-146 (Grain LFSR of
 * R/sponge/poseidon/grain_lfsr.rs).  ark_out: (full+partial) x (rate+1) elements, mds_out:
 * (rate+1)^2 elements, Montgomery.  Host-only, once per parameter set. */
cpb_status cpb_poseidon_find_ark_and_mds(int field_id, uint64_t prime_bits, int rate, int full_rounds,
                                         int partial_rounds, int skip_matrices, uint64_t* ark_out,
                                         uint64_t* mds_out);
/* PoseidonDefaultConfigField::get_default_poseidon_parameters, traits.rs:59-103.  The entry tables belong to a field
 * (`impl PoseidonDefaultConfig<N> for FrConfig`): the reference has them for its BLS12-381 Fr test field only
 * (R/sponge/test.rs:13-32, rate 2..8, capacity 1); any other field, or a rate without an entry, -> CPB_BAD_PARAMS (the
 * tables' alpha = 5 is not even a permutation of BLS12-377 Fr).  Writes the shape; a second call of
 * cpb_poseidon_find_ark_and_mds with that shape yields ark/mds. */
cpb_status cpb_poseidon_default_entry(int field_id, int rate, int optimized_for_weights, uint64_t* alpha, int* full_rounds,
                                      int* partial_rounds, int* skip_matrices);

/* PoseidonConfig::new, R/sponge/poseidon/mod.rs:189-217.  ark: (full+partial) x t, mds: t x t
 * (t = rate+capacity), Montgomery limbs, copied.  Uploads the device round schedule. */
cpb_status cpb_poseidon_ctx_create(int field_id, int rate, int capacity, int full_rounds, int partial_rounds,
                                   uint64_t alpha, const uint64_t* ark, const uint64_t* mds, int device,
                                   cpb_poseidon_ctx** out);
void cpb_poseidon_ctx_destroy(cpb_poseidon_ctx* ctx);
/* 1 when the partial rounds run in sparse form, 0 for the dense fallback (same results). */
int cpb_poseidon_ctx_is_sparse(const cpb_poseidon_ctx* ctx);
int cpb_poseidon_ctx_field(const cpb_poseidon_ctx* ctx);
int cpb_poseidon_ctx_device(const cpb_poseidon_ctx* ctx);

/* n independent permutations of t-element states: PoseidonSponge::permute, mod.rs:98-121. */
cpb_status cpb_poseidon_permute_batch(cpb_poseidon_ctx* ctx, const uint64_t* states_in, uint64_t* states_out, size_t n);
cpb_status cpb_poseidon_permute_batch_dev(cpb_poseidon_ctx* ctx, const uint64_t* states_in, uint64_t* states_out,
                                          size_t n, void* stream);

/* n x crh::poseidon::CRH::evaluate (R/crh/poseidon/mod.rs:30-40): input i is the `len` elements
 * at in + 4*len*i; out[i] one element.  len == 0 is allowed (one permutation of the zero state). */
cpb_status cpb_poseidon_crh_batch(cpb_poseidon_ctx* ctx, const uint64_t* in, size_t len, uint64_t* out, size_t n);
cpb_status cpb_poseidon_crh_batch_dev(cpb_poseidon_ctx* ctx, const uint64_t* in, size_t len, uint64_t* out, size_t n,
                                      void* stream);

/* n independent sponges: PoseidonSponge::new -> absorb(len native elements) -> squeeze_native_field_elements(n_squeeze)
 * (R/sponge/poseidon/mod.rs:220-257, 323-345); out: n x n_squeeze elements.  n_squeeze = 1 is the CRH. */
cpb_status cpb_poseidon_sponge_batch(cpb_poseidon_ctx* ctx, const uint64_t* in, size_t len, uint64_t* out, size_t n_squeeze, size_t n);
cpb_status cpb_poseidon_sponge_batch_dev(cpb_poseidon_ctx* ctx, const uint64_t* in, size_t len, uint64_t* out, size_t n_squeeze,
                                         size_t n, void* stream);

/* n x crh::poseidon::TwoToOneCRH::compress / evaluate (mod.rs:58-79): pairs[i] = (left, right). */
cpb_status cpb_poseidon_compress_batch(cpb_poseidon_ctx* ctx, const uint64_t* pairs, uint64_t* out, size_t n);
cpb_status cpb_poseidon_compress_batch_dev(cpb_poseidon_ctx* ctx, const uint64_t* pairs, uint64_t* out, size_t n,
                                           void* stream);

/* ---- Batched duplex sponges -------------------------------------------------------------------------------------- */
/* DuplexSpongeMode (R/sponge/mod.rs): squeezing == 0 is Absorbing{next_absorb_index = index}, 1 is Squeezing{next_squeeze_index}. */
typedef struct cpb_sponge_mode {
    int squeezing;
    size_t index;
} cpb_sponge_mode;
/* n independent PoseidonSponge<F> over one context that share one mode: states (n x t elements, Montgomery, the layout of
 * cpb_poseidon_permute_batch) are updated in place and *mode (host memory) is read and advanced by every call.  Each call applies
 * the same operation to every sponge with the mode rules of the reference (R/sponge/poseidon/mod.rs:124-186, 236-257, 323-345):
 *   absorb         k native elements per sponge from in + 4*k*i; k == 0 does nothing;
 *   absorb_bytes   the byte string of `len` bytes at in + stride*i (stride 0: one string for every sponge), encoded as
 *                  Absorb for [u8] (R/sponge/absorb.rs:137-141): an 8-byte little-endian length, then the bytes, in
 *                  31-byte little-endian chunks, i.e. ceil((len + 8) / 31) elements;
 *   squeeze        squeeze_native_field_elements(m) to out + 4*m*i, as Montgomery limbs or (canonical != 0) as canonical
 *                  integers; m == 0 still permutes from Absorbing mode.
 * Argument checks, before any device work, in this order: mode == NULL -> CPB_NULL_POINTER, mode->squeezing not 0 or 1 ->
 * CPB_BAD_PARAMS; sizes beyond 2^62 bytes -> CPB_BAD_LENGTH; a buffer the call reads or writes (n > 0) NULL -> CPB_NULL_POINTER;
 * ctx NULL -> CPB_NULL_POINTER; mode->index > rate -> CPB_BAD_PARAMS.  n == 0 advances the mode and launches nothing: the mode
 * belongs to the batch.  On an error the mode is unchanged.
 * Host forms: host arrays, copied in and out.  _dev forms: device arrays, enqueued on `stream` without host synchronisation
 * (CUDA-graph capturable). */
cpb_status cpb_poseidon_duplex_absorb(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* mode, const uint64_t* in, size_t k,
                                      size_t n);
cpb_status cpb_poseidon_duplex_absorb_dev(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* mode, const uint64_t* in, size_t k,
                                          size_t n, void* stream);
cpb_status cpb_poseidon_duplex_absorb_bytes(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* mode, const uint8_t* in, size_t len,
                                            size_t stride, size_t n);
cpb_status cpb_poseidon_duplex_absorb_bytes_dev(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* mode, const uint8_t* in,
                                                size_t len, size_t stride, size_t n, void* stream);
cpb_status cpb_poseidon_duplex_squeeze(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* mode, uint64_t* out, size_t m,
                                       int canonical, size_t n);
cpb_status cpb_poseidon_duplex_squeeze_dev(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* mode, uint64_t* out, size_t m,
                                           int canonical, size_t n, void* stream);
/* Ragged duplex calls: n sponges with a mode EACH, modes[i] (n cpb_sponge_mode), and a span each under the layout of the ragged
 * batches below: offsets holds n + 1 uint64_t and sponge i's span is buf[offsets[i] .. offsets[i+1]), in elements (field data) or
 * in bytes (byte strings); offsets[0] need not be 0.  Every sponge follows the reference's rules from its own mode and gets its new
 * mode written back:
 *   absorb_ragged         sponge i absorbs the native elements of its span of `values`;
 *   absorb_bytes_ragged   sponge i absorbs its span of `bytes` as one [u8] value (its own 8-byte length, then 31-byte chunks),
 *                         as cpb_poseidon_duplex_absorb_bytes does for that string;
 *   squeeze_ragged        sponge i runs squeeze_native_field_elements(offsets[i+1] - offsets[i]) into its span of `out`, as
 *                         Montgomery limbs or (canonical != 0) canonical integers; 0 elements still permute from Absorbing mode.
 * The mode layout: 16 bytes, squeezing in bytes 0..3 (bytes 4..7 are padding and are not read), index at byte 8.  A written mode
 * has its first 8-byte word whole, padding zeroed, so an int64 array of (n, 2) holds [squeezing, index] per row.
 * Argument checks, before any device work, in this order: n >= 2^32 -> CPB_BAD_LENGTH; n == 0 -> CPB_OK, nothing launched;
 * states, modes or offsets NULL -> CPB_NULL_POINTER.  Host forms then: decreasing offsets -> CPB_BAD_LENGTH; a NULL data buffer
 * while the spans are not all empty -> CPB_NULL_POINTER; a mode with squeezing not 0 or 1 -> CPB_BAD_PARAMS.  Then ctx NULL ->
 * CPB_NULL_POINTER, and for host forms a mode with index > rate -> CPB_BAD_PARAMS.  On an error states, modes and outputs are
 * unchanged.  Spans are clamped as in the ragged batches: a decreasing pair is an empty span, and nothing outside
 * [offsets[0], offsets[n]) is read or written.
 * Host forms: host arrays; only buf[offsets[0] .. offsets[n]) is copied, indexed from offsets[0]; one host synchronisation.
 * _dev forms: every array is device memory and the modes are updated in place; nothing in device memory is checked.  A sponge
 * whose mode is invalid (squeezing, read from bytes 0..3, not 0 or 1, or index > rate) is left untouched -- state and mode as they
 * were -- and its squeeze span is written as zeros; the other sponges are unaffected.  The device sorts the sponges by their
 * permutation count first; scratch comes from the stream-ordered pool and nothing synchronises the host (CUDA-graph capturable). */
cpb_status cpb_poseidon_duplex_absorb_ragged(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* modes, const uint64_t* values,
                                             const uint64_t* offsets, size_t n);
cpb_status cpb_poseidon_duplex_absorb_ragged_dev(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* modes, const uint64_t* values,
                                                 const uint64_t* offsets, size_t n, void* stream);
cpb_status cpb_poseidon_duplex_absorb_bytes_ragged(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* modes, const uint8_t* bytes,
                                                   const uint64_t* offsets, size_t n);
cpb_status cpb_poseidon_duplex_absorb_bytes_ragged_dev(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* modes, const uint8_t* bytes,
                                                       const uint64_t* offsets, size_t n, void* stream);
cpb_status cpb_poseidon_duplex_squeeze_ragged(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* modes, uint64_t* out,
                                              const uint64_t* offsets, int canonical, size_t n);
cpb_status cpb_poseidon_duplex_squeeze_ragged_dev(cpb_poseidon_ctx* ctx, uint64_t* states, cpb_sponge_mode* modes, uint64_t* out,
                                                  const uint64_t* offsets, int canonical, size_t n, void* stream);

/* ---- Merkle tree, field leaves ---------------------------------------------------------- */
/* MerkleTree::new (R/merkle_tree/mod.rs:411-422) for Config{Leaf=[F], LeafDigest=InnerDigest=F,
 * IdentityDigestConverter, LeafHash=poseidon::CRH, TwoToOneHash=poseidon::TwoToOneCRH}
 * (R/merkle_tree/tests/mod.rs:198-206).  leaves: n x leaf_len elements.  Outputs the reference's
 * two arrays: leaf_nodes[n], non_leaf_nodes[n-1] in heap order (root at 0; children of i at
 * 2i+1, 2i+2; mod.rs:383-395).  n must be a power of two > 1 (else CPB_NOT_POW2). */
cpb_status cpb_merkle_poseidon_build(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* leaves,
                                     size_t leaf_len, size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes);
cpb_status cpb_merkle_poseidon_build_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx,
                                         const uint64_t* leaves, size_t leaf_len, size_t n, uint64_t* leaf_nodes,
                                         uint64_t* non_leaf_nodes, void* stream);
/* Number of kernel launches one cpb_merkle_poseidon_build_dev over n leaves issues with this two-to-one context
 * (0 when n is not a power of two > 1). */
size_t cpb_merkle_poseidon_launch_count(const cpb_poseidon_ctx* node_ctx, size_t n);
/* MerkleTree::new_with_leaf_digest (mod.rs:424-523): inner levels only. */
cpb_status cpb_merkle_poseidon_from_digests(cpb_poseidon_ctx* node_ctx, const uint64_t* leaf_digests, size_t n,
                                            uint64_t* non_leaf_nodes);
cpb_status cpb_merkle_poseidon_from_digests_dev(cpb_poseidon_ctx* node_ctx, const uint64_t* leaf_digests, size_t n,
                                                uint64_t* non_leaf_nodes, void* stream);

/* n x Path::verify (R/merkle_tree/mod.rs:172-212) for the field-leaf Config against one root: path i is
 * (leaf_sibling_hashes[i], auth_paths[i*path_len .. (i+1)*path_len) ordered root side first as Path.auth_path,
 * leaf_indexes[i]); ok[i] = 1 when the recomputed root matches.  Tree height = path_len + 2. */
cpb_status cpb_merkle_poseidon_verify_batch(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                            const uint64_t* leaves, size_t leaf_len, const uint64_t* leaf_sibling_hashes,
                                            const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes, uint8_t* ok,
                                            size_t n);
cpb_status cpb_merkle_poseidon_verify_batch_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                                const uint64_t* leaves, size_t leaf_len, const uint64_t* leaf_sibling_hashes,
                                                const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes,
                                                uint8_t* ok, size_t n, void* stream);

/* ---- Merkle tree update (Poseidon inner nodes) ------------------------------------------------------------------ */
/* k x MerkleTree::update (R/merkle_tree/mod.rs:690-701), or MerkleTree::check_update (:706-725) for all k at once when
 * asserted_root != NULL, on a tree in the reference's layout: leaf_nodes[n], non_leaf_nodes[n-1] in heap order, updated IN PLACE.
 * Any tree whose inner hash is poseidon::TwoToOneCRH: field leaves, new_with_leaf_digest / blank trees, and through the digest
 * form the Pedersen-leaf tree of cpb_merkle_mixed_build (hash the new leaves with cpb_pedersen_crh_x_batch first).
 * Semantics: the result equals k sequential update(indexes[i], leaf i) calls in input order, so when an index repeats its last
 * occurrence wins.  With asserted_root the new root is computed first and both arrays are written only when it equals
 * *asserted_root; otherwise the tree stays bit for bit untouched.  `applied` (nullable) receives 1 when the tree was written
 * (always, without asserted_root) and 0 otherwise.  asserted_root must not point into the tree.
 * Rules: n a power of two > 1 (else CPB_NOT_POW2); k >= 2^32 -> CPB_BAD_LENGTH; k == 0 is a no-op returning CPB_OK, `applied` then
 * says whether the current root equals asserted_root.
 * The digest forms take new_leaf_digests[k] (leaf digests, e.g. CRH outputs); the leaf forms take new_leaves[k x leaf_len] and hash
 * all k of them with poseidon::CRH on the same stream first.
 * _dev forms: every pointer is device memory (`applied` a uint8_t); an index >= n is skipped and nothing outside the caller's arrays
 * is read or written (indexes are not checked on the host).  No host synchronisation: scratch (about sum over levels l of
 * min(k, 2^l) elements, at most 2n - 1, plus a few words per index) comes from the stream-ordered pool, and the launches depend on
 * the tree height only -- one grid per level while a level is wide, one four-warp team launch for the levels above.
 * Host forms: host arrays, `applied` an int*; an index >= n -> CPB_BAD_PARAMS before any copy.  The tree is not copied: the host
 * works out which untouched siblings the touched nodes read, uploads those with the indexes and the new leaves, runs the same
 * device code and copies back only the touched nodes. */
cpb_status cpb_merkle_poseidon_update_digests_dev(cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                                                  const uint64_t* indexes, const uint64_t* new_leaf_digests, size_t k,
                                                  const uint64_t* asserted_root, uint8_t* applied, void* stream);
cpb_status cpb_merkle_poseidon_update_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                          size_t n, const uint64_t* indexes, const uint64_t* new_leaves, size_t leaf_len, size_t k,
                                          const uint64_t* asserted_root, uint8_t* applied, void* stream);
cpb_status cpb_merkle_poseidon_update_digests(cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, size_t n,
                                              const uint64_t* indexes, const uint64_t* new_leaf_digests, size_t k, const uint64_t* asserted_root,
                                              int* applied);
cpb_status cpb_merkle_poseidon_update(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                      size_t n, const uint64_t* indexes, const uint64_t* new_leaves, size_t leaf_len, size_t k,
                                      const uint64_t* asserted_root, int* applied);

/* ---- Poseidon over inputs of different lengths (ragged batches) --------------------------------------------------- */
/* The reference's Poseidon input and field leaf are unsized slices (CRHScheme::Input = [F], R/crh/poseidon/mod.rs:19-41;
 * Config::Leaf = [F], R/merkle_tree/tests/mod.rs:198-206).  A ragged batch is `values`, field elements back to back, and
 * `offsets`, n + 1 uint64_t: input i is values[offsets[i] .. offsets[i+1]) (element indices; offsets[0] need not be 0) --
 * one prefix sum over a Vec<Vec<F>>.  Zero-padding to a common length is not equivalent (absorbing zeros that start a new
 * rate block adds a permutation), so each input is hashed at its own length.
 * Host forms: offsets must not decrease (else CPB_BAD_LENGTH); only values[offsets[0] .. offsets[n]) is copied.
 * _dev forms: offsets (device memory) must not decrease; this is not checked, but a decreasing pair hashes as an empty input
 * and nothing outside values[offsets[0] .. offsets[n]) is read.  n >= 2^32 -> CPB_BAD_LENGTH; n == 0 -> CPB_OK, no launch.
 * The device sorts the inputs by permutation count before hashing (stream-ordered scratch, no host synchronisation). */
cpb_status cpb_poseidon_crh_ragged_batch(cpb_poseidon_ctx* ctx, const uint64_t* values, const uint64_t* offsets, uint64_t* out, size_t n);
cpb_status cpb_poseidon_crh_ragged_batch_dev(cpb_poseidon_ctx* ctx, const uint64_t* values, const uint64_t* offsets, uint64_t* out,
                                             size_t n, void* stream);
/* n sponges: absorb input i, squeeze n_squeeze native elements to out[i * n_squeeze ..]. */
cpb_status cpb_poseidon_sponge_ragged_batch(cpb_poseidon_ctx* ctx, const uint64_t* values, const uint64_t* offsets, uint64_t* out,
                                            size_t n_squeeze, size_t n);
cpb_status cpb_poseidon_sponge_ragged_batch_dev(cpb_poseidon_ctx* ctx, const uint64_t* values, const uint64_t* offsets, uint64_t* out,
                                                size_t n_squeeze, size_t n, void* stream);
/* MerkleTree::new over leaves of different lengths (mod.rs:411-422 hashes each leaf at its own length): the ragged leaf hash,
 * then the inner levels as cpb_merkle_poseidon_from_digests.  Outputs and rules as cpb_merkle_poseidon_build. */
cpb_status cpb_merkle_poseidon_build_ragged(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* values,
                                            const uint64_t* offsets, size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes);
cpb_status cpb_merkle_poseidon_build_ragged_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* values,
                                                const uint64_t* offsets, size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes,
                                                void* stream);
/* cpb_merkle_poseidon_verify_batch with leaf i = values[offsets[i] .. offsets[i+1]). */
cpb_status cpb_merkle_poseidon_verify_ragged_batch(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                                   const uint64_t* values, const uint64_t* offsets, const uint64_t* leaf_sibling_hashes,
                                                   const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes, uint8_t* ok,
                                                   size_t n);
cpb_status cpb_merkle_poseidon_verify_ragged_batch_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                                       const uint64_t* values, const uint64_t* offsets, const uint64_t* leaf_sibling_hashes,
                                                       const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes,
                                                       uint8_t* ok, size_t n, void* stream);

/* ---- Pedersen CRH / commitment over a twisted-Edwards curve -------------------------------- */
/* pedersen::Parameters{generators: Vec<Vec<C>>} (R/crh/pedersen/mod.rs:28-31) and, when n_rand > 0,
 * commitment::pedersen::Parameters.randomness_generator (R/commitment/pedersen/mod.rs:17-21).
 * generators_xy: num_windows x window_size affine points (x, y), generators[w][j] at index
 * w*window_size + j; rand_generators_xy: n_rand points (the reference uses MODULUS_BIT_SIZE of the
 * scalar field, :51-52), may be NULL when n_rand == 0.  The shim normalises the reference's
 * projective points to affine before the call.  Points must be on the curve (else
 * CPB_BAD_PARAMS); nothing else is assumed about them.  Builds the per-byte subset-sum tables on
 * the GPU. */
cpb_status cpb_pedersen_ctx_create(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy,
                                   size_t n_rand, const uint64_t* rand_generators_xy, int device,
                                   cpb_pedersen_ctx** out);
/* Same, choosing how many consecutive input bits one table lookup covers: 8 = 24 KB tables per chunk streamed through
 * shared memory by TMA; 9..22 = larger L2/HBM-resident tables gathered per lookup (fewer additions per hash, results
 * identical; table bytes = ceil(bits / chunk_bits) * 96 * 2^chunk_bits: 0.4 GB at 16, 5.2 GB at 20 for a 1024-bit
 * input); 0 = library default (the widest of 18 / 16 / 12 / 8 whose tables stay under 2 GiB). */
cpb_status cpb_pedersen_ctx_create_ex(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy,
                                      size_t n_rand, const uint64_t* rand_generators_xy, int device, int chunk_bits,
                                      cpb_pedersen_ctx** out);
void cpb_pedersen_ctx_destroy(cpb_pedersen_ctx* ctx);

/* n x pedersen::CRH::evaluate (R/crh/pedersen/mod.rs:76-129): input i is the `len` bytes at
 * in + i*stride, zero-padded by the callee to WINDOW_SIZE*NUM_WINDOWS/8 bytes (:94-99); bit k of
 * byte b selects generator 8b+k (:200-209).  len*8 > WINDOW_SIZE*NUM_WINDOWS -> CPB_BAD_LENGTH
 * (the reference panics, :82-89).  out_xy: n affine points. */
cpb_status cpb_pedersen_crh_batch(cpb_pedersen_ctx* ctx, const uint8_t* in, size_t len, size_t stride,
                                  uint64_t* out_xy, size_t n);
cpb_status cpb_pedersen_crh_batch_dev(cpb_pedersen_ctx* ctx, const uint8_t* in, size_t len, size_t stride,
                                      uint64_t* out_xy, size_t n, void* stream);
/* n x PedersenCRHCompressor<C, TECompressor, W>::evaluate (R/crh/injective_map/mod.rs:22-62): the
 * x-coordinate of the CRH output, one base-field element each. */
cpb_status cpb_pedersen_crh_x_batch(cpb_pedersen_ctx* ctx, const uint8_t* in, size_t len, size_t stride,
                                    uint64_t* out_x, size_t n);
cpb_status cpb_pedersen_crh_x_batch_dev(cpb_pedersen_ctx* ctx, const uint8_t* in, size_t len, size_t stride,
                                        uint64_t* out_x, size_t n, void* stream);
/* n x pedersen::TwoToOneCRH::compress (R/crh/pedersen/mod.rs:187-197): children_xy = n x (left, right)
 * affine points, each serialised uncompressed (x || y, 32-byte LE canonical; R/macros.rs:3-13) and
 * hashed as in `evaluate` (:152-182).  The _dev form needs 128*n bytes of device scratch. */
cpb_status cpb_pedersen_two_to_one_batch(cpb_pedersen_ctx* ctx, const uint64_t* children_xy, uint64_t* out_xy, size_t n);
cpb_status cpb_pedersen_two_to_one_batch_dev(cpb_pedersen_ctx* ctx, const uint64_t* children_xy, uint64_t* out_xy,
                                             size_t n, void* scratch_128n, void* stream);
/* n x CommitmentScheme::commit (R/commitment/pedersen/mod.rs:62-105): CRH of the padded input plus
 * sum_k bit_k(r) * randomness_generator[k]; randomness_le32 = n x 32-byte little-endian canonical
 * scalars (`randomness.0.into_bigint()`, :93).  len > WINDOW_SIZE*NUM_WINDOWS (the reference's own
 * guard compares bytes with bits, :69) or len*8 > WINDOW_SIZE*NUM_WINDOWS -> CPB_BAD_LENGTH. */
cpb_status cpb_pedersen_commit_batch(cpb_pedersen_ctx* ctx, const uint8_t* in, size_t len, size_t stride,
                                     const uint8_t* randomness_le32, uint64_t* out_xy, size_t n);
cpb_status cpb_pedersen_commit_batch_dev(cpb_pedersen_ctx* ctx, const uint8_t* in, size_t len, size_t stride,
                                         const uint8_t* randomness_le32, uint64_t* out_xy, size_t n, void* stream);

/* ---- Bowe-Hopwood Pedersen CRH (R/crh/bowe_hopwood/mod.rs) ------------------------------------------ */
/* bowe_hopwood::Parameters{generators: Vec<Vec<TEProjective<P>>>} (mod.rs:33-37): num_windows segments of
 * window_size generators (one per 3-bit chunk), affine (x, y), generators[w][j] at index w*window_size + j. */
cpb_status cpb_bowe_hopwood_ctx_create(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy, int device,
                                       cpb_bowe_hopwood_ctx** out);
void cpb_bowe_hopwood_ctx_destroy(cpb_bowe_hopwood_ctx* ctx);
/* n x bowe_hopwood::CRH::evaluate (mod.rs:115-185): output = x-coordinate (one base-field element).  Only the
 * 3-bit chunks the input covers contribute, so the digest depends on `len`.  len*8 > 3*window_size*num_windows
 * -> CPB_BAD_LENGTH (the reference panics, :121-129). */
cpb_status cpb_bowe_hopwood_crh_batch(cpb_bowe_hopwood_ctx* ctx, const uint8_t* in, size_t len, size_t stride, uint64_t* out_x, size_t n);
cpb_status cpb_bowe_hopwood_crh_batch_dev(cpb_bowe_hopwood_ctx* ctx, const uint8_t* in, size_t len, size_t stride, uint64_t* out_x,
                                          size_t n, void* stream);
/* n x bowe_hopwood::TwoToOneCRH::compress (mod.rs:228-240): children_x = n x (left, right) base-field elements,
 * serialised (32-byte LE canonical each) into the zeroed window_size*num_windows/8-byte buffer of `evaluate`
 * (mod.rs:200-226).  The _dev form needs cpb_bowe_hopwood_two_to_one_scratch_bytes(ctx, n) bytes of device scratch. */
cpb_status cpb_bowe_hopwood_two_to_one_batch(cpb_bowe_hopwood_ctx* ctx, const uint64_t* children_x, uint64_t* out_x, size_t n);
cpb_status cpb_bowe_hopwood_two_to_one_batch_dev(cpb_bowe_hopwood_ctx* ctx, const uint64_t* children_x, uint64_t* out_x, size_t n,
                                                 void* scratch, void* stream);
size_t cpb_bowe_hopwood_two_to_one_scratch_bytes(const cpb_bowe_hopwood_ctx* ctx, size_t n);

/* ---- Merkle tree, byte leaves -------------------------------------------------------------- */
/* MerkleTree::new for Config{Leaf=[u8], LeafHash=pedersen::CRH, LeafInnerDigestConverter=
 * ByteDigestConverter, TwoToOneHash=pedersen::TwoToOneCRH} -- JubJubMerkleTreeParams of
 * R/merkle_tree/tests/mod.rs:19-33.  Digests are affine points (8 words).  The _dev form needs
 * 64*n bytes of device scratch. */
cpb_status cpb_merkle_pedersen_build(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, const uint8_t* leaves,
                                     size_t leaf_len, size_t n, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy);
cpb_status cpb_merkle_pedersen_build_dev(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, const uint8_t* leaves,
                                         size_t leaf_len, size_t leaf_stride, size_t n, uint64_t* leaf_nodes_xy,
                                         uint64_t* non_leaf_nodes_xy, void* scratch_64n, void* stream);

/* ---- Merkle tree update (Pedersen inner nodes) ------------------------------------------------------------------ */
/* k x MerkleTree::update / check_update on a byte tree of cpb_merkle_pedersen_build (inner hash pedersen::TwoToOneCRH), with the
 * rules of cpb_merkle_poseidon_update* word for word: the result equals k sequential updates in input order (the last occurrence
 * of a repeated index wins); with asserted_root_xy (8 words) nothing is written unless the new root matches, and `applied` says
 * which happened; k == 0 is a no-op whose `applied` says whether the current root equals asserted_root_xy; n not a power of two
 * > 1 -> CPB_NOT_POW2; k >= 2^32 -> CPB_BAD_LENGTH before any array is read; _dev forms skip an index >= n, host forms return
 * CPB_BAD_PARAMS for it before any copy.  Digests are affine points (8 words each, as the build writes them).
 * The digest forms take new_leaf_digests_xy[k] (e.g. cpb_pedersen_crh_batch outputs); the leaf forms take byte leaves and hash
 * all k of them with leaf_ctx on the same stream first: leaf i at new_leaves + i * leaf_stride (_dev form) or packed k x leaf_len
 * (host form); leaf_len * 8 > WINDOW_SIZE * NUM_WINDOWS of leaf_ctx -> CPB_BAD_LENGTH, as the CRH; leaf_stride < leaf_len with
 * k > 1 -> CPB_BAD_PARAMS.  Both curves and every chunk
 * width of cpb_pedersen_ctx_create_ex.
 * _dev forms: device pointers, no host synchronisation, scratch from the stream-ordered pool (about sum over levels l of
 * min(k, 2^l) points plus 128 bytes per slot of the widest inner level); launches depend on the tree height only -- per wide inner
 * level one row kernel and the node context's hash and normalisation, then one warp-per-node launch for the narrow levels above.  Host forms: host arrays; only the siblings the touched
 * nodes read are uploaded and only the touched nodes come back. */
cpb_status cpb_merkle_pedersen_update_digests_dev(cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy, size_t n,
                                                  const uint64_t* indexes, const uint64_t* new_leaf_digests_xy, size_t k,
                                                  const uint64_t* asserted_root_xy, uint8_t* applied, void* stream);
cpb_status cpb_merkle_pedersen_update_dev(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy,
                                          uint64_t* non_leaf_nodes_xy, size_t n, const uint64_t* indexes, const uint8_t* new_leaves,
                                          size_t leaf_len, size_t leaf_stride, size_t k, const uint64_t* asserted_root_xy, uint8_t* applied,
                                          void* stream);
cpb_status cpb_merkle_pedersen_update_digests(cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy, size_t n,
                                              const uint64_t* indexes, const uint64_t* new_leaf_digests_xy, size_t k,
                                              const uint64_t* asserted_root_xy, int* applied);
cpb_status cpb_merkle_pedersen_update(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, uint64_t* leaf_nodes_xy, uint64_t* non_leaf_nodes_xy,
                                      size_t n, const uint64_t* indexes, const uint8_t* new_leaves, size_t leaf_len, size_t k,
                                      const uint64_t* asserted_root_xy, int* applied);
/* MerkleTree::new for Config{Leaf=[u8], LeafHash=PedersenCRHCompressor<C,TECompressor,W>,
 * IdentityDigestConverter, TwoToOneHash=poseidon::TwoToOneCRH<Fq>} (BASELINE config 5): leaf digest =
 * x-coordinate, a base-field element; the Poseidon field must be the curve's base field. */
cpb_status cpb_merkle_mixed_build(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint8_t* leaves,
                                  size_t leaf_len, size_t n, uint64_t* leaf_nodes, uint64_t* non_leaf_nodes);
cpb_status cpb_merkle_mixed_build_dev(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint8_t* leaves,
                                      size_t leaf_len, size_t leaf_stride, size_t n, uint64_t* leaf_nodes,
                                      uint64_t* non_leaf_nodes, void* stream);

/* ---- Merkle path verification (Pedersen leaves) ------------------------------------------------------------------- */
/* n x Path::verify (R/merkle_tree/mod.rs:172-212) for the byte tree of cpb_merkle_pedersen_build against one root (8 words,
 * affine x, y).  Proof i = (leaf_sibling_hashes_xy[i], auth_paths_xy[i*path_len .. (i+1)*path_len) root side first as
 * Path.auth_path, leaf_indexes[i]); ok[i] = 1 when the recomputed root equals root_xy in both coordinates, else 0.  Tree height =
 * path_len + 2.
 * Order of hashing, as the reference: the claimed leaf hash (pedersen::CRH of leaf i with leaf_ctx) and the leaf sibling go through
 * TwoToOneHash::evaluate of the converted digests, sides chosen by index bit 0 (bit set: the computed node is the right child);
 * auth-path level j = 1 .. path_len (auth_paths[i*path_len + path_len - j]) then goes through compress with bit j.  Both steps hash
 * the 128-byte ByteDigestConverter row x_l || y_l || x_r || y_r cut to the node context's TwoToOneCRH length, as the build does.
 * Bits of leaf_indexes[i] above path_len are ignored, as in the reference; no form rejects a large index (the verifier does not
 * know the tree).
 * Argument checks, on the host before any device work, in this order:
 *   1. path_len > 62 -> CPB_BAD_PARAMS; _dev form: leaf_stride < leaf_len with n > 1 -> CPB_BAD_PARAMS;
 *   2. a null buffer with n > 0 (leaves only when leaf_len > 0, auth_paths only when path_len > 0) -> CPB_NULL_POINTER;
 *   3. a null context -> CPB_NULL_POINTER; leaf and node contexts on different devices or curves -> CPB_BAD_PARAMS;
 *   4. leaf_len * 8 > WINDOW_SIZE * NUM_WINDOWS of leaf_ctx -> CPB_BAD_LENGTH, as the CRH; the node row length is checked against
 *      node_ctx as cpb_pedersen_two_to_one_batch does.
 * Then n == 0 returns CPB_OK without reading any array or writing `ok`.
 * Elements are reduced Montgomery limbs; an unreduced one may give any verdict but nothing outside the caller's arrays is read or
 * written.
 * _dev form: every pointer is device memory, leaf i at leaves + i * leaf_stride.  No host synchronisation; scratch (192 bytes per
 * proof) comes from the stream-ordered pool; 3 * path_len + 6 kernel launches whatever n (the leaf hash and its normalisation, per
 * level a row kernel and the node context's hash and normalisation, a comparison), so the call can be captured in a CUDA graph.
 * Host form: leaves packed n x leaf_len; the arrays go up on leaf_ctx's stream, the _dev code runs there, ok comes back. */
cpb_status cpb_merkle_pedersen_verify_batch(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, const uint64_t* root_xy,
                                            const uint8_t* leaves, size_t leaf_len, const uint64_t* leaf_sibling_hashes_xy,
                                            const uint64_t* auth_paths_xy, size_t path_len, const uint64_t* leaf_indexes,
                                            uint8_t* ok, size_t n);
cpb_status cpb_merkle_pedersen_verify_batch_dev(cpb_pedersen_ctx* leaf_ctx, cpb_pedersen_ctx* node_ctx, const uint64_t* root_xy,
                                                const uint8_t* leaves, size_t leaf_len, size_t leaf_stride,
                                                const uint64_t* leaf_sibling_hashes_xy, const uint64_t* auth_paths_xy, size_t path_len,
                                                const uint64_t* leaf_indexes, uint8_t* ok, size_t n, void* stream);
/* The same for the tree of cpb_merkle_mixed_build: leaf digest = PedersenCRHCompressor x-coordinate (one base-field element),
 * nodes poseidon::TwoToOneCRH; root, siblings and auth-path nodes are field elements (4 words).  Rules as above, except for the
 * contexts: a Poseidon field that is not the curve's base field, or another device, -> CPB_BAD_PARAMS, as the mixed build; a
 * Poseidon node rate < 2 -> CPB_UNSUPPORTED, as cpb_merkle_poseidon_verify_batch.  The _dev form takes 3 kernel launches for
 * any path_len and n (leaf hash, normalisation, one fold kernel with one thread per proof) and 32 bytes of pool scratch per proof. */
cpb_status cpb_merkle_mixed_verify_batch(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                         const uint8_t* leaves, size_t leaf_len, const uint64_t* leaf_sibling_hashes,
                                         const uint64_t* auth_paths, size_t path_len, const uint64_t* leaf_indexes,
                                         uint8_t* ok, size_t n);
cpb_status cpb_merkle_mixed_verify_batch_dev(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, const uint64_t* root,
                                             const uint8_t* leaves, size_t leaf_len, size_t leaf_stride,
                                             const uint64_t* leaf_sibling_hashes, const uint64_t* auth_paths, size_t path_len,
                                             const uint64_t* leaf_indexes, uint8_t* ok, size_t n, void* stream);

/* ---- Merkle tree across several GPUs ------------------------------------------------------------ */
/* The reference builds a tree in one process (MerkleTree::new, R/merkle_tree/mod.rs:411-523).  On G = 2^g GPUs the leaves
 * are sharded contiguously: rank k owns leaves [k*n/G, (k+1)*n/G), builds that subtree (its nodes in LOCAL heap order, as
 * if it were a tree of its own), the G subtree roots are exchanged once and every rank computes the g top levels
 * (`top_nodes`: G-1 digests in heap order, root first).  Because the reference's node array is heap-ordered by level,
 * local level l of rank k is the k-th contiguous slice of global level l+g.  Two-to-one hash: poseidon::TwoToOneCRH
 * (rate 2, capacity 1, alpha >= 2).
 *
 * (a) One process per GPU.  Each rank creates a cpb_exchange on its device, publishes its 64-byte CUDA-IPC handle to the
 * others by any means (torch.distributed, MPI, a file), and connects.  The *_sharded calls are collective: every rank
 * issues them in the same order.  The last kernel of the local build pushes the rank's root into every peer's exchange
 * buffer over NVLink (peer stores), waits for theirs and computes the top levels -- no host round trip, no second launch.
 * (b) One process, several GPUs: the cpb_multi group further down. */
cpb_status cpb_exchange_create(int device, int world, int rank, cpb_exchange** out);
void cpb_exchange_destroy(cpb_exchange* ex);
int cpb_exchange_world(const cpb_exchange* ex);
int cpb_exchange_rank(const cpb_exchange* ex);
cpb_status cpb_exchange_ipc_handle(cpb_exchange* ex, uint8_t handle_out[64]);
/* handles: world x 64 bytes, entry r = rank r's handle (the own entry is ignored). */
cpb_status cpb_exchange_connect_ipc(cpb_exchange* ex, const uint8_t* handles);
/* All `world` exchanges live in THIS process (all[r] has rank r): enables peer access and wires them directly. */
cpb_status cpb_exchange_connect_local(cpb_exchange** all, int world);

/* This rank's part of MerkleTree::new: leaves (n_local x leaf_len elements, n_local a power of two > 1) -> leaf_nodes
 * [n_local], non_leaf_nodes [n_local - 1] (local heap order), top_nodes [world - 1] (identical on every rank; unused
 * when world == 1).  _dev: device pointers on the exchange's device, asynchronous on `stream`. */
cpb_status cpb_merkle_poseidon_build_sharded_dev(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, cpb_exchange* ex,
                                                 const uint64_t* leaves, size_t leaf_len, size_t n_local, uint64_t* leaf_nodes,
                                                 uint64_t* non_leaf_nodes, uint64_t* top_nodes, void* stream);
cpb_status cpb_merkle_poseidon_build_sharded(cpb_poseidon_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, cpb_exchange* ex,
                                             const uint64_t* leaves, size_t leaf_len, size_t n_local, uint64_t* leaf_nodes,
                                             uint64_t* non_leaf_nodes, uint64_t* top_nodes);
/* new_with_leaf_digest, sharded: this rank's leaf digests -> its inner nodes + the replicated top (used by the mixed tree). */
cpb_status cpb_merkle_poseidon_from_digests_sharded_dev(cpb_poseidon_ctx* node_ctx, cpb_exchange* ex, const uint64_t* leaf_digests,
                                                        size_t n_local, uint64_t* non_leaf_nodes, uint64_t* top_nodes, void* stream);
/* BASELINE config 5, sharded: Pedersen leaf hash (x-coordinate) + Poseidon levels; see cpb_merkle_mixed_build_dev. */
cpb_status cpb_merkle_mixed_build_sharded_dev(cpb_pedersen_ctx* leaf_ctx, cpb_poseidon_ctx* node_ctx, cpb_exchange* ex,
                                              const uint8_t* leaves, size_t leaf_len, size_t leaf_stride, size_t n_local,
                                              uint64_t* leaf_nodes, uint64_t* non_leaf_nodes, uint64_t* top_nodes, void* stream);

/* (b) One process, several GPUs.  `devices`: ndev distinct device ids, ndev a power of two.  The root exchange is the fused
 * peer-memory kernel when every pair of devices has peer access, otherwise (or with CPB_MULTI_EXCHANGE=nccl in the
 * environment) one ncclAllGather of the subtree roots over communicators from ncclCommInitAll; libnccl.so.2 is loaded on
 * first use (CPB_NCCL_ERROR when it is missing or a call fails). */
cpb_status cpb_multi_create(int ndev, const int* devices, cpb_multi** out);
void cpb_multi_destroy(cpb_multi* m);
int cpb_multi_uses_nccl(const cpb_multi* m);
/* MerkleTree::new (R/merkle_tree/mod.rs:411-422) over HOST arrays in the reference's layout -- leaves: n x leaf_len
 * elements; leaf_nodes[n]; non_leaf_nodes[n-1] in GLOBAL heap order -- computed on the ndev devices of `m`:
 * leaf_ctxs[d] / node_ctxs[d] are contexts of the same parameters created on devices[d].  Copies are pipelined with the
 * hashing per device; one host thread per device.  n / ndev must be >= 2. */
cpb_status cpb_merkle_poseidon_build_multi(cpb_multi* m, cpb_poseidon_ctx* const* leaf_ctxs, cpb_poseidon_ctx* const* node_ctxs,
                                           const uint64_t* leaves, size_t leaf_len, size_t n, uint64_t* leaf_nodes,
                                           uint64_t* non_leaf_nodes);

/* ---- wire formats --------------------------------------------------------------------------------- */
/* `CanonicalSerialize` / `CanonicalDeserialize` images of the types that cross the boundary (derives at
 * R/sponge/poseidon/mod.rs:25, R/crh/pedersen/mod.rs:28, R/merkle_tree/mod.rs:139,239), for hosts that exchange parameters
 * or proofs with an arkworks process as bytes (a Rust host serialises with ark-serialize itself).  Host code, no GPU.
 * Leaf encodings are ark-serialize / ark-ff / ark-ec 0.4 conventions (dependencies of the reference, not vendored;
 * restated, not pinned by reference vectors): u64/usize = 8 bytes LE; Vec<T> = u64 length + elements; Fp = ceil(bits/8)
 * bytes LE of the canonical value; twisted-Edwards affine point compressed = y with bit 7 of the last byte set when x > -x,
 * uncompressed = x || y.  Errors: CPB_BAD_LENGTH = unexpected end / trailing bytes / output buffer too small,
 * CPB_BAD_PARAMS = "invalid data" (unreduced element, not a curve point, not in the prime-order subgroup when `validate`).
 * Serialisers write `*written`; with out == NULL they only report the size. */
size_t cpb_field_serialized_size(int field_id);
cpb_status cpb_field_serialize(int field_id, const uint64_t* mont, size_t n, uint8_t* out);
cpb_status cpb_field_deserialize(int field_id, const uint8_t* in, size_t n, uint64_t* mont_out);
size_t cpb_point_serialized_size(int curve_id, int compress);
cpb_status cpb_point_serialize(int curve_id, const uint64_t* xy, size_t n, int compress, uint8_t* out);
cpb_status cpb_point_deserialize(int curve_id, const uint8_t* in, size_t n, int compress, int validate, uint64_t* xy_out);
/* PoseidonConfig{full_rounds, partial_rounds, alpha, ark, mds, rate, capacity} (R/sponge/poseidon/mod.rs:26-45). */
cpb_status cpb_poseidon_config_serialize(int field_id, int rate, int capacity, int full_rounds, int partial_rounds, uint64_t alpha,
                                         const uint64_t* ark, const uint64_t* mds, uint8_t* out, size_t out_cap, size_t* written);
/* ark_out / mds_out may be NULL: the shape outputs alone (first pass), then a second call with buffers. */
cpb_status cpb_poseidon_config_deserialize(int field_id, const uint8_t* in, size_t len, int* rate, int* capacity, int* full_rounds,
                                           int* partial_rounds, uint64_t* alpha, uint64_t* ark_out, size_t ark_cap_elems,
                                           uint64_t* mds_out, size_t mds_cap_elems);
/* crh::pedersen::Parameters{generators: Vec<Vec<C>>} (R/crh/pedersen/mod.rs:28-31); points as affine. */
cpb_status cpb_pedersen_parameters_serialize(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy, int compress,
                                             uint8_t* out, size_t out_cap, size_t* written);
cpb_status cpb_pedersen_parameters_deserialize(int curve_id, const uint8_t* in, size_t len, int compress, int validate, int* window_size,
                                               int* num_windows, uint64_t* generators_xy_out, size_t cap_points);
/* merkle_tree::Path (R/merkle_tree/mod.rs:139-152) and MultiPath (:239-254).  Digest kinds: 0 = field element (id = cpb_field),
 * 1 = compressed / 2 = uncompressed affine point (id = cpb_curve); leaf and inner digests may differ (Config::LeafDigest /
 * InnerDigest).  MultiPath is passed flattened: n paths, suffix_lengths[n], `suffixes` = the suffix digests back to back. */
cpb_status cpb_path_serialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, const uint64_t* leaf_sibling_hash,
                              const uint64_t* auth_path, size_t path_len, uint64_t leaf_index, uint8_t* out, size_t out_cap, size_t* written);
cpb_status cpb_path_deserialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, int validate, const uint8_t* in, size_t len,
                                uint64_t* leaf_sibling_hash, uint64_t* auth_path, size_t path_cap, size_t* path_len, uint64_t* leaf_index);
cpb_status cpb_multipath_serialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, size_t n, const uint64_t* leaf_siblings_hashes,
                                   const uint64_t* prefix_lengths, const uint64_t* suffix_lengths, const uint64_t* suffixes,
                                   const uint64_t* leaf_indexes, uint8_t* out, size_t out_cap, size_t* written);
/* With leaf_siblings_hashes == NULL only *n_paths and *n_suffix_digests are written (size query). */
cpb_status cpb_multipath_deserialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, int validate, const uint8_t* in, size_t len,
                                     size_t* n_paths, size_t* n_suffix_digests, uint64_t* leaf_siblings_hashes, uint64_t* prefix_lengths,
                                     uint64_t* suffix_lengths, uint64_t* suffixes, uint64_t* leaf_indexes, size_t cap_paths,
                                     size_t cap_suffix_digests);

/* ---- Schnorr signatures, ElGamal encryption and the Blake2s commitment over Jubjub and ed-on-BLS12-377 ---------------- */
/* signature::schnorr::Schnorr<EdwardsProjective, Blake2s256> (R/signature/schnorr/mod.rs) and encryption::elgamal::ElGamal
 * (R/encryption/elgamal/mod.rs) for C = ark_ed_on_bls12_381 (Jubjub), the curve of both reference test suites
 * (R/signature/mod.rs:52-105, R/encryption/elgamal/mod.rs:102-128), and for C = ark_ed_on_bls12_377, the curve of the reference's
 * signature benchmark (R/benches/signature.rs:5-10); commitment::blake2s::Commitment (R/commitment/blake2s/mod.rs).  The curve is
 * the context's (cpb_te_base_ctx_create_ex).
 * Layouts: a scalar is an Fr element of the context's curve (CPB_JUBJUB_FR for Jubjub, CPB_ED_ON_BLS12_377_FR for
 * ed-on-BLS12-377) as Montgomery limbs, 4 x uint64; a point is affine over the curve's base field
 * x || y, 8 x uint64; a signature is (prover_response s, verifier_challenge e), 8 x uint64; a ciphertext (c1, c2), 16 x uint64.
 * Messages are ragged bytes: message i = msgs[msg_offsets[i] .. msg_offsets[i+1]), msg_offsets has n + 1 uint64 (the rules of the
 * ragged Poseidon batches above: host forms reject decreasing offsets with CPB_BAD_LENGTH and copy only msgs[offsets[0] ..
 * offsets[n]); _dev forms hash a decreasing pair as an empty message).  n >= 2^32 -> CPB_BAD_LENGTH; n == 0 -> CPB_OK, no launch.
 * PRECONDITIONS.  Public keys, messages and ciphertext points are not checked to be on the curve, and scalars not checked to be
 * reduced, as for field elements elsewhere.  Secret scalars (sk, nonces, ElGamal randomness) index precomputed tables with
 * data-dependent addresses: the computation is not constant time (the reference's `mul` is not either).
 * A _dev call issues several launches on `stream`, takes its scratch from the stream-ordered pool and never synchronises the host. */
typedef struct cpb_te_base_ctx cpb_te_base_ctx;
/* Parameters{generator} of both schemes (schnorr/mod.rs:24-29 without the salt, elgamal/mod.rs:14-16), affine (x, y).  Builds the
 * fixed-base tables of the generator on the device: a Pedersen context (library default chunk width) whose 256 generators are
 * 2^k G, so s*G is the Pedersen hash of the 32-byte little-endian canonical scalar.  cpb_te_base_ctx_create is the Jubjub form:
 * curve_id != CPB_JUBJUB -> CPB_UNSUPPORTED, as it always was.  cpb_te_base_ctx_create_ex takes curve_id CPB_JUBJUB or
 * CPB_ED_ON_BLS12_377 (any other id -> CPB_UNSUPPORTED) and is otherwise the same call; a library that exports it has signatures and
 * encryption over ed-on-BLS12-377.  Both: a generator that is not a reduced point on the curve -> CPB_BAD_PARAMS.
 * Nothing else is assumed about it: it need not lie in the prime-order subgroup. */
cpb_status cpb_te_base_ctx_create(int curve_id, const uint64_t* generator_xy, int device, cpb_te_base_ctx** out);
cpb_status cpb_te_base_ctx_create_ex(int curve_id, const uint64_t* generator_xy, int device, cpb_te_base_ctx** out);
void cpb_te_base_ctx_destroy(cpb_te_base_ctx* ctx);
/* keygen of both schemes (schnorr/mod.rs:65-78, elgamal/mod.rs:55-67): out[i] = scalars[i] * G. */
cpb_status cpb_te_base_mul_batch(cpb_te_base_ctx* ctx, const uint64_t* scalars, uint64_t* out_xy, size_t n);
cpb_status cpb_te_base_mul_batch_dev(cpb_te_base_ctx* ctx, const uint64_t* scalars, uint64_t* out_xy, size_t n, void* stream);
/* Schnorr::sign (schnorr/mod.rs:80-115), one loop iteration per item with the given nonce k: R = k*G, e =
 * Fr::from_random_bytes(Blake2s256(salt || compress(R) || u64_le(len) || msg)), s = k - e*sk.  salt: 32 bytes in HOST memory in both
 * forms (Parameters.salt), copied into the launch.  signed_out[i] = 0 when the challenge is not a field element: the digest
 * keeps its low MODULUS_BIT_SIZE bits and must be below r, which fails for about 1 - r / 2^bits of nonces (Jubjub: 252 bits,
 * 9.4 %; ed-on-BLS12-377: 251 bits, 41.7 %); the caller draws a new nonce for that item, as the reference's loop does.  sigs_out[i] is then (0, 0). */
cpb_status cpb_schnorr_sign_batch(cpb_te_base_ctx* ctx, const uint8_t* salt, const uint64_t* sks, const uint64_t* nonces, const uint8_t* msgs,
                                  const uint64_t* msg_offsets, uint64_t* sigs_out, uint8_t* signed_out, size_t n);
cpb_status cpb_schnorr_sign_batch_dev(cpb_te_base_ctx* ctx, const uint8_t* salt, const uint64_t* sks, const uint64_t* nonces, const uint8_t* msgs,
                                      const uint64_t* msg_offsets, uint64_t* sigs_out, uint8_t* signed_out, size_t n, void* stream);
/* Schnorr::verify (schnorr/mod.rs:117-148): R' = s*G + e*pk, ok_out[i] = 1 when from_random_bytes(Blake2s256(salt || compress(R') ||
 * u64_le(len) || msg)) is Some(e') and e' == e. */
cpb_status cpb_schnorr_verify_batch(cpb_te_base_ctx* ctx, const uint8_t* salt, const uint64_t* pks_xy, const uint8_t* msgs,
                                    const uint64_t* msg_offsets, const uint64_t* sigs, uint8_t* ok_out, size_t n);
cpb_status cpb_schnorr_verify_batch_dev(cpb_te_base_ctx* ctx, const uint8_t* salt, const uint64_t* pks_xy, const uint8_t* msgs,
                                        const uint64_t* msg_offsets, const uint64_t* sigs, uint8_t* ok_out, size_t n, void* stream);
/* Schnorr::randomize_public_key (schnorr/mod.rs:150-174): out[i] = pk[i] + m*G with m = sum_b bitrev8(byte_b) 2^(8b) over the `len`
 * bytes at randomness + i*stride (bytes_to_bits, :185-194, read as little-endian bits), the exact integer of any length, not reduced
 * mod r.  len >= 2^24 -> CPB_BAD_LENGTH; host forms: len > stride (n > 1) -> CPB_BAD_LENGTH. */
cpb_status cpb_schnorr_randomize_public_key_batch(cpb_te_base_ctx* ctx, const uint64_t* pks_xy, const uint8_t* randomness, size_t len,
                                                  size_t stride, uint64_t* out_xy, size_t n);
cpb_status cpb_schnorr_randomize_public_key_batch_dev(cpb_te_base_ctx* ctx, const uint64_t* pks_xy, const uint8_t* randomness, size_t len,
                                                      size_t stride, uint64_t* out_xy, size_t n, void* stream);
/* Schnorr::randomize_signature (schnorr/mod.rs:176-198): (s - e*m, e) in Fr, m as above reduced mod r. */
cpb_status cpb_schnorr_randomize_signature_batch(cpb_te_base_ctx* ctx, const uint64_t* sigs, const uint8_t* randomness, size_t len,
                                                 size_t stride, uint64_t* sigs_out, size_t n);
cpb_status cpb_schnorr_randomize_signature_batch_dev(cpb_te_base_ctx* ctx, const uint64_t* sigs, const uint8_t* randomness, size_t len,
                                                     size_t stride, uint64_t* sigs_out, size_t n, void* stream);
/* ElGamal::encrypt (elgamal/mod.rs:69-84): (r*G, m + r*pk); ElGamal::decrypt (:86-101): c2 - sk*c1. */
cpb_status cpb_elgamal_encrypt_batch(cpb_te_base_ctx* ctx, const uint64_t* pks_xy, const uint64_t* msgs_xy, const uint64_t* rands,
                                     uint64_t* ciphertexts_out, size_t n);
cpb_status cpb_elgamal_encrypt_batch_dev(cpb_te_base_ctx* ctx, const uint64_t* pks_xy, const uint64_t* msgs_xy, const uint64_t* rands,
                                         uint64_t* ciphertexts_out, size_t n, void* stream);
cpb_status cpb_elgamal_decrypt_batch(cpb_te_base_ctx* ctx, const uint64_t* sks, const uint64_t* ciphertexts, uint64_t* msgs_out, size_t n);
cpb_status cpb_elgamal_decrypt_batch_dev(cpb_te_base_ctx* ctx, const uint64_t* sks, const uint64_t* ciphertexts, uint64_t* msgs_out, size_t n,
                                         void* stream);
/* commitment::blake2s::Commitment::commit (R/commitment/blake2s/mod.rs:21-32): out32[i] = Blake2s256(input_i || randomness32[i]);
 * inputs are ragged bytes under the message rules above. */
cpb_status cpb_blake2s_commit_batch(int device, const uint8_t* in, const uint64_t* offsets, const uint8_t* randomness32, uint8_t* out32,
                                    size_t n);
cpb_status cpb_blake2s_commit_batch_dev(int device, const uint8_t* in, const uint64_t* offsets, const uint8_t* randomness32, uint8_t* out32,
                                        size_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CPB200_H */
