// pedersen_internal.cuh -- what the Pedersen context (cpb_pedersen.cu) shares with other translation units of the library: the
// context itself and the hash launch behind every Pedersen entry point.  The Pedersen-node Merkle update
// (cpb_merkle_update_pedersen.cu) hashes its levels through it, so both paths give the same bytes for every window.
#pragma once
#include <mutex>

#include "common.cuh"

namespace cpb {

struct PedersenDev {
    int chunk_bits;      // 8: shared-memory (TMA-staged) tables; 9..22: L2 / HBM resident tables, gathered per lookup
    int n_in_chunks;     // ceil(input bits that can be set / chunk_bits); with 8-bit chunks = input bytes
    int n_rand_chunks;   // ceil(#randomness generators / chunk_bits), 0 without commitment parameters
    int zero;            // always 0 (see PoseidonDev::zero)
};

}  // namespace cpb

struct cpb_pedersen_ctx {
    int curve_id = 0, field_id = 0, device = 0, sms = 132;
    int window_size = 0, num_windows = 0, n_rand = 0;
    size_t nbits = 0;
    cpb::PedersenDev dev{};
    cpb::u32* d_consts = nullptr;
    cpb::u32* d_table = nullptr;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    cpb::Scratch arena;      // the host-pointer entry points' device copies (HostStage), under mu
};

namespace cpb {

// n hashes of `len`-byte messages `stride` bytes apart (and 32-byte randomness for commitments): the context's hash kernel
// (k_pedersen_hash for 8-bit chunks, k_pedersen_hash_gather above), then k_pedersen_normalise into `out` -- mode 0: n x (x, y),
// mode 1: n x x, Montgomery form.  Projective scratch from the stream-ordered pool; no host synchronisation.
cpb_status launch_hash(cpb_pedersen_ctx* c, const uint8_t* in, size_t len, size_t stride, const uint8_t* rand32, u32* out, size_t n,
                       int mode, cudaStream_t st);

// The length rules of the reference: R/crh/pedersen/mod.rs:82-89 (CRH) and R/commitment/pedersen/mod.rs:69-71.
cpb_status check_len(const cpb_pedersen_ctx* c, size_t len, bool commit);

// TwoToOneCRH::evaluate buffer length, R/crh/pedersen/mod.rs:171: (HALF + HALF) / 8 with HALF = bits / 2, at most the 128 bytes
// of two serialised points (a longer buffer is zero padding).
size_t two_to_one_len(const cpb_pedersen_ctx* c);

}  // namespace cpb
