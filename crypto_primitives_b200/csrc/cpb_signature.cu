// cpb_signature.cu -- CUDA kernels + C-ABI for Schnorr signatures (R/signature/schnorr/mod.rs), ElGamal encryption
// (R/encryption/elgamal/mod.rs) over Jubjub and ed-on-BLS12-377, and the Blake2s commitment (R/commitment/blake2s/mod.rs);
// include/cpb200.h.
//
// Fixed-base products s*G run on the Pedersen table machinery: the context owns a Pedersen context whose 256 generators
// are 2^k G (window 256 x 1), and hashing the 32-byte little-endian canonical scalar selects exactly the generators of
// its set bits.  Everything else is one thread per item:
//   k_fr_to_bytes          Fr Montgomery limbs -> 32-byte canonical scalars (the Pedersen input)
//   k_schnorr_sign         compress R, Blake2s(salt || R || len || msg), from_random_bytes, s = k - e*sk
//   k_schnorr_verify       e*pk (variable base) + s*G (mixed addition), affine, compress, hash, compare
//   k_schnorr_rand_pk      m*G over the randomness bytes (variable base, exact integer) + pk
//   k_schnorr_rand_sig     s - e*m in Fr
//   k_elgamal_encrypt      c2 = r*pk + m (c1 = r*G from the tables)
//   k_elgamal_decrypt      c2 - sk*c1
//   k_blake2s_commit       Blake2s(input || r)
// Every kernel but the commitment is a template on the curve (SigCurve below); a context dispatches on its curve id.
// A call issues several launches on one stream and never synchronises the host; scratch comes from the stream-ordered
// pool.  Secret scalars index tables with data-dependent indices: this code is not constant time (nor is the reference's).
#include <cstring>
#include <vector>

#include "blake2s.cuh"
#include "common.cuh"
#include "curve_desc.hpp"
#include "hostfp.hpp"
#include "te_ops.cuh"

namespace cpb {

// A curve of the signature layer: base field Fq and scalar field Fr as device field tags, with their C-ABI ids.
template <class Q, class R, int CURVE, int FQ_ID, int FR_ID> struct SigCurve {
    typedef Q Fq;
    typedef R Fr;
    static constexpr int kCurve = CURVE, kFqId = FQ_ID, kFrId = FR_ID;
    static constexpr int kFrNibbles = (R::BITS + 3) / 4;   // nibbles of a canonical scalar (below r < 2^BITS)
    static_assert(Q::ID == FQ_ID && R::ID == FR_ID, "field tags and ids disagree");
};
typedef SigCurve<Bls12_381_Fr, Jubjub_Fr, CPB_JUBJUB, CPB_BLS12_381_FR, CPB_JUBJUB_FR> JubjubSig;                     // r < 2^252: 63
typedef SigCurve<Bls12_377_Fr, Ed_On_Bls12_377_Fr, CPB_ED_ON_BLS12_377, CPB_BLS12_377_FR, CPB_ED_ON_BLS12_377_FR> Ed377Sig;  // r < 2^251: 63
static_assert(JubjubSig::kFrNibbles == 63 && Ed377Sig::kFrNibbles == 63, "te_mul_var digit count");
constexpr int kSigBlock = 128;

struct Salt {
    u32 w[8];
};

// consts (u32 words): [0..8) base modulus, [8..16) 2d (Montgomery), [16..24) scalar modulus, [24..40) generator (x, y)
struct SigConsts {
    u32 pm[8], d2[8], sm[8];
};
__device__ __forceinline__ void ld_consts(SigConsts& c, const u32* consts, int zero) {
    const u32* ct = consts + (int)threadIdx.x * zero;    // a run-time offset keeps the moduli in registers (fp.cuh)
    ld_elem(c.pm, ct);
    ld_elem(c.d2, ct + 8);
    ld_elem(c.sm, ct + 16);
}

__device__ __forceinline__ void msg_range(const u64* off, long i, u64& start, u64& len) {
    const u64 a = off[i], b = off[i + 1];
    start = a;
    len = b > a ? b - a : 0;                             // a decreasing pair hashes as an empty message
}

template <class C> __device__ __forceinline__ void affine_add(TePoint& acc, const u32* x, const u32* y, const SigConsts& c) {
    u32 yp[8], ym[8], t2d[8];
    te_niels<typename C::Fq>(yp, ym, t2d, x, y, c.d2, c.pm);
    te_madd<typename C::Fq>(acc, yp, ym, t2d, c.pm);
}

// Schnorr challenge: from_random_bytes(Blake2s256(salt || compress(R) || u64_le(len) || msg)), R affine
template <class C>
__device__ __forceinline__ bool schnorr_challenge(u32* e, const Salt& salt, const u32* rx, const u32* ry, const uint8_t* msg,
                                                  u64 len, const SigConsts& c) {
    u32 hdr[18], dg[8];
#pragma unroll
    for (int i = 0; i < 8; i++) hdr[i] = salt.w[i];
    te_compress<typename C::Fq>(hdr + 8, rx, ry, c.pm);
    hdr[16] = (u32)len;
    hdr[17] = (u32)(len >> 32);
    blake2s_256(dg, B2sSchnorr{hdr, msg}, 72 + len);
    return fr_from_random_bytes<typename C::Fr>(e, dg, c.sm);
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_fr_to_bytes(const u32* __restrict__ consts, const u32* __restrict__ sc, int stride_words, u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 a[8];
    ld_elem(a, sc + stride_words * i);
    fp_to_canonical<typename C::Fr>(a, a, c.sm);
    st_elem(out + 8 * i, a);
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_schnorr_sign(const u32* __restrict__ consts, Salt salt, const u32* __restrict__ r_xy, const u32* __restrict__ nonces,
               const u32* __restrict__ sks, const uint8_t* __restrict__ msgs, const u64* __restrict__ off, u32* __restrict__ sigs,
               uint8_t* __restrict__ signed_out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 rx[8], ry[8], e[8], s[8];
    ld_elem(rx, r_xy + 16 * i);
    ld_elem(ry, r_xy + 16 * i + 8);
    u64 start, len;
    msg_range(off, i, start, len);
    const bool ok = schnorr_challenge<C>(e, salt, rx, ry, msgs + start, len, c);
    if (ok) {
        u32 k[8], sk[8];
        ld_elem(k, nonces + 8 * i);
        ld_elem(sk, sks + 8 * i);
        fp_mul<typename C::Fr>(s, e, sk, c.sm);
        fp_sub<typename C::Fr>(s, k, s);                            // prover_response = k - e*sk (mod.rs:106)
    } else {
        fp_zero(s);
        fp_zero(e);
    }
    st_elem(sigs + 16 * i, s);
    st_elem(sigs + 16 * i + 8, e);
    signed_out[i] = ok ? 1 : 0;
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_schnorr_verify(const u32* __restrict__ consts, Salt salt, const u32* __restrict__ sg_xy, const u32* __restrict__ pks,
                 const uint8_t* __restrict__ msgs, const u64* __restrict__ off, const u32* __restrict__ sigs, uint8_t* __restrict__ ok_out,
                 long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 e[8], x[8], y[8];
    ld_elem(e, sigs + 16 * i + 8);
    fp_to_canonical<typename C::Fr>(e, e, c.sm);
    ld_elem(x, pks + 16 * i);
    ld_elem(y, pks + 16 * i + 8);
    TePoint acc;
    te_mul_var<typename C::Fq>(acc, x, y, ScalarWords{e, C::kFrNibbles}, c.d2, c.pm);      // e*pk
    ld_elem(x, sg_xy + 16 * i);
    ld_elem(y, sg_xy + 16 * i + 8);
    affine_add<C>(acc, x, y, c);                                                  // + s*G (mod.rs:124-127)
    te_to_affine<typename C::Fq>(x, y, acc, c.pm);
    u64 start, len;
    msg_range(off, i, start, len);
    u32 e2[8];
    const bool valid = schnorr_challenge<C>(e2, salt, x, y, msgs + start, len, c);
    ld_elem(e, sigs + 16 * i + 8);
    ok_out[i] = valid && fp_eq(e, e2) ? 1 : 0;
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_schnorr_rand_pk(const u32* __restrict__ consts, const u32* __restrict__ pks, const uint8_t* __restrict__ rnd, long len, long stride,
                  u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 gx[8], gy[8], x[8], y[8];
    ld_elem(gx, consts + 24);
    ld_elem(gy, consts + 32);
    TePoint acc;
    te_mul_var<typename C::Fq>(acc, gx, gy, ScalarBitrevBytes{rnd + i * stride, (u64)len}, c.d2, c.pm);
    ld_elem(x, pks + 16 * i);
    ld_elem(y, pks + 16 * i + 8);
    affine_add<C>(acc, x, y, c);
    te_to_affine<typename C::Fq>(x, y, acc, c.pm);
    st_elem(out + 16 * i, x);
    st_elem(out + 16 * i + 8, y);
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_schnorr_rand_sig(const u32* __restrict__ consts, const u32* __restrict__ sigs, const uint8_t* __restrict__ rnd, long len, long stride,
                   u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 r2[8], c256[8], m[8], v[8], s[8], e[8];
#pragma unroll
    for (int k = 0; k < 8; k++) r2[k] = C::Fr::R2(k);
    fp_zero(c256);
    c256[0] = 256;
    fp_mul<typename C::Fr>(c256, c256, r2, c.sm);
    fp_zero(m);
    const uint8_t* p = rnd + i * stride;
#pragma unroll 1
    for (long b = len - 1; b >= 0; b--) {                // multiplier = sum_b bitrev8(byte_b) 256^b in Fr (mod.rs:161-168)
        fp_mul<typename C::Fr>(m, m, c256, c.sm);
        fp_zero(v);
        v[0] = bitrev8(p[b]);
        fp_mul<typename C::Fr>(v, v, r2, c.sm);
        fp_add<typename C::Fr>(m, m, v);
    }
    ld_elem(s, sigs + 16 * i);
    ld_elem(e, sigs + 16 * i + 8);
    fp_mul<typename C::Fr>(m, e, m, c.sm);
    fp_sub<typename C::Fr>(s, s, m);
    st_elem(out + 16 * i, s);
    st_elem(out + 16 * i + 8, e);
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_elgamal_encrypt(const u32* __restrict__ consts, const u32* __restrict__ c1_xy, const u32* __restrict__ pks, const u32* __restrict__ ms,
                  const u32* __restrict__ rs, u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 r[8], x[8], y[8];
    ld_elem(r, rs + 8 * i);
    fp_to_canonical<typename C::Fr>(r, r, c.sm);
    ld_elem(x, pks + 16 * i);
    ld_elem(y, pks + 16 * i + 8);
    TePoint acc;
    te_mul_var<typename C::Fq>(acc, x, y, ScalarWords{r, C::kFrNibbles}, c.d2, c.pm);      // s = r*pk
    ld_elem(x, ms + 16 * i);
    ld_elem(y, ms + 16 * i + 8);
    affine_add<C>(acc, x, y, c);                                                  // c2 = m + s
    te_to_affine<typename C::Fq>(x, y, acc, c.pm);
    st_elem(out + 32 * i + 16, x);
    st_elem(out + 32 * i + 24, y);
    ld_elem(x, c1_xy + 16 * i);
    ld_elem(y, c1_xy + 16 * i + 8);
    st_elem(out + 32 * i, x);
    st_elem(out + 32 * i + 8, y);
}

template <class C>
__global__ void __launch_bounds__(kSigBlock)
k_elgamal_decrypt(const u32* __restrict__ consts, const u32* __restrict__ sks, const u32* __restrict__ cts, u32* __restrict__ out, long n,
                  int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 sk[8], x[8], y[8];
    ld_elem(sk, sks + 8 * i);
    fp_to_canonical<typename C::Fr>(sk, sk, c.sm);
    ld_elem(x, cts + 32 * i);
    ld_elem(y, cts + 32 * i + 8);
    TePoint acc;
    te_mul_var<typename C::Fq>(acc, x, y, ScalarWords{sk, C::kFrNibbles}, c.d2, c.pm);     // s = sk*c1
    te_neg<typename C::Fq>(acc);
    ld_elem(x, cts + 32 * i + 16);
    ld_elem(y, cts + 32 * i + 24);
    affine_add<C>(acc, x, y, c);                                                  // m = c2 - s
    te_to_affine<typename C::Fq>(x, y, acc, c.pm);
    st_elem(out + 16 * i, x);
    st_elem(out + 16 * i + 8, y);
}

__global__ void __launch_bounds__(kSigBlock)
k_blake2s_commit(const uint8_t* __restrict__ in, const u64* __restrict__ off, const uint8_t* __restrict__ rnd, uint8_t* __restrict__ out,
                 long n) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u64 start, len;
    msg_range(off, i, start, len);
    u32 dg[8];
    blake2s_256(dg, B2sConcat{in + start, len, rnd + 32 * i}, len + 32);
#pragma unroll
    for (int k = 0; k < 32; k++) out[32 * i + k] = (uint8_t)(dg[k >> 2] >> (8 * (k & 3)));
}

}  // namespace cpb

using namespace cpb;

struct cpb_te_base_ctx {
    int curve_id = 0, device = 0;
    cpb_pedersen_ctx* ped = nullptr;       // generators 2^k G, k < 256, window 256 x 1
    u32* d_consts = nullptr;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    Scratch arena;      // the host-pointer entry points' device copies (HostStage), under mu
};

namespace {

int grid_of(size_t n) { return (int)((n + kSigBlock - 1) / kSigBlock); }

cpb_status launched(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(CPB_CUDA_ERROR, "%s launch failed: %s", what, cudaGetErrorString(e));
    return CPB_OK;
}

// Stream-ordered device scratch, freed on the same stream when the call returns.
struct PoolBuf {
    void* p = nullptr;
    cudaStream_t st;
    explicit PoolBuf(cudaStream_t s) : st(s) {}
    cpb_status alloc(size_t bytes) {
        CPB_CUDA(cudaMallocAsync(&p, bytes ? bytes : 1, st));
        return CPB_OK;
    }
    ~PoolBuf() {
        if (p) cudaFreeAsync(p, st);
    }
    template <class T> T* as() const { return (T*)p; }
};

cpb_status check_n(size_t n) {
    if (n >= ((size_t)1 << 32)) return fail(CPB_BAD_LENGTH, "batch of %zu items: n must be below 2^32", n);
    return CPB_OK;
}

// randomize_public_key: the byte string's nibble count must fit the multiplication loop's int counter
cpb_status check_rand_len(size_t len) {
    if (len >= ((size_t)1 << 24)) return fail(CPB_BAD_LENGTH, "randomness of %zu bytes: at most 2^24 - 1", len);
    return CPB_OK;
}

cpb_status check_offsets(const uint64_t* off, size_t n) {
    for (size_t i = 0; i < n; i++)
        if (off[i + 1] < off[i]) return fail(CPB_BAD_LENGTH, "offsets decrease at %zu", i);
    return CPB_OK;
}

cpb_status ctx_check(const cpb_te_base_ctx* c) {
    if (!c) return fail(CPB_NULL_POINTER, "null context");
    return CPB_OK;
}

Salt salt_of(const uint8_t* s) {
    Salt r;
    memcpy(r.w, s, 32);
    return r;
}

// s*G for n scalars read at sc + stride_words*i (Fr Montgomery) -> out_xy (n x 16 words), through the Pedersen tables.
template <class C> cpb_status base_mul_dev(cpb_te_base_ctx* c, const u32* sc, int stride_words, u32* out_xy, size_t n, cudaStream_t st) {
    PoolBuf bytes(st);
    CPB_TRY(bytes.alloc(32 * n));
    k_fr_to_bytes<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, sc, stride_words, bytes.as<u32>(), (long)n, 0);
    CPB_TRY(launched("k_fr_to_bytes"));
    return cpb_pedersen_crh_batch_dev(c->ped, bytes.as<uint8_t>(), 32, 32, (uint64_t*)out_xy, n, st);
}

template <class C> cpb_status sign_dev(cpb_te_base_ctx* c, const Salt& salt, const u32* sks, const u32* nonces, const uint8_t* msgs, const u64* off,
                    u32* sigs, uint8_t* signed_out, size_t n, cudaStream_t st) {
    PoolBuf r(st);
    CPB_TRY(r.alloc(64 * n));
    CPB_TRY(base_mul_dev<C>(c, nonces, 8, r.as<u32>(), n, st));
    k_schnorr_sign<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, salt, r.as<u32>(), nonces, sks, msgs, off, sigs, signed_out, (long)n, 0);
    return launched("k_schnorr_sign");
}

template <class C> cpb_status verify_dev(cpb_te_base_ctx* c, const Salt& salt, const u32* pks, const uint8_t* msgs, const u64* off, const u32* sigs,
                      uint8_t* ok, size_t n, cudaStream_t st) {
    PoolBuf sg(st);
    CPB_TRY(sg.alloc(64 * n));
    CPB_TRY(base_mul_dev<C>(c, sigs, 16, sg.as<u32>(), n, st));
    k_schnorr_verify<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, salt, sg.as<u32>(), pks, msgs, off, sigs, ok, (long)n, 0);
    return launched("k_schnorr_verify");
}

template <class C> cpb_status encrypt_dev(cpb_te_base_ctx* c, const u32* pks, const u32* ms, const u32* rs, u32* out, size_t n, cudaStream_t st) {
    PoolBuf c1(st);
    CPB_TRY(c1.alloc(64 * n));
    CPB_TRY(base_mul_dev<C>(c, rs, 8, c1.as<u32>(), n, st));
    k_elgamal_encrypt<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, c1.as<u32>(), pks, ms, rs, out, (long)n, 0);
    return launched("k_elgamal_encrypt");
}

template <class C> cpb_status rand_pk_dev(cpb_te_base_ctx* c, const u32* pks, const uint8_t* rnd, size_t len, size_t stride, u32* out, size_t n,
                                          cudaStream_t st) {
    k_schnorr_rand_pk<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, pks, rnd, (long)len, (long)stride, out, (long)n, 0);
    return launched("k_schnorr_rand_pk");
}

template <class C> cpb_status rand_sig_dev(cpb_te_base_ctx* c, const u32* sigs, const uint8_t* rnd, size_t len, size_t stride, u32* out, size_t n,
                                           cudaStream_t st) {
    k_schnorr_rand_sig<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, sigs, rnd, (long)len, (long)stride, out, (long)n, 0);
    return launched("k_schnorr_rand_sig");
}

template <class C> cpb_status decrypt_dev(cpb_te_base_ctx* c, const u32* sks, const u32* cts, u32* out, size_t n, cudaStream_t st) {
    k_elgamal_decrypt<C><<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, sks, cts, out, (long)n, 0);
    return launched("k_elgamal_decrypt");
}

// fn(C{}) for the context's curve: every launch of a context runs that curve's kernel instances.
template <class Fn> cpb_status on_curve(const cpb_te_base_ctx* c, Fn&& fn) {
    switch (c->curve_id) {
        case CPB_JUBJUB: return fn(JubjubSig{});
        case CPB_ED_ON_BLS12_377: return fn(Ed377Sig{});
    }
    return fail(CPB_INTERNAL_ERROR, "context of curve %d", c->curve_id);
}

// The checks of each operation, in the header's order, shared by its two forms; n == 0 passes them and the call is done.  `host`: the
// host form's checks of its host arrays, which come before the context.
cpb_status check_msgs(const uint8_t* msgs, const uint64_t* off, size_t n) {
    CPB_TRY(check_offsets(off, n));
    if (!msgs && off[n] != off[0]) return fail(CPB_NULL_POINTER, "null messages");
    return CPB_OK;
}
cpb_status check_plain(const cpb_te_base_ctx* c, bool buffers, size_t n) {       // base_mul, encrypt, decrypt
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!buffers) return fail(CPB_NULL_POINTER, "null array");
    return ctx_check(c);
}
cpb_status check_signing(const cpb_te_base_ctx* c, bool buffers, const uint8_t* msgs, const uint64_t* off, size_t n, bool host) {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!buffers) return fail(CPB_NULL_POINTER, "null array");
    if (host) CPB_TRY(check_msgs(msgs, off, n));
    return ctx_check(c);
}
cpb_status check_randomize(const cpb_te_base_ctx* c, bool buffers, size_t len, size_t stride, size_t n, bool public_key, bool host) {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!buffers) return fail(CPB_NULL_POINTER, "null array");
    if (host && len > stride && n > 1) return fail(CPB_BAD_LENGTH, "randomness length %zu exceeds the stride %zu", len, stride);
    if (public_key) CPB_TRY(check_rand_len(len));
    return ctx_check(c);
}
cpb_status check_blake2s(const uint8_t* in, const uint64_t* offsets, bool buffers, size_t n, bool host) {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!buffers) return fail(CPB_NULL_POINTER, "null array");
    if (host) {
        CPB_TRY(check_offsets(offsets, n));
        if (!in && offsets[n] != offsets[0]) return fail(CPB_NULL_POINTER, "null input");
    }
    return CPB_OK;
}
cpb_status blake2s_dev(const uint8_t* in, const u64* offsets, const uint8_t* randomness32, uint8_t* out32, size_t n, cudaStream_t st) {
    k_blake2s_commit<<<grid_of(n), kSigBlock, 0, st>>>(in, offsets, randomness32, out32, (long)n);
    return launched("k_blake2s_commit");
}

// Ragged messages go up as the span [off[0], off[n]) with offsets rebased to start at 0.
std::vector<uint64_t> rebased(const uint64_t* off, size_t n) {
    std::vector<uint64_t> rel(n + 1);
    for (size_t i = 0; i <= n; i++) rel[i] = off[i] - off[0];
    return rel;
}

// Affine doubling over the host field (a = -1, either curve): x3 = 2xy / (1 + d x^2 y^2), y3 = (y^2 + x^2) / (1 - d x^2 y^2).
void host_double(const host::Field& F, const host::Fe& d, host::Fe& x, host::Fe& y) {
    host::Fe xx = F.mul(x, x), yy = F.mul(y, y), xy = F.mul(x, y);
    host::Fe k = F.mul(d, F.mul(xx, yy));
    host::Fe nx = F.mul(F.add(xy, xy), F.inv(F.add(F.one(), k)));
    host::Fe ny = F.mul(F.add(yy, xx), F.inv(F.sub(F.one(), k)));
    x = nx;
    y = ny;
}

}  // namespace

extern "C" {

// The Jubjub-only form, with its contract unchanged: every other curve id is CPB_UNSUPPORTED, before the generator is read.
cpb_status cpb_te_base_ctx_create(int curve_id, const uint64_t* generator_xy, int device, cpb_te_base_ctx** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out) return fail(CPB_NULL_POINTER, "null out");
    *out = nullptr;
    if (curve_id != CPB_JUBJUB)
        return fail(CPB_UNSUPPORTED, "curve %d: cpb_te_base_ctx_create is the Jubjub form; cpb_te_base_ctx_create_ex takes ed-on-BLS12-377",
                    curve_id);
    return cpb_te_base_ctx_create_ex(curve_id, generator_xy, device, out);
    });
}

cpb_status cpb_te_base_ctx_create_ex(int curve_id, const uint64_t* generator_xy, int device, cpb_te_base_ctx** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out) return fail(CPB_NULL_POINTER, "null out");
    *out = nullptr;
    host::CurveDesc cd;
    if (!host::curve_desc(curve_id, cd)) return fail(CPB_UNSUPPORTED, "curve %d: signatures and encryption exist for Jubjub and ed-on-BLS12-377", curve_id);
    if (!generator_xy) return fail(CPB_NULL_POINTER, "null generator");
    host::Field F(host::field_modulus(cd.field_id));
    host::Fe d = cd.d(F);
    host::Fe x, y;
    memcpy(x.l, generator_xy, 32);
    memcpy(y.l, generator_xy + 4, 32);
    if (!F.is_canonical(x) || !F.is_canonical(y)) return fail(CPB_BAD_PARAMS, "generator coordinates are not reduced");
    {
        host::Fe xx = F.mul(x, x), yy = F.mul(y, y);
        if (F.sub(yy, xx) != F.add(F.one(), F.mul(d, F.mul(xx, yy)))) return fail(CPB_BAD_PARAMS, "generator is not on the curve");
    }
    std::vector<uint64_t> gens(256 * 8);
    for (int k = 0; k < 256; k++) {                      // generator k = 2^k G: bit k of the LE scalar selects it
        memcpy(&gens[8 * k], x.l, 32);
        memcpy(&gens[8 * k + 4], y.l, 32);
        host_double(F, d, x, y);
    }
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));
    keep_pool_memory(device);
    cpb_te_base_ctx* c = new cpb_te_base_ctx();
    c->curve_id = curve_id;
    c->device = device;
    cpb_status st = cpb_pedersen_ctx_create_ex(curve_id, 256, 1, gens.data(), 0, nullptr, device, 0, &c->ped);
    if (st != CPB_OK) { delete c; return st; }
    host::Fe d2 = F.add(d, d);
    uint64_t consts[20];
    memcpy(consts, F.p, 32);
    memcpy(consts + 4, d2.l, 32);
    memcpy(consts + 8, cd.order(), 32);
    memcpy(consts + 12, generator_xy, 64);
    cudaError_t e = cudaMalloc(&c->d_consts, sizeof consts);
    if (e == cudaSuccess) e = cudaMemcpy(c->d_consts, consts, sizeof consts, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        cpb_pedersen_ctx_destroy(c->ped);
        if (c->d_consts) cudaFree(c->d_consts);
        delete c;
        return fail(CPB_CUDA_ERROR, "te base context build failed: %s", cudaGetErrorString(e));
    }
    *out = c;
    return CPB_OK;
    });
}

void cpb_te_base_ctx_destroy(cpb_te_base_ctx* c) {
    if (!c) return;
    DeviceGuard g(c->device);
    if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
    if (c->d_consts) cudaFree(c->d_consts);
    cpb_pedersen_ctx_destroy(c->ped);
    delete c;
}

// ---- device-pointer forms
cpb_status cpb_te_base_mul_batch_dev(cpb_te_base_ctx* c, const uint64_t* scalars, uint64_t* out_xy, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_plain(c, scalars && out_xy, n));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) { return base_mul_dev<decltype(k)>(c, (const u32*)scalars, 8, (u32*)out_xy, n, (cudaStream_t)stream); });
    });
}

cpb_status cpb_schnorr_sign_batch_dev(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* sks, const uint64_t* nonces, const uint8_t* msgs,
                                      const uint64_t* msg_offsets, uint64_t* sigs_out, uint8_t* signed_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_signing(c, salt && sks && nonces && msg_offsets && sigs_out && signed_out, msgs, msg_offsets, n, false));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) {
        return sign_dev<decltype(k)>(c, salt_of(salt), (const u32*)sks, (const u32*)nonces, msgs, (const u64*)msg_offsets, (u32*)sigs_out,
                                     signed_out, n, (cudaStream_t)stream);
    });
    });
}

cpb_status cpb_schnorr_verify_batch_dev(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* pks_xy, const uint8_t* msgs,
                                        const uint64_t* msg_offsets, const uint64_t* sigs, uint8_t* ok_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_signing(c, salt && pks_xy && msg_offsets && sigs && ok_out, msgs, msg_offsets, n, false));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) {
        return verify_dev<decltype(k)>(c, salt_of(salt), (const u32*)pks_xy, msgs, (const u64*)msg_offsets, (const u32*)sigs, ok_out, n,
                                       (cudaStream_t)stream);
    });
    });
}

cpb_status cpb_schnorr_randomize_public_key_batch_dev(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint8_t* randomness, size_t len,
                                                      size_t stride, uint64_t* out_xy, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_randomize(c, pks_xy && out_xy && (!len || randomness), len, stride, n, true, false));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) {
        return rand_pk_dev<decltype(k)>(c, (const u32*)pks_xy, randomness, len, stride, (u32*)out_xy, n, (cudaStream_t)stream);
    });
    });
}

cpb_status cpb_schnorr_randomize_signature_batch_dev(cpb_te_base_ctx* c, const uint64_t* sigs, const uint8_t* randomness, size_t len,
                                                     size_t stride, uint64_t* sigs_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_randomize(c, sigs && sigs_out && (!len || randomness), len, stride, n, false, false));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) {
        return rand_sig_dev<decltype(k)>(c, (const u32*)sigs, randomness, len, stride, (u32*)sigs_out, n, (cudaStream_t)stream);
    });
    });
}

cpb_status cpb_elgamal_encrypt_batch_dev(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint64_t* msgs_xy, const uint64_t* rands,
                                         uint64_t* ciphertexts_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_plain(c, pks_xy && msgs_xy && rands && ciphertexts_out, n));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) {
        return encrypt_dev<decltype(k)>(c, (const u32*)pks_xy, (const u32*)msgs_xy, (const u32*)rands, (u32*)ciphertexts_out, n, (cudaStream_t)stream);
    });
    });
}

cpb_status cpb_elgamal_decrypt_batch_dev(cpb_te_base_ctx* c, const uint64_t* sks, const uint64_t* ciphertexts, uint64_t* msgs_out, size_t n,
                                         void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_plain(c, sks && ciphertexts && msgs_out, n));
    if (n == 0) return CPB_OK;
    DeviceGuard g(c->device);
    return on_curve(c, [&](auto k) {
        return decrypt_dev<decltype(k)>(c, (const u32*)sks, (const u32*)ciphertexts, (u32*)msgs_out, n, (cudaStream_t)stream);
    });
    });
}

cpb_status cpb_blake2s_commit_batch_dev(int device, const uint8_t* in, const uint64_t* offsets, const uint8_t* randomness32, uint8_t* out32,
                                        size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_blake2s(in, offsets, offsets && randomness32 && out32, n, false));
    if (n == 0) return CPB_OK;
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));
    return blake2s_dev(in, (const u64*)offsets, randomness32, out32, n, (cudaStream_t)stream);
    });
}

// ---- host-pointer forms: the _dev form's core on the context arena and stream (HostStage), under the context mutex
cpb_status cpb_te_base_mul_batch(cpb_te_base_ctx* c, const uint64_t* scalars, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_plain(c, scalars && out_xy, n));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostStage S(c->arena, c->stream);
    const size_t o_s = S.in(scalars, 32 * n), o_o = S.out(out_xy, 64 * n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) { return base_mul_dev<decltype(k)>(c, S.at<u32>(o_s), 8, S.at<u32>(o_o), n, c->stream); }));
    return S.download();
    });
}

cpb_status cpb_schnorr_sign_batch(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* sks, const uint64_t* nonces, const uint8_t* msgs,
                                  const uint64_t* msg_offsets, uint64_t* sigs_out, uint8_t* signed_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_signing(c, salt && sks && nonces && msg_offsets && sigs_out && signed_out, msgs, msg_offsets, n, true));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    const std::vector<uint64_t> rel = rebased(msg_offsets, n);
    HostStage S(c->arena, c->stream);
    const size_t o_sk = S.in(sks, 32 * n), o_k = S.in(nonces, 32 * n), o_m = S.in(msgs + msg_offsets[0], rel[n]),
                 o_off = S.in(rel.data(), 8 * (n + 1)), o_sig = S.out(sigs_out, 64 * n), o_ok = S.out(signed_out, n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) {
        return sign_dev<decltype(k)>(c, salt_of(salt), S.at<u32>(o_sk), S.at<u32>(o_k), S.at<uint8_t>(o_m), S.at<u64>(o_off), S.at<u32>(o_sig),
                                     S.at<uint8_t>(o_ok), n, c->stream);
    }));
    return S.download();
    });
}

cpb_status cpb_schnorr_verify_batch(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* pks_xy, const uint8_t* msgs,
                                    const uint64_t* msg_offsets, const uint64_t* sigs, uint8_t* ok_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_signing(c, salt && pks_xy && msg_offsets && sigs && ok_out, msgs, msg_offsets, n, true));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    const std::vector<uint64_t> rel = rebased(msg_offsets, n);
    HostStage S(c->arena, c->stream);
    const size_t o_pk = S.in(pks_xy, 64 * n), o_sig = S.in(sigs, 64 * n), o_m = S.in(msgs + msg_offsets[0], rel[n]),
                 o_off = S.in(rel.data(), 8 * (n + 1)), o_ok = S.out(ok_out, n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) {
        return verify_dev<decltype(k)>(c, salt_of(salt), S.at<u32>(o_pk), S.at<uint8_t>(o_m), S.at<u64>(o_off), S.at<u32>(o_sig),
                                       S.at<uint8_t>(o_ok), n, c->stream);
    }));
    return S.download();
    });
}

cpb_status cpb_schnorr_randomize_public_key_batch(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint8_t* randomness, size_t len,
                                                  size_t stride, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_randomize(c, pks_xy && out_xy && (!len || randomness), len, stride, n, true, true));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostStage S(c->arena, c->stream);
    const size_t o_pk = S.in(pks_xy, 64 * n), o_r = S.in(randomness, (n - 1) * stride + len), o_o = S.out(out_xy, 64 * n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) {
        return rand_pk_dev<decltype(k)>(c, S.at<u32>(o_pk), S.at<uint8_t>(o_r), len, stride, S.at<u32>(o_o), n, c->stream);
    }));
    return S.download();
    });
}

cpb_status cpb_schnorr_randomize_signature_batch(cpb_te_base_ctx* c, const uint64_t* sigs, const uint8_t* randomness, size_t len, size_t stride,
                                                 uint64_t* sigs_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_randomize(c, sigs && sigs_out && (!len || randomness), len, stride, n, false, true));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostStage S(c->arena, c->stream);
    const size_t o_s = S.in(sigs, 64 * n), o_r = S.in(randomness, (n - 1) * stride + len), o_o = S.out(sigs_out, 64 * n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) {
        return rand_sig_dev<decltype(k)>(c, S.at<u32>(o_s), S.at<uint8_t>(o_r), len, stride, S.at<u32>(o_o), n, c->stream);
    }));
    return S.download();
    });
}

cpb_status cpb_elgamal_encrypt_batch(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint64_t* msgs_xy, const uint64_t* rands,
                                     uint64_t* ciphertexts_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_plain(c, pks_xy && msgs_xy && rands && ciphertexts_out, n));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostStage S(c->arena, c->stream);
    const size_t o_pk = S.in(pks_xy, 64 * n), o_m = S.in(msgs_xy, 64 * n), o_r = S.in(rands, 32 * n), o_o = S.out(ciphertexts_out, 128 * n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) {
        return encrypt_dev<decltype(k)>(c, S.at<u32>(o_pk), S.at<u32>(o_m), S.at<u32>(o_r), S.at<u32>(o_o), n, c->stream);
    }));
    return S.download();
    });
}

cpb_status cpb_elgamal_decrypt_batch(cpb_te_base_ctx* c, const uint64_t* sks, const uint64_t* ciphertexts, uint64_t* msgs_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_plain(c, sks && ciphertexts && msgs_out, n));
    if (n == 0) return CPB_OK;
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostStage S(c->arena, c->stream);
    const size_t o_sk = S.in(sks, 32 * n), o_ct = S.in(ciphertexts, 128 * n), o_o = S.out(msgs_out, 64 * n);
    CPB_TRY(S.upload());
    CPB_TRY(on_curve(c, [&](auto k) { return decrypt_dev<decltype(k)>(c, S.at<u32>(o_sk), S.at<u32>(o_ct), S.at<u32>(o_o), n, c->stream); }));
    return S.download();
    });
}

// No context: a local arena and a stream of its own, both released before the call returns.
cpb_status cpb_blake2s_commit_batch(int device, const uint8_t* in, const uint64_t* offsets, const uint8_t* randomness32, uint8_t* out32,
                                    size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_blake2s(in, offsets, offsets && randomness32 && out32, n, true));
    if (n == 0) return CPB_OK;
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));
    cudaStream_t st = nullptr;
    CPB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    Scratch arena;
    const std::vector<uint64_t> rel = rebased(offsets, n);
    const cpb_status r = [&]() -> cpb_status {
        HostStage S(arena, st);
        const size_t o_in = S.in(in + offsets[0], rel[n]), o_off = S.in(rel.data(), 8 * (n + 1)), o_r = S.in(randomness32, 32 * n),
                     o_o = S.out(out32, 32 * n);
        CPB_TRY(S.upload());
        CPB_TRY(blake2s_dev(S.at<uint8_t>(o_in), S.at<u64>(o_off), S.at<uint8_t>(o_r), S.at<uint8_t>(o_o), n, st));
        return S.download();
    }();
    cudaStreamDestroy(st);
    return r;
    });
}

}  // extern "C"
