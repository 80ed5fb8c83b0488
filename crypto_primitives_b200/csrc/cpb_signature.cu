// cpb_signature.cu -- CUDA kernels + C-ABI for Schnorr signatures (R/signature/schnorr/mod.rs), ElGamal encryption
// (R/encryption/elgamal/mod.rs) over Jubjub, and the Blake2s commitment (R/commitment/blake2s/mod.rs); include/cpb200.h.
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
// A call issues several launches on one stream and never synchronises the host; scratch comes from the stream-ordered
// pool.  Secret scalars index tables with data-dependent indices: this code is not constant time (nor is the reference's).
#include <cstring>
#include <vector>

#include "blake2s.cuh"
#include "common.cuh"
#include "hostfp.hpp"
#include "te_ops.cuh"

namespace cpb {

typedef Bls12_381_Fr JqF;      // Jubjub base field
typedef Jubjub_Fr JrF;         // Jubjub scalar field
constexpr int kSigBlock = 128;
constexpr int kFrNibbles = 63;  // canonical Fr scalars are below r < 2^252

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

__device__ __forceinline__ void affine_add(TePoint& acc, const u32* x, const u32* y, const SigConsts& c) {
    u32 yp[8], ym[8], t2d[8];
    te_niels<JqF>(yp, ym, t2d, x, y, c.d2, c.pm);
    te_madd<JqF>(acc, yp, ym, t2d, c.pm);
}

// Schnorr challenge: from_random_bytes(Blake2s256(salt || compress(R) || u64_le(len) || msg)), R affine
__device__ __forceinline__ bool schnorr_challenge(u32* e, const Salt& salt, const u32* rx, const u32* ry, const uint8_t* msg,
                                                  u64 len, const SigConsts& c) {
    u32 hdr[18], dg[8];
#pragma unroll
    for (int i = 0; i < 8; i++) hdr[i] = salt.w[i];
    te_compress<JqF>(hdr + 8, rx, ry, c.pm);
    hdr[16] = (u32)len;
    hdr[17] = (u32)(len >> 32);
    blake2s_256(dg, B2sSchnorr{hdr, msg}, 72 + len);
    return fr_from_random_bytes<JrF>(e, dg, c.sm);
}

__global__ void __launch_bounds__(kSigBlock)
k_fr_to_bytes(const u32* __restrict__ consts, const u32* __restrict__ sc, int stride_words, u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 a[8];
    ld_elem(a, sc + stride_words * i);
    fp_to_canonical<JrF>(a, a, c.sm);
    st_elem(out + 8 * i, a);
}

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
    const bool ok = schnorr_challenge(e, salt, rx, ry, msgs + start, len, c);
    if (ok) {
        u32 k[8], sk[8];
        ld_elem(k, nonces + 8 * i);
        ld_elem(sk, sks + 8 * i);
        fp_mul<JrF>(s, e, sk, c.sm);
        fp_sub<JrF>(s, k, s);                            // prover_response = k - e*sk (mod.rs:106)
    } else {
        fp_zero(s);
        fp_zero(e);
    }
    st_elem(sigs + 16 * i, s);
    st_elem(sigs + 16 * i + 8, e);
    signed_out[i] = ok ? 1 : 0;
}

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
    fp_to_canonical<JrF>(e, e, c.sm);
    ld_elem(x, pks + 16 * i);
    ld_elem(y, pks + 16 * i + 8);
    TePoint acc;
    te_mul_var<JqF>(acc, x, y, ScalarWords{e, kFrNibbles}, c.d2, c.pm);      // e*pk
    ld_elem(x, sg_xy + 16 * i);
    ld_elem(y, sg_xy + 16 * i + 8);
    affine_add(acc, x, y, c);                                                  // + s*G (mod.rs:124-127)
    te_to_affine<JqF>(x, y, acc, c.pm);
    u64 start, len;
    msg_range(off, i, start, len);
    u32 e2[8];
    const bool valid = schnorr_challenge(e2, salt, x, y, msgs + start, len, c);
    ld_elem(e, sigs + 16 * i + 8);
    ok_out[i] = valid && fp_eq(e, e2) ? 1 : 0;
}

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
    te_mul_var<JqF>(acc, gx, gy, ScalarBitrevBytes{rnd + i * stride, (u64)len}, c.d2, c.pm);
    ld_elem(x, pks + 16 * i);
    ld_elem(y, pks + 16 * i + 8);
    affine_add(acc, x, y, c);
    te_to_affine<JqF>(x, y, acc, c.pm);
    st_elem(out + 16 * i, x);
    st_elem(out + 16 * i + 8, y);
}

__global__ void __launch_bounds__(kSigBlock)
k_schnorr_rand_sig(const u32* __restrict__ consts, const u32* __restrict__ sigs, const uint8_t* __restrict__ rnd, long len, long stride,
                   u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 r2[8], c256[8], m[8], v[8], s[8], e[8];
#pragma unroll
    for (int k = 0; k < 8; k++) r2[k] = JrF::R2(k);
    fp_zero(c256);
    c256[0] = 256;
    fp_mul<JrF>(c256, c256, r2, c.sm);
    fp_zero(m);
    const uint8_t* p = rnd + i * stride;
#pragma unroll 1
    for (long b = len - 1; b >= 0; b--) {                // multiplier = sum_b bitrev8(byte_b) 256^b in Fr (mod.rs:161-168)
        fp_mul<JrF>(m, m, c256, c.sm);
        fp_zero(v);
        v[0] = bitrev8(p[b]);
        fp_mul<JrF>(v, v, r2, c.sm);
        fp_add<JrF>(m, m, v);
    }
    ld_elem(s, sigs + 16 * i);
    ld_elem(e, sigs + 16 * i + 8);
    fp_mul<JrF>(m, e, m, c.sm);
    fp_sub<JrF>(s, s, m);
    st_elem(out + 16 * i, s);
    st_elem(out + 16 * i + 8, e);
}

__global__ void __launch_bounds__(kSigBlock)
k_elgamal_encrypt(const u32* __restrict__ consts, const u32* __restrict__ c1_xy, const u32* __restrict__ pks, const u32* __restrict__ ms,
                  const u32* __restrict__ rs, u32* __restrict__ out, long n, int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 r[8], x[8], y[8];
    ld_elem(r, rs + 8 * i);
    fp_to_canonical<JrF>(r, r, c.sm);
    ld_elem(x, pks + 16 * i);
    ld_elem(y, pks + 16 * i + 8);
    TePoint acc;
    te_mul_var<JqF>(acc, x, y, ScalarWords{r, kFrNibbles}, c.d2, c.pm);      // s = r*pk
    ld_elem(x, ms + 16 * i);
    ld_elem(y, ms + 16 * i + 8);
    affine_add(acc, x, y, c);                                                  // c2 = m + s
    te_to_affine<JqF>(x, y, acc, c.pm);
    st_elem(out + 32 * i + 16, x);
    st_elem(out + 32 * i + 24, y);
    ld_elem(x, c1_xy + 16 * i);
    ld_elem(y, c1_xy + 16 * i + 8);
    st_elem(out + 32 * i, x);
    st_elem(out + 32 * i + 8, y);
}

__global__ void __launch_bounds__(kSigBlock)
k_elgamal_decrypt(const u32* __restrict__ consts, const u32* __restrict__ sks, const u32* __restrict__ cts, u32* __restrict__ out, long n,
                  int zero) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    u32 sk[8], x[8], y[8];
    ld_elem(sk, sks + 8 * i);
    fp_to_canonical<JrF>(sk, sk, c.sm);
    ld_elem(x, cts + 32 * i);
    ld_elem(y, cts + 32 * i + 8);
    TePoint acc;
    te_mul_var<JqF>(acc, x, y, ScalarWords{sk, kFrNibbles}, c.d2, c.pm);     // s = sk*c1
    te_neg<JqF>(acc);
    ld_elem(x, cts + 32 * i + 16);
    ld_elem(y, cts + 32 * i + 24);
    affine_add(acc, x, y, c);                                                  // m = c2 - s
    te_to_affine<JqF>(x, y, acc, c.pm);
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
cpb_status base_mul_dev(cpb_te_base_ctx* c, const u32* sc, int stride_words, u32* out_xy, size_t n, cudaStream_t st) {
    PoolBuf bytes(st);
    CPB_TRY(bytes.alloc(32 * n));
    k_fr_to_bytes<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, sc, stride_words, bytes.as<u32>(), (long)n, 0);
    CPB_TRY(launched("k_fr_to_bytes"));
    return cpb_pedersen_crh_batch_dev(c->ped, bytes.as<uint8_t>(), 32, 32, (uint64_t*)out_xy, n, st);
}

cpb_status sign_dev(cpb_te_base_ctx* c, const Salt& salt, const u32* sks, const u32* nonces, const uint8_t* msgs, const u64* off,
                    u32* sigs, uint8_t* signed_out, size_t n, cudaStream_t st) {
    PoolBuf r(st);
    CPB_TRY(r.alloc(64 * n));
    CPB_TRY(base_mul_dev(c, nonces, 8, r.as<u32>(), n, st));
    k_schnorr_sign<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, salt, r.as<u32>(), nonces, sks, msgs, off, sigs, signed_out, (long)n, 0);
    return launched("k_schnorr_sign");
}

cpb_status verify_dev(cpb_te_base_ctx* c, const Salt& salt, const u32* pks, const uint8_t* msgs, const u64* off, const u32* sigs,
                      uint8_t* ok, size_t n, cudaStream_t st) {
    PoolBuf sg(st);
    CPB_TRY(sg.alloc(64 * n));
    CPB_TRY(base_mul_dev(c, sigs, 16, sg.as<u32>(), n, st));
    k_schnorr_verify<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, salt, sg.as<u32>(), pks, msgs, off, sigs, ok, (long)n, 0);
    return launched("k_schnorr_verify");
}

cpb_status encrypt_dev(cpb_te_base_ctx* c, const u32* pks, const u32* ms, const u32* rs, u32* out, size_t n, cudaStream_t st) {
    PoolBuf c1(st);
    CPB_TRY(c1.alloc(64 * n));
    CPB_TRY(base_mul_dev(c, rs, 8, c1.as<u32>(), n, st));
    k_elgamal_encrypt<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, c1.as<u32>(), pks, ms, rs, out, (long)n, 0);
    return launched("k_elgamal_encrypt");
}

// Host-form plumbing: uploads on the context's stream, one synchronisation at the end.
struct HostCall {
    cudaStream_t st;
    std::vector<void*> bufs;
    explicit HostCall(cudaStream_t s) : st(s) {}
    ~HostCall() {
        for (void* p : bufs) cudaFreeAsync(p, st);
        cudaStreamSynchronize(st);
    }
    template <class T> cpb_status alloc(T*& d, size_t bytes) {
        void* p = nullptr;
        CPB_CUDA(cudaMallocAsync(&p, bytes ? bytes : 1, st));
        bufs.push_back(p);
        d = (T*)p;
        return CPB_OK;
    }
    template <class T> cpb_status up(T*& d, const void* h, size_t bytes) {
        CPB_TRY(alloc(d, bytes));
        if (bytes) CPB_CUDA(cudaMemcpyAsync((void*)d, h, bytes, cudaMemcpyHostToDevice, st));
        return CPB_OK;
    }
    cpb_status down(void* h, const void* d, size_t bytes) {
        if (bytes) CPB_CUDA(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st));
        CPB_CUDA(cudaStreamSynchronize(st));
        return CPB_OK;
    }
    // ragged messages: only bytes [off[0], off[n]) are copied; device offsets are rebased to start at 0
    cpb_status messages(const uint8_t*& d_msgs, const u64*& d_off, const uint8_t* msgs, const uint64_t* off, size_t n) {
        std::vector<uint64_t> rel(n + 1);
        for (size_t i = 0; i <= n; i++) rel[i] = off[i] - off[0];
        uint8_t* m = nullptr;
        u64* o = nullptr;
        CPB_TRY(up(m, msgs + off[0], rel[n]));
        CPB_TRY(up(o, rel.data(), 8 * (n + 1)));
        d_msgs = m;
        d_off = o;
        return CPB_OK;
    }
};

// Affine doubling over the host field (a = -1): x3 = 2xy / (1 + d x^2 y^2), y3 = (y^2 + x^2) / (1 - d x^2 y^2).
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

cpb_status cpb_te_base_ctx_create(int curve_id, const uint64_t* generator_xy, int device, cpb_te_base_ctx** out) {
    return cpb::guarded([&]() -> cpb_status {
    if (!out) return fail(CPB_NULL_POINTER, "null out");
    *out = nullptr;
    if (curve_id != CPB_JUBJUB)
        return fail(CPB_UNSUPPORTED, "curve %d: signatures and encryption need scalar-field arithmetic on the device, which exists for Jubjub only",
                    curve_id);
    if (!generator_xy) return fail(CPB_NULL_POINTER, "null generator");
    host::Field F(host::field_modulus(CPB_BLS12_381_FR));
    host::Fe d = F.neg(F.mul(F.from_u64(10240), F.inv(F.from_u64(10241))));
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
    cpb_status st = cpb_pedersen_ctx_create_ex(CPB_JUBJUB, 256, 1, gens.data(), 0, nullptr, device, 0, &c->ped);
    if (st != CPB_OK) { delete c; return st; }
    host::Fe d2 = F.add(d, d);
    uint64_t consts[20];
    memcpy(consts, F.p, 32);
    memcpy(consts + 4, d2.l, 32);
    memcpy(consts + 8, host::field_modulus(CPB_JUBJUB_FR), 32);
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
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!scalars || !out_xy) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    return base_mul_dev(c, (const u32*)scalars, 8, (u32*)out_xy, n, (cudaStream_t)stream);
    });
}

cpb_status cpb_schnorr_sign_batch_dev(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* sks, const uint64_t* nonces, const uint8_t* msgs,
                                      const uint64_t* msg_offsets, uint64_t* sigs_out, uint8_t* signed_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!salt || !sks || !nonces || !msg_offsets || !sigs_out || !signed_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    return sign_dev(c, salt_of(salt), (const u32*)sks, (const u32*)nonces, msgs, (const u64*)msg_offsets, (u32*)sigs_out, signed_out, n,
                    (cudaStream_t)stream);
    });
}

cpb_status cpb_schnorr_verify_batch_dev(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* pks_xy, const uint8_t* msgs,
                                        const uint64_t* msg_offsets, const uint64_t* sigs, uint8_t* ok_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!salt || !pks_xy || !msg_offsets || !sigs || !ok_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    return verify_dev(c, salt_of(salt), (const u32*)pks_xy, msgs, (const u64*)msg_offsets, (const u32*)sigs, ok_out, n, (cudaStream_t)stream);
    });
}

cpb_status cpb_schnorr_randomize_public_key_batch_dev(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint8_t* randomness, size_t len,
                                                      size_t stride, uint64_t* out_xy, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!pks_xy || !out_xy || (len && !randomness)) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(check_rand_len(len));
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    k_schnorr_rand_pk<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, (const u32*)pks_xy, randomness, (long)len, (long)stride, (u32*)out_xy,
                                                       (long)n, 0);
    return launched("k_schnorr_rand_pk");
    });
}

cpb_status cpb_schnorr_randomize_signature_batch_dev(cpb_te_base_ctx* c, const uint64_t* sigs, const uint8_t* randomness, size_t len,
                                                     size_t stride, uint64_t* sigs_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!sigs || !sigs_out || (len && !randomness)) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    k_schnorr_rand_sig<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, (const u32*)sigs, randomness, (long)len, (long)stride, (u32*)sigs_out,
                                                        (long)n, 0);
    return launched("k_schnorr_rand_sig");
    });
}

cpb_status cpb_elgamal_encrypt_batch_dev(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint64_t* msgs_xy, const uint64_t* rands,
                                         uint64_t* ciphertexts_out, size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!pks_xy || !msgs_xy || !rands || !ciphertexts_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    return encrypt_dev(c, (const u32*)pks_xy, (const u32*)msgs_xy, (const u32*)rands, (u32*)ciphertexts_out, n, (cudaStream_t)stream);
    });
}

cpb_status cpb_elgamal_decrypt_batch_dev(cpb_te_base_ctx* c, const uint64_t* sks, const uint64_t* ciphertexts, uint64_t* msgs_out, size_t n,
                                         void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!sks || !ciphertexts || !msgs_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    DeviceGuard g(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    k_elgamal_decrypt<<<grid_of(n), kSigBlock, 0, st>>>(c->d_consts, (const u32*)sks, (const u32*)ciphertexts, (u32*)msgs_out, (long)n, 0);
    return launched("k_elgamal_decrypt");
    });
}

cpb_status cpb_blake2s_commit_batch_dev(int device, const uint8_t* in, const uint64_t* offsets, const uint8_t* randomness32, uint8_t* out32,
                                        size_t n, void* stream) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!offsets || !randomness32 || !out32) return fail(CPB_NULL_POINTER, "null array");
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));
    k_blake2s_commit<<<grid_of(n), kSigBlock, 0, (cudaStream_t)stream>>>(in, (const u64*)offsets, randomness32, out32, (long)n);
    return launched("k_blake2s_commit");
    });
}

// ---- host-pointer forms
cpb_status cpb_te_base_mul_batch(cpb_te_base_ctx* c, const uint64_t* scalars, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!scalars || !out_xy) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_s, *d_o;
    CPB_TRY(h.up(d_s, scalars, 32 * n));
    CPB_TRY(h.alloc(d_o, 64 * n));
    CPB_TRY(base_mul_dev(c, d_s, 8, d_o, n, c->stream));
    return h.down(out_xy, d_o, 64 * n);
    });
}

cpb_status cpb_schnorr_sign_batch(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* sks, const uint64_t* nonces, const uint8_t* msgs,
                                  const uint64_t* msg_offsets, uint64_t* sigs_out, uint8_t* signed_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!salt || !sks || !nonces || !msg_offsets || !sigs_out || !signed_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(check_offsets(msg_offsets, n));
    if (!msgs && msg_offsets[n] != msg_offsets[0]) return fail(CPB_NULL_POINTER, "null messages");
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_sk, *d_k, *d_sig;
    uint8_t* d_ok;
    const uint8_t* d_m;
    const u64* d_off;
    CPB_TRY(h.up(d_sk, sks, 32 * n));
    CPB_TRY(h.up(d_k, nonces, 32 * n));
    CPB_TRY(h.messages(d_m, d_off, msgs, msg_offsets, n));
    CPB_TRY(h.alloc(d_sig, 64 * n));
    CPB_TRY(h.alloc(d_ok, n));
    CPB_TRY(sign_dev(c, salt_of(salt), d_sk, d_k, d_m, d_off, d_sig, d_ok, n, c->stream));
    CPB_CUDA(cudaMemcpyAsync(signed_out, d_ok, n, cudaMemcpyDeviceToHost, c->stream));
    return h.down(sigs_out, d_sig, 64 * n);
    });
}

cpb_status cpb_schnorr_verify_batch(cpb_te_base_ctx* c, const uint8_t* salt, const uint64_t* pks_xy, const uint8_t* msgs,
                                    const uint64_t* msg_offsets, const uint64_t* sigs, uint8_t* ok_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!salt || !pks_xy || !msg_offsets || !sigs || !ok_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(check_offsets(msg_offsets, n));
    if (!msgs && msg_offsets[n] != msg_offsets[0]) return fail(CPB_NULL_POINTER, "null messages");
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_pk, *d_sig;
    uint8_t* d_ok;
    const uint8_t* d_m;
    const u64* d_off;
    CPB_TRY(h.up(d_pk, pks_xy, 64 * n));
    CPB_TRY(h.up(d_sig, sigs, 64 * n));
    CPB_TRY(h.messages(d_m, d_off, msgs, msg_offsets, n));
    CPB_TRY(h.alloc(d_ok, n));
    CPB_TRY(verify_dev(c, salt_of(salt), d_pk, d_m, d_off, d_sig, d_ok, n, c->stream));
    return h.down(ok_out, d_ok, n);
    });
}

cpb_status cpb_schnorr_randomize_public_key_batch(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint8_t* randomness, size_t len,
                                                  size_t stride, uint64_t* out_xy, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!pks_xy || !out_xy || (len && !randomness)) return fail(CPB_NULL_POINTER, "null array");
    if (len > stride && n > 1) return fail(CPB_BAD_LENGTH, "randomness length %zu exceeds the stride %zu", len, stride);
    CPB_TRY(check_rand_len(len));
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_pk, *d_o;
    uint8_t* d_r;
    const size_t rbytes = n ? (n - 1) * stride + len : 0;
    CPB_TRY(h.up(d_pk, pks_xy, 64 * n));
    CPB_TRY(h.up(d_r, randomness, rbytes));
    CPB_TRY(h.alloc(d_o, 64 * n));
    CPB_TRY(cpb_schnorr_randomize_public_key_batch_dev(c, (const uint64_t*)d_pk, d_r, len, stride, (uint64_t*)d_o, n, c->stream));
    return h.down(out_xy, d_o, 64 * n);
    });
}

cpb_status cpb_schnorr_randomize_signature_batch(cpb_te_base_ctx* c, const uint64_t* sigs, const uint8_t* randomness, size_t len, size_t stride,
                                                 uint64_t* sigs_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!sigs || !sigs_out || (len && !randomness)) return fail(CPB_NULL_POINTER, "null array");
    if (len > stride && n > 1) return fail(CPB_BAD_LENGTH, "randomness length %zu exceeds the stride %zu", len, stride);
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_s, *d_o;
    uint8_t* d_r;
    const size_t rbytes = n ? (n - 1) * stride + len : 0;
    CPB_TRY(h.up(d_s, sigs, 64 * n));
    CPB_TRY(h.up(d_r, randomness, rbytes));
    CPB_TRY(h.alloc(d_o, 64 * n));
    CPB_TRY(cpb_schnorr_randomize_signature_batch_dev(c, (const uint64_t*)d_s, d_r, len, stride, (uint64_t*)d_o, n, c->stream));
    return h.down(sigs_out, d_o, 64 * n);
    });
}

cpb_status cpb_elgamal_encrypt_batch(cpb_te_base_ctx* c, const uint64_t* pks_xy, const uint64_t* msgs_xy, const uint64_t* rands,
                                     uint64_t* ciphertexts_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!pks_xy || !msgs_xy || !rands || !ciphertexts_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_pk, *d_m, *d_r, *d_o;
    CPB_TRY(h.up(d_pk, pks_xy, 64 * n));
    CPB_TRY(h.up(d_m, msgs_xy, 64 * n));
    CPB_TRY(h.up(d_r, rands, 32 * n));
    CPB_TRY(h.alloc(d_o, 128 * n));
    CPB_TRY(encrypt_dev(c, d_pk, d_m, d_r, d_o, n, c->stream));
    return h.down(ciphertexts_out, d_o, 128 * n);
    });
}

cpb_status cpb_elgamal_decrypt_batch(cpb_te_base_ctx* c, const uint64_t* sks, const uint64_t* ciphertexts, uint64_t* msgs_out, size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!sks || !ciphertexts || !msgs_out) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(ctx_check(c));
    std::lock_guard<std::mutex> lk(c->mu);
    DeviceGuard g(c->device);
    HostCall h(c->stream);
    u32 *d_sk, *d_ct, *d_o;
    CPB_TRY(h.up(d_sk, sks, 32 * n));
    CPB_TRY(h.up(d_ct, ciphertexts, 128 * n));
    CPB_TRY(h.alloc(d_o, 64 * n));
    CPB_TRY(cpb_elgamal_decrypt_batch_dev(c, (const uint64_t*)d_sk, (const uint64_t*)d_ct, (uint64_t*)d_o, n, c->stream));
    return h.down(msgs_out, d_o, 64 * n);
    });
}

cpb_status cpb_blake2s_commit_batch(int device, const uint8_t* in, const uint64_t* offsets, const uint8_t* randomness32, uint8_t* out32,
                                    size_t n) {
    return cpb::guarded([&]() -> cpb_status {
    CPB_TRY(check_n(n));
    if (n == 0) return CPB_OK;
    if (!offsets || !randomness32 || !out32) return fail(CPB_NULL_POINTER, "null array");
    CPB_TRY(check_offsets(offsets, n));
    if (!in && offsets[n] != offsets[0]) return fail(CPB_NULL_POINTER, "null input");
    DeviceGuard g(device);
    if (!g.ok) { cudaGetLastError(); return fail(CPB_NO_DEVICE, "cudaSetDevice(%d) failed: no usable CUDA device", device); }
    CPB_TRY(check_device_arch(device));
    cudaStream_t st = nullptr;
    CPB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cpb_status r;
    {
        HostCall h(st);
        const uint8_t* d_in;
        const u64* d_off;
        uint8_t *d_r, *d_o;
        r = h.messages(d_in, d_off, in, offsets, n);
        if (r == CPB_OK) r = h.up(d_r, randomness32, 32 * n);
        if (r == CPB_OK) r = h.alloc(d_o, 32 * n);
        if (r == CPB_OK) r = cpb_blake2s_commit_batch_dev(device, d_in, (const uint64_t*)d_off, d_r, d_o, n, st);
        if (r == CPB_OK) r = h.down(out32, d_o, 32 * n);
    }
    cudaStreamDestroy(st);
    return r;
    });
}

}  // extern "C"
