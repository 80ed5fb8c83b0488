// repro_verify_forms.cu -- two forms of the Schnorr verification kernel (csrc/cpb_signature.cu: k_schnorr_verify) on one item
// with known intermediates:
//   form A: the challenge converted out of place (ec) while the Montgomery e stays live for the final comparison;
//   form B: the challenge converted in place and reloaded for the comparison (the library's form).
// Each form runs as compiled for the library and once more storing its intermediates next to the oracle's values.
// Item: Jubjub generator of Schnorr.setup(SplitMix64(7)), sk = 5, k = 7, message "Hi"; expected values from the oracle.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 tools/repro_verify_forms.cu -o repro && ./repro
#include <cstdio>
#include <cstring>

#include "../crypto_primitives_b200/csrc/blake2s.cuh"
#include "../crypto_primitives_b200/csrc/hostfp.hpp"
#include "../crypto_primitives_b200/csrc/te_ops.cuh"

using namespace cpb;
typedef Bls12_381_Fr JqF;
typedef Jubjub_Fr JrF;

static const uint32_t PKX[8] = {0x7332de39u, 0x26f034a6u, 0x4b5225a5u, 0xd3368dd1u, 0x386fe531u, 0xe7da2e69u, 0x3b0f2adeu, 0x630971b9u};
static const uint32_t PKY[8] = {0x5deac8bfu, 0x52cb8e37u, 0x53973161u, 0xe580dc3cu, 0x5bcde519u, 0xa500d385u, 0xfef5bdc8u, 0x7220fea3u};
static const uint32_t SGX[8] = {0xdbb1565au, 0x80bef5b2u, 0xabc8cfd9u, 0x80c8a3deu, 0x1c5f1e92u, 0x8a95cfb7u, 0x874f41adu, 0xf427f0eu};
static const uint32_t SGY[8] = {0xbb28987eu, 0xff0253f9u, 0x34bb2ca2u, 0xa09ad506u, 0x7a589084u, 0x8934521u, 0x98abc3a2u, 0x66ed9d0du};
static const uint32_t EMONT[8] = {0xb99f212bu, 0x8153cf3bu, 0x3e53f859u, 0x9a034303u, 0xaa774948u, 0x74c48bffu, 0x39c95ad7u, 0xbfb0aa0u};
static const uint32_t ECAN[8] = {0xdac764dcu, 0x8997036bu, 0xc91dde79u, 0x21951f91u, 0x93c252d0u, 0x4aaabb6eu, 0xd7eb78d9u, 0xa5f3361u};
static const uint32_t EPKX[8] = {0x1c079a84u, 0x3add9966u, 0x15b5da94u, 0x41c5dda2u, 0x2c244f06u, 0xd37ddb26u, 0x41416592u, 0x2ab8359bu};
static const uint32_t EPKY[8] = {0x4a6af739u, 0x1ddf4111u, 0xda8c83c8u, 0x595e062au, 0x11d44ca6u, 0x5c0dc30au, 0x12bd956u, 0x3273113u};
static const uint32_t RPX[8] = {0x39853d1fu, 0xd80692f7u, 0x42637639u, 0x86f7d3f5u, 0x20d766cbu, 0xcd691f16u, 0x196594d1u, 0x4a0e1b27u};
static const uint32_t RPY[8] = {0x595001f2u, 0xf3d8445cu, 0xde93a3f9u, 0xcfc3113cu, 0x6ba6410u, 0xa0f26af9u, 0x89c2c22eu, 0x6b0c54fau};
static const uint8_t SALT[32] = {215, 13, 50, 89, 228, 225, 203, 99, 28, 102, 60, 244, 215, 60, 76, 4,
                                 2, 42, 177, 186, 128, 64, 152, 230, 203, 41, 62, 103, 112, 235, 58, 149};

constexpr int kSigBlock = 128;
struct Salt {
    u32 w[8];
};
struct SigConsts {
    u32 pm[8], d2[8], sm[8];
};
__device__ __forceinline__ void ld_consts(SigConsts& c, const u32* consts, int zero) {
    const u32* ct = consts + (int)threadIdx.x * zero;
    ld_elem(c.pm, ct);
    ld_elem(c.d2, ct + 8);
    ld_elem(c.sm, ct + 16);
}
__device__ __forceinline__ void msg_range(const u64* off, long i, u64& start, u64& len) {
    const u64 a = off[i], b = off[i + 1];
    start = a;
    len = b > a ? b - a : 0;
}
__device__ __forceinline__ void affine_add(TePoint& acc, const u32* x, const u32* y, const SigConsts& c) {
    u32 yp[8], ym[8], t2d[8];
    te_niels<JqF>(yp, ym, t2d, x, y, c.d2, c.pm);
    te_madd<JqF>(acc, yp, ym, t2d, c.pm);
}
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
// dbg (DBG only, canonical values): [0..8) e canonical, [8..24) e*pk, [24..40) R', [40..48) e2 (Montgomery)
__device__ void dbg_point(u32* o, const TePoint& acc, const u32* pm) {
    u32 x[8], y[8];
    te_to_affine<JqF>(x, y, acc, pm);
    fp_to_canonical<JqF>(x, x, pm);
    fp_to_canonical<JqF>(y, y, pm);
    st_elem(o, x);
    st_elem(o + 8, y);
}

// FORM_A = the first form of k_schnorr_verify, verbatim; otherwise the library's form, verbatim.
template <bool FORM_A, bool DBG>
__global__ void __launch_bounds__(kSigBlock)
k_verify(const u32* __restrict__ consts, Salt salt, const u32* __restrict__ sg_xy, const u32* __restrict__ pks,
         const uint8_t* __restrict__ msgs, const u64* __restrict__ off, const u32* __restrict__ sigs, uint8_t* __restrict__ ok_out,
         long n, int zero, u32* dbg) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SigConsts c;
    ld_consts(c, consts, zero);
    if (FORM_A) {
        u32 e[8], ec[8], px[8], py[8], x[8], y[8];
        ld_elem(e, sigs + 16 * i + 8);
        ld_elem(px, pks + 16 * i);
        ld_elem(py, pks + 16 * i + 8);
        fp_to_canonical<JrF>(ec, e, c.sm);
        if (DBG) st_elem(dbg, ec);
        TePoint acc;
        te_mul_var<JqF>(acc, px, py, ScalarWords{ec, 63}, c.d2, c.pm);
        if (DBG) dbg_point(dbg + 8, acc, c.pm);
        ld_elem(x, sg_xy + 16 * i);
        ld_elem(y, sg_xy + 16 * i + 8);
        affine_add(acc, x, y, c);
        te_to_affine<JqF>(x, y, acc, c.pm);
        if (DBG) dbg_point(dbg + 24, acc, c.pm);
        u64 start, len;
        msg_range(off, i, start, len);
        u32 e2[8];
        const bool valid = schnorr_challenge(e2, salt, x, y, msgs + start, len, c);
        if (DBG) st_elem(dbg + 40, e2);
        ok_out[i] = valid && fp_eq(e, e2) ? 1 : 0;
    } else {
        u32 e[8], x[8], y[8];
        ld_elem(e, sigs + 16 * i + 8);
        fp_to_canonical<JrF>(e, e, c.sm);
        if (DBG) st_elem(dbg, e);
        ld_elem(x, pks + 16 * i);
        ld_elem(y, pks + 16 * i + 8);
        TePoint acc;
        te_mul_var<JqF>(acc, x, y, ScalarWords{e, 63}, c.d2, c.pm);
        if (DBG) dbg_point(dbg + 8, acc, c.pm);
        ld_elem(x, sg_xy + 16 * i);
        ld_elem(y, sg_xy + 16 * i + 8);
        affine_add(acc, x, y, c);
        te_to_affine<JqF>(x, y, acc, c.pm);
        if (DBG) dbg_point(dbg + 24, acc, c.pm);
        u64 start, len;
        msg_range(off, i, start, len);
        u32 e2[8];
        const bool valid = schnorr_challenge(e2, salt, x, y, msgs + start, len, c);
        if (DBG) st_elem(dbg + 40, e2);
        ld_elem(e, sigs + 16 * i + 8);
        ok_out[i] = valid && fp_eq(e, e2) ? 1 : 0;
    }
}

static void show(const char* what, const u32* got, const u32* exp) {
    bool ok = !memcmp(got, exp, 32);
    printf("  %-10s %s", what, ok ? "ok  " : "DIFF");
    for (int i = 7; i >= 0; i--) printf(" %08x", got[i]);
    printf("\n");
}

int main() {
    host::Field F(host::field_modulus(0));
    host::Fe d = F.neg(F.mul(F.from_u64(10240), F.inv(F.from_u64(10241))));
    host::Fe d2 = F.add(d, d);
    u32 consts[24], sg[16], pk[16], sig[16] = {};
    memcpy(consts, F.p, 32);
    memcpy(consts + 8, d2.l, 32);
    memcpy(consts + 16, host::field_modulus(2), 32);
    memcpy(pk, PKX, 32);
    memcpy(pk + 8, PKY, 32);
    memcpy(sg, SGX, 32);
    memcpy(sg + 8, SGY, 32);
    memcpy(sig + 8, EMONT, 32);                        // s is not read: s*G is given
    u64 off[2] = {0, 2};
    Salt salt;
    memcpy(salt.w, SALT, 32);
    u32 *d_c, *d_sg, *d_pk, *d_sig, *d_dbg;
    u64* d_off;
    uint8_t *d_msg, *d_ok;
    cudaMalloc(&d_c, sizeof consts);
    cudaMalloc(&d_sg, sizeof sg);
    cudaMalloc(&d_pk, sizeof pk);
    cudaMalloc(&d_sig, sizeof sig);
    cudaMalloc(&d_off, sizeof off);
    cudaMalloc(&d_msg, 16);
    cudaMalloc(&d_ok, 4);
    cudaMalloc(&d_dbg, 4 * 48 * 4);
    cudaMemcpy(d_c, consts, sizeof consts, cudaMemcpyHostToDevice);
    cudaMemcpy(d_sg, sg, sizeof sg, cudaMemcpyHostToDevice);
    cudaMemcpy(d_pk, pk, sizeof pk, cudaMemcpyHostToDevice);
    cudaMemcpy(d_sig, sig, sizeof sig, cudaMemcpyHostToDevice);
    cudaMemcpy(d_off, off, sizeof off, cudaMemcpyHostToDevice);
    cudaMemcpy(d_msg, "Hi", 2, cudaMemcpyHostToDevice);
    cudaMemset(d_dbg, 0, 4 * 48 * 4);
    k_verify<true, false><<<1, 1>>>(d_c, salt, d_sg, d_pk, d_msg, d_off, d_sig, d_ok + 0, 1, 0, nullptr);
    k_verify<false, false><<<1, 1>>>(d_c, salt, d_sg, d_pk, d_msg, d_off, d_sig, d_ok + 1, 1, 0, nullptr);
    k_verify<true, true><<<1, 1>>>(d_c, salt, d_sg, d_pk, d_msg, d_off, d_sig, d_ok + 2, 1, 0, d_dbg);
    k_verify<false, true><<<1, 1>>>(d_c, salt, d_sg, d_pk, d_msg, d_off, d_sig, d_ok + 3, 1, 0, d_dbg + 48);
    uint8_t ok[4];
    u32 dbg[96];
    cudaError_t err = cudaMemcpy(ok, d_ok, 4, cudaMemcpyDeviceToHost);
    if (err == cudaSuccess) err = cudaMemcpy(dbg, d_dbg, sizeof dbg, cudaMemcpyDeviceToHost);
    if (err != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(err)); return 1; }
    printf("verdicts (expected 1): form A %u, form B %u, form A instrumented %u, form B instrumented %u\n", ok[0], ok[1], ok[2], ok[3]);
    for (int f = 0; f < 2; f++) {
        const u32* o = dbg + 48 * f;
        printf("form %c (instrumented)\n", f ? 'B' : 'A');
        show("e canon", o, ECAN);
        show("e*pk x", o + 8, EPKX);
        show("e*pk y", o + 16, EPKY);
        show("R' x", o + 24, RPX);
        show("R' y", o + 32, RPY);
        show("e2", o + 40, EMONT);
    }
    return 0;
}
