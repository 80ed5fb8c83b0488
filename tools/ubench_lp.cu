// ubench_lp.cu -- limb-parallel (8 lanes per element, csrc/fp_lp.cuh) against one-thread-per-element (csrc/fp.cuh) field
// arithmetic: (1) bit-exactness of lp_mul / lp_add / lp_sub against fp_mul / fp_add / fp_sub on pattern-limb operands (limbs
// drawn from {0, 1, 2^32-1, 2^31, 2^32-2, random}: every carry path is hit constantly), (2) latency of a dependent chain of
// multiplications for a lone warp -- what bounds the small levels of a tree.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I crypto_primitives_b200/csrc -o tools/ubench_lp tools/ubench_lp.cu
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "fp.cuh"
#include "fp_lp.cuh"
using namespace cpb;

// ---- host: -p^-1 mod 2^256 by Newton iteration on 8 x 32-bit limbs
static void mul_lo256(const u32* a, const u32* b, u32* r) {
    u64 acc[9] = {0};
    u32 out[8];
    for (int i = 0; i < 8; i++) {
        u64 lo = 0, hi = 0;        // column i as 128-bit sum
        unsigned __int128 s = 0;
        for (int k = 0; k <= i; k++) s += (unsigned __int128)a[k] * b[i - k];
        s += acc[i];
        out[i] = (u32)s;
        unsigned __int128 c = s >> 32;
        if (i + 1 < 9) acc[i + 1] += (u64)c;     // fits: sums of < 8 products >> 32 plus carry
        (void)lo; (void)hi;
    }
    memcpy(r, out, 32);
}
static void neg_inv256(const u32* p, u32* ninv) {
    u32 x[8] = {1, 0, 0, 0, 0, 0, 0, 0};
    for (int it = 0; it < 9; it++) {
        u32 px[8], t[8];
        mul_lo256(p, x, px);                         // p*x
        // t = 2 - px
        u64 borrow = 0;
        for (int i = 0; i < 8; i++) {
            u64 d = (u64)(i == 0 ? 2u : 0u) - px[i] - borrow;
            t[i] = (u32)d;
            borrow = (d >> 63) & 1;
        }
        mul_lo256(x, t, x);
    }
    u64 borrow = 0;
    for (int i = 0; i < 8; i++) {
        u64 d = (u64)0 - x[i] - borrow;
        ninv[i] = (u32)d;
        borrow = (d >> 63) & 1;
    }
}
static bool ge256(const u32* a, const u32* b) {
    for (int i = 7; i >= 0; i--) { if (a[i] > b[i]) return true; if (a[i] < b[i]) return false; }
    return true;
}
static void sub256(u32* a, const u32* b) {
    u64 borrow = 0;
    for (int i = 0; i < 8; i++) { u64 d = (u64)a[i] - b[i] - borrow; a[i] = (u32)d; borrow = (d >> 63) & 1; }
}

template <class F> __global__ void k_ref(const u32* a, const u32* b, u32* mul, u32* add, u32* sub, long n) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 x[8], y[8], r[8], pm[8];
    fp_modulus<F>(pm);
    ld_elem(x, a + 8 * i); ld_elem(y, b + 8 * i);
    fp_mul<F>(r, x, y, pm); st_elem(mul + 8 * i, r);
    fp_add<F>(r, x, y); st_elem(add + 8 * i, r);
    fp_sub<F>(r, x, y); st_elem(sub + 8 * i, r);
}
__global__ void k_lp(const u32* a, const u32* b, const u32* pl, const u32* nl, u32* mul, u32* add, u32* sub, long n) {
    const long e = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;       // element index; n is a multiple of 4 per warp
    const int lane = threadIdx.x & 31;
    LpLane C;
    C.g = lane & 7; C.sh = 8 * (lane >> 3); C.p = pl[C.g]; C.ninv = nl[C.g];
    const long ee = e < n ? e : n - 1;
    const u32 x = a[8 * ee + C.g], y = b[8 * ee + C.g];
    const u32 m = lp_mul(x, y, C), s = lp_add(x, y, C), d = lp_sub(x, y, C);
    if (e < n) { mul[8 * e + C.g] = m; add[8 * e + C.g] = s; sub[8 * e + C.g] = d; }
}
template <class F> __global__ void k_chain_ref(u32* out, int iters, long long* cyc) {
    u32 x[8], y[8], pm[8];
    fp_modulus<F>(pm);
    for (int i = 0; i < 8; i++) { x[i] = F::R2(i) ^ threadIdx.x; y[i] = F::ONE(i) + threadIdx.x; }
    x[7] &= 0x0fffffffu; y[7] &= 0x0fffffffu;
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; i++) fp_mul<F>(x, x, y, pm);
    long long t1 = clock64();
    st_elem(out + 8 * threadIdx.x, x);
    if (threadIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_chain_lp(const u32* pl, const u32* nl, u32* out, int iters, long long* cyc) {
    const int lane = threadIdx.x & 31;
    LpLane C;
    C.g = lane & 7; C.sh = 8 * (lane >> 3); C.p = pl[C.g]; C.ninv = nl[C.g];
    u32 x = 0x1234567u * (lane + 1), y = 0x7654321u * (lane + 3);
    if (C.g == 7) { x &= 0x0fffffffu; y &= 0x0fffffffu; }
    long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; i++) x = lp_mul(x, y, C);
    long long t1 = clock64();
    out[threadIdx.x] = x;
    if (threadIdx.x == 0) *cyc = t1 - t0;
}

template <class F> int run(const char* name, int n_elems) {
    u32 p[8], ninv[8];
    for (int i = 0; i < 8; i++) p[i] = F::P(i);
    neg_inv256(p, ninv);
    {   // check: p * (-ninv) == 1 mod 2^256  <=>  p*ninv == -1
        u32 t[8]; mul_lo256(p, ninv, t);
        for (int i = 0; i < 8; i++) if (t[i] != 0xffffffffu) { printf("%s: ninv wrong\n", name); return 1; }
    }
    std::vector<u32> a(8 * (size_t)n_elems), b(8 * (size_t)n_elems);
    const u32 pat[6] = {0u, 1u, 0xffffffffu, 0x80000000u, 0xfffffffeu, 0x7fffffffu};
    srand(12345);
    auto gen = [&](u32* e) {
        for (int i = 0; i < 8; i++) { int c = rand() % 9; e[i] = c < 6 ? pat[c] : ((u32)rand() << 16) ^ (u32)rand() ^ ((u32)rand() << 31); }
        while (ge256(e, p)) sub256(e, p);
    };
    for (int i = 0; i < n_elems; i++) { gen(&a[8 * i]); gen(&b[8 * i]); }
    for (int i = 0; i < 8; i++) { a[i] = p[i]; b[i] = p[i]; }                 // (p-1) * (p-1)
    a[0] -= 1; b[0] -= 1;
    u32 *da, *db, *dp, *dn, *r[6];
    cudaMalloc(&da, a.size() * 4); cudaMalloc(&db, b.size() * 4); cudaMalloc(&dp, 32); cudaMalloc(&dn, 32);
    for (auto& q : r) cudaMalloc(&q, a.size() * 4);
    cudaMemcpy(da, a.data(), a.size() * 4, cudaMemcpyHostToDevice); cudaMemcpy(db, b.data(), b.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dp, p, 32, cudaMemcpyHostToDevice); cudaMemcpy(dn, ninv, 32, cudaMemcpyHostToDevice);
    k_ref<F><<<(n_elems + 127) / 128, 128>>>(da, db, r[0], r[1], r[2], n_elems);
    k_lp<<<(n_elems * 8 + 127) / 128, 128>>>(da, db, dp, dn, r[3], r[4], r[5], n_elems);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); return 1; }
    std::vector<u32> h[6];
    for (int i = 0; i < 6; i++) { h[i].resize(a.size()); cudaMemcpy(h[i].data(), r[i], a.size() * 4, cudaMemcpyDeviceToHost); }
    long bad[3] = {0, 0, 0};
    for (int op = 0; op < 3; op++)
        for (int i = 0; i < n_elems; i++)
            if (memcmp(&h[op][8 * i], &h[op + 3][8 * i], 32)) {
                if (bad[op]++ < 2) {
                    printf("%s op %d elem %d differs\n  a ", name, op, i);
                    for (int k = 7; k >= 0; k--) printf("%08x", a[8 * i + k]);
                    printf("\n  b ");
                    for (int k = 7; k >= 0; k--) printf("%08x", b[8 * i + k]);
                    printf("\n  ref ");
                    for (int k = 7; k >= 0; k--) printf("%08x", h[op][8 * i + k]);
                    printf("\n  lp  ");
                    for (int k = 7; k >= 0; k--) printf("%08x", h[op + 3][8 * i + k]);
                    printf("\n");
                }
            }
    printf("%s: %d pattern-limb operand pairs: mul mismatches %ld, add %ld, sub %ld\n", name, n_elems, bad[0], bad[1], bad[2]);
    long long *dc, hc;
    cudaMalloc(&dc, 8);
    const int iters = 2000;
    for (int rep = 0; rep < 2; rep++) k_chain_ref<F><<<1, 32>>>(r[0], iters, dc);
    cudaMemcpy(&hc, dc, 8, cudaMemcpyDeviceToHost);
    printf("%s: one thread per element, lone warp: %.1f cycles per dependent fp_mul\n", name, (double)hc / iters);
    for (int rep = 0; rep < 2; rep++) k_chain_lp<<<1, 32>>>(dp, dn, r[0], iters, dc);
    cudaMemcpy(&hc, dc, 8, cudaMemcpyDeviceToHost);
    printf("%s: 8 lanes per element, lone warp:    %.1f cycles per dependent lp_mul\n", name, (double)hc / iters);
    return (bad[0] || bad[1] || bad[2]) ? 1 : 0;
}

int main() {
    int rc = 0;
    rc |= run<Bn254_Fr>("bn254", 1 << 20);
    rc |= run<Bls12_381_Fr>("bls12_381", 1 << 20);
    rc |= run<Jubjub_Fr>("jubjub_fr", 1 << 18);
    rc |= run<Bls12_377_Fr>("bls12_377", 1 << 18);
    printf(rc ? "FAILED\n" : "lp self-test ok\n");
    return rc;
}
