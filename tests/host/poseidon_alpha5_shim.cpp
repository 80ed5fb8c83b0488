// CPU build of the compile-time alpha = 5 path of the device Poseidon code (pos_hash_single<F, T, A5 = true> and pos_sbox5 in
// crypto_primitives_b200/csrc/poseidon.cuh, PTX primitives emulated) on the product's own schedule and digit tables
// (poseidon_host.hpp), for tests/test_poseidon_bn254_alu.py.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
using namespace cpb;

static PoseidonDev to_dev(const host::PoseidonSchedule& S) {
    PoseidonDev D;
    D.t = S.t; D.rate = S.rate; D.cap = S.capacity; D.rf = S.rf; D.rp = S.rp; D.sparse = S.sparse; D.alpha = S.alpha;
    D.off_c = S.off_c; D.off_m = S.off_m; D.off_mpre = S.off_mpre; D.off_cp0 = S.off_cp0; D.off_pc = S.off_pc;
    D.off_sp = S.off_sp; D.off_arkp = S.off_arkp; D.off_mod = S.off_mod; D.off_sc0 = S.off_sc0; D.n_elems = S.n_elems; D.zero = 0;
    D.tab = S.tabs.empty() ? nullptr : reinterpret_cast<const u32*>(S.tabs.data());
    return D;
}

// One CRH evaluation per input (len <= rate, capacity >= 1), as k_poseidon_crh<F, T, SINGLE = true, A5 = true> runs it.
template <class F, int T> static void run(const PoseidonDev& D, const u32* cs, const u32* in, long len, long n, u32* out) {
    u32 pm[8];
    ld_elem(pm, cs + 8 * D.off_mod);
    for (long i = 0; i < n; i++) pos_hash_single<F, T, true>(out + 8 * i, 1, in + 8 * len * i, (int)len, D, cs, pm);
}
template <class F> static int run_t(const PoseidonDev& D, const u32* cs, const u32* in, long len, long n, u32* out) {
    switch (D.t) {
        case 2: run<F, 2>(D, cs, in, len, n, out); return 0;
        case 3: run<F, 3>(D, cs, in, len, n, out); return 0;
        case 4: run<F, 4>(D, cs, in, len, n, out); return 0;
        case 5: run<F, 5>(D, cs, in, len, n, out); return 0;
        case 6: run<F, 6>(D, cs, in, len, n, out); return 0;
        case 7: run<F, 7>(D, cs, in, len, n, out); return 0;
        case 8: run<F, 8>(D, cs, in, len, n, out); return 0;
        case 9: run<F, 9>(D, cs, in, len, n, out); return 0;
    }
    return 1;
}

// Montgomery limbs in and out; the config's alpha must be 5.  Returns -1 on a bad field, width, length or exponent, else the
// schedule's sparse flag.
extern "C" int host_poseidon_crh_alpha5(int field, int rate, int cap, int rf, int rp, const uint64_t* ark, const uint64_t* mds,
                                        int allow_sparse, const uint64_t* in, long len, long n, uint64_t* out) {
    if (!host::field_modulus(field) || cap < 1 || len > rate) return -1;
    host::Field HF(host::field_modulus(field));
    host::PoseidonParams P;
    P.rate = rate; P.capacity = cap; P.full_rounds = rf; P.partial_rounds = rp; P.alpha = 5;
    const int t = rate + cap;
    P.ark.resize((size_t)(rf + rp) * t);
    P.mds.resize((size_t)t * t);
    memcpy(P.ark.data(), ark, P.ark.size() * 32);
    memcpy(P.mds.data(), mds, P.mds.size() * 32);
    const host::PoseidonSchedule S = host::derive_schedule(HF, P, allow_sparse != 0);
    const PoseidonDev D = to_dev(S);
    const u32* cs = reinterpret_cast<const u32*>(S.consts.data());
    const u32* i32 = reinterpret_cast<const u32*>(in);
    u32* o32 = reinterpret_cast<u32*>(out);
    int rc = 1;
    switch (field) {
        case 0: rc = run_t<Bls12_381_Fr>(D, cs, i32, len, n, o32); break;
        case 1: rc = run_t<Bn254_Fr>(D, cs, i32, len, n, o32); break;
        case 2: rc = run_t<Jubjub_Fr>(D, cs, i32, len, n, o32); break;
        case 3: rc = run_t<Bls12_377_Fr>(D, cs, i32, len, n, o32); break;
    }
    return rc ? -1 : S.sparse;
}

// The partial-round S-box of the BN254 hash kernel on given operands: x^5 / R^4 (Montgomery) with the lazy products, for x < 2p.
extern "C" void host_bn254_sbox5_lazy(const uint32_t* x, long n, uint32_t* out) {
    u32 pm[8];
    fp_modulus<Bn254_Fr>(pm);
    for (long i = 0; i < n; i++) {
        u32 v[8];
        memcpy(v, x + 8 * i, 32);
        pos_sbox5<Bn254_Fr, true>(v, pm);
        memcpy(out + 8 * i, v, 32);
    }
}
