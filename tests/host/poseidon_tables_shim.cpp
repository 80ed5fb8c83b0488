// CPU build of the digit-table path of the device Poseidon code (fp_dot_tab in crypto_primitives_b200/csrc/fp.cuh,
// pos_permute_split in poseidon.cuh, PTX primitives emulated) on the product's own schedule and tables (poseidon_host.hpp), for
// tests/test_poseidon_digit_tables.py.  Not part of the product.
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

static host::PoseidonSchedule make_schedule(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                            const uint64_t* mds, int allow_sparse) {
    host::Field F(host::field_modulus(field));
    host::PoseidonParams P;
    P.rate = rate; P.capacity = cap; P.full_rounds = rf; P.partial_rounds = rp; P.alpha = alpha;
    const int t = rate + cap;
    P.ark.resize((size_t)(rf + rp) * t);
    P.mds.resize((size_t)t * t);
    memcpy(P.ark.data(), ark, P.ark.size() * 32);
    memcpy(P.mds.data(), mds, P.mds.size() * 32);
    return host::derive_schedule(F, P, allow_sparse != 0);
}

// The schedule's digit tables (4 x u64 per element) when out has room for them; returns their element count, -1 on a bad field.
extern "C" long host_poseidon_digit_tables(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                           const uint64_t* mds, uint64_t* out, long max_elems) {
    if (!host::field_modulus(field)) return -1;
    const host::PoseidonSchedule S = make_schedule(field, rate, cap, rf, rp, alpha, ark, mds, 1);
    const long n = (long)(S.tabs.size() / 4);
    if (out && n <= max_elems) memcpy(out, S.tabs.data(), S.tabs.size() * 8);
    return n;
}

// One CRH evaluation per input, as k_poseidon_crh<F, T, SINGLE = true> runs it (len <= rate, capacity >= 1), or the general
// sponge (one permutation per block) when `sponge`.
template <class F, int T>
static void run(const PoseidonDev& D, const u32* cs, const u32* in, long len, long n, int sponge, u32* out) {
    u32 pm[8];
    ld_elem(pm, cs + 8 * D.off_mod);
    for (long i = 0; i < n; i++) {
        if (sponge) pos_sponge<F, T>(out + 8 * i, 1, in + 8 * len * i, len, D, cs, pm);
        else pos_hash_single<F, T>(out + 8 * i, 1, in + 8 * len * i, (int)len, D, cs, pm);
    }
}
template <class F> static int run_t(const PoseidonDev& D, const u32* cs, const u32* in, long len, long n, int sponge, u32* out) {
    switch (D.t) {
        case 2: run<F, 2>(D, cs, in, len, n, sponge, out); return 0;
        case 3: run<F, 3>(D, cs, in, len, n, sponge, out); return 0;
        case 4: run<F, 4>(D, cs, in, len, n, sponge, out); return 0;
        case 5: run<F, 5>(D, cs, in, len, n, sponge, out); return 0;
        case 6: run<F, 6>(D, cs, in, len, n, sponge, out); return 0;
        case 7: run<F, 7>(D, cs, in, len, n, sponge, out); return 0;
        case 8: run<F, 8>(D, cs, in, len, n, sponge, out); return 0;
        case 9: run<F, 9>(D, cs, in, len, n, sponge, out); return 0;
    }
    return 1;
}

// Montgomery limbs in and out.  Returns -1 on a bad field, width or length, -2 when a sparse schedule has no tables, else the
// schedule's sparse flag.
extern "C" int host_poseidon_crh_tables(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                        const uint64_t* mds, int allow_sparse, const uint64_t* in, long len, long n, int sponge,
                                        uint64_t* out) {
    if (!host::field_modulus(field) || cap < 1 || (!sponge && len > rate)) return -1;
    const host::PoseidonSchedule S = make_schedule(field, rate, cap, rf, rp, alpha, ark, mds, allow_sparse);
    const PoseidonDev D = to_dev(S);
    if (S.sparse && !D.tab) return -2;
    const u32* cs = reinterpret_cast<const u32*>(S.consts.data());
    const u32* i32 = reinterpret_cast<const u32*>(in);
    u32* o32 = reinterpret_cast<u32*>(out);
    int rc = 1;
    switch (field) {
        case 0: rc = run_t<Bls12_381_Fr>(D, cs, i32, len, n, sponge, o32); break;
        case 1: rc = run_t<Bn254_Fr>(D, cs, i32, len, n, sponge, o32); break;
        case 2: rc = run_t<Jubjub_Fr>(D, cs, i32, len, n, sponge, o32); break;
        case 3: rc = run_t<Bls12_377_Fr>(D, cs, i32, len, n, sponge, o32); break;
    }
    return rc ? -1 : S.sparse;
}

// fp_dot_tab at full width: r[i] = sum_j a[i][j] * c[i][j] / R (+ y[i]) mod p for T = nt terms (1..3), U = unit (0/1).  a: any
// 256-bit values (8 x u32 each), c: Montgomery constants < p, y < p.  Tables built by the schedule's own push_digit_table.
template <class F, int T, int U> static void dot_tab_n(const uint64_t* mod, const u32* a, const uint64_t* c, const u32* y, long n, u32* r) {
    host::Field HF(mod);
    u32 pm[8];
    fp_modulus<F>(pm);
    for (long i = 0; i < n; i++) {
        std::vector<u64> tab;
        for (int j = 0; j < T; j++) {
            host::Fe e;
            memcpy(e.l, c + 4 * (T * i + j), 32);
            host::push_digit_table(HF, e, tab);
        }
        fp_dot_tab<F, T, U>(r + 8 * i, reinterpret_cast<const u32(*)[8]>(a + 8 * T * i), reinterpret_cast<const u32*>(tab.data()), pm,
                            y + 8 * i);
    }
}
template <class F> static int dot_tab_f(int nt, int unit, const uint64_t* mod, const u32* a, const uint64_t* c, const u32* y, long n, u32* r) {
    const int key = 2 * nt + unit;
    switch (key) {
        case 2: dot_tab_n<F, 1, 0>(mod, a, c, y, n, r); return 0;
        case 3: dot_tab_n<F, 1, 1>(mod, a, c, y, n, r); return 0;
        case 4: dot_tab_n<F, 2, 0>(mod, a, c, y, n, r); return 0;
        case 5: dot_tab_n<F, 2, 1>(mod, a, c, y, n, r); return 0;
        case 6: dot_tab_n<F, 3, 0>(mod, a, c, y, n, r); return 0;
        case 7: dot_tab_n<F, 3, 1>(mod, a, c, y, n, r); return 0;
    }
    return -1;
}
extern "C" int host_dot_tab(int field, int nt, int unit, const uint32_t* a, const uint64_t* c, const uint32_t* y, long n, uint32_t* r) {
    const uint64_t* mod = host::field_modulus(field);
    if (!mod) return -1;
    switch (field) {
        case 0: return dot_tab_f<Bls12_381_Fr>(nt, unit, mod, a, c, y, n, r);
        case 1: return dot_tab_f<Bn254_Fr>(nt, unit, mod, a, c, y, n, r);
        case 2: return dot_tab_f<Jubjub_Fr>(nt, unit, mod, a, c, y, n, r);
        case 3: return dot_tab_f<Bls12_377_Fr>(nt, unit, mod, a, c, y, n, r);
    }
    return -1;
}
