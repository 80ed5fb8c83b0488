// CPU build of the batched duplex's host/device-shared code (crypto_primitives_b200/csrc/poseidon_duplex.cuh: duplex_plan,
// duplex_mode_valid, the [u8] chunk encoding and the per-sponge body pos_duplex on the product's own schedule; PTX primitives
// emulated) for tests/test_poseidon_duplex_host.py.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon_duplex.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
using namespace cpb;

// out: noop, permute_first, start, boundaries, squeezing', index'
extern "C" void host_duplex_plan(int squeeze, int squeezing, long index, long rate, long count, long* out) {
    const DuplexPlan p = duplex_plan(squeeze != 0, DuplexMode{squeezing, index}, rate, count);
    out[0] = p.noop;
    out[1] = p.permute_first;
    out[2] = p.start;
    out[3] = p.boundaries;
    out[4] = p.mode.squeezing;
    out[5] = p.mode.index;
}

extern "C" int host_duplex_mode_valid(int squeezing, unsigned long long index, long rate) { return duplex_mode_valid(squeezing, index, rate); }

extern "C" long host_duplex_byte_elems(long len) { return duplex_byte_elems(len); }

// Chunk j of the encoding of str[0 .. len): canonical (mont == 0) or in Montgomery form of field `field`, as the kernel adds it.
template <class F> static void to_mont(u32* x) {
    u32 pm[8], r2[8];
    fp_modulus<F>(pm);
    for (int k = 0; k < 8; k++) r2[k] = F::R2(k);
    fp_mul<F>(x, x, r2, pm);
}
extern "C" int host_duplex_byte_chunk(const unsigned char* str, long len, long j, int mont, int field, u32* out) {
    duplex_byte_chunk(out, str, len, j);
    if (!mont) return 0;
    switch (field) {
        case 0: to_mont<Bls12_381_Fr>(out); return 0;
        case 1: to_mont<Bn254_Fr>(out); return 0;
        case 2: to_mont<Jubjub_Fr>(out); return 0;
        case 3: to_mont<Bls12_377_Fr>(out); return 0;
    }
    return -1;
}

static PoseidonDev to_dev(const host::PoseidonSchedule& S) {
    PoseidonDev D;
    D.t = S.t; D.rate = S.rate; D.cap = S.capacity; D.rf = S.rf; D.rp = S.rp; D.sparse = S.sparse; D.alpha = S.alpha;
    D.off_c = S.off_c; D.off_m = S.off_m; D.off_mpre = S.off_mpre; D.off_cp0 = S.off_cp0; D.off_pc = S.off_pc;
    D.off_sp = S.off_sp; D.off_arkp = S.off_arkp; D.off_mod = S.off_mod; D.off_sc0 = S.off_sc0; D.n_elems = S.n_elems; D.zero = 0;
    return D;
}

template <class F, int T> static void run(u32* states, const DuplexOp& op, long n, const PoseidonDev& D, const u32* cs) {
    u32 pm[8];
    ld_elem(pm, cs + 8 * D.off_mod);
    for (long i = 0; i < n; i++) pos_duplex<F, T>(states + 8 * T * i, op, i, D, cs, pm);
}
template <class F> static int run_t(u32* states, const DuplexOp& op, long n, const PoseidonDev& D, const u32* cs) {
    switch (D.t) {
        case 2: run<F, 2>(states, op, n, D, cs); return 0;
        case 3: run<F, 3>(states, op, n, D, cs); return 0;
        case 4: run<F, 4>(states, op, n, D, cs); return 0;
        case 5: run<F, 5>(states, op, n, D, cs); return 0;
    }
    return 1;
}

// One batch call as the library makes it: duplex_plan on the mode, then pos_duplex for every sponge (what k_poseidon_duplex runs per
// thread).  kind: DuplexKind; count: k or m (ignored for kAbsorbBytes: duplex_byte_elems(len)).  Montgomery limbs; t = 2..5.
// Returns -1 on a bad field or width, else the schedule's sparse flag.
extern "C" int host_duplex_run(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                               const uint64_t* mds, uint64_t* states, long n, int kind, long count, const uint64_t* in,
                               const unsigned char* bytes, long len, long stride, uint64_t* out, int* squeezing, long* index) {
    const uint64_t* mod = host::field_modulus(field);
    if (!mod || cap < 1) return -1;
    host::Field F(mod);
    host::PoseidonParams P;
    P.rate = rate; P.capacity = cap; P.full_rounds = rf; P.partial_rounds = rp; P.alpha = alpha;
    const int t = rate + cap;
    P.ark.resize((size_t)(rf + rp) * t);
    P.mds.resize((size_t)t * t);
    memcpy(P.ark.data(), ark, P.ark.size() * 32);
    memcpy(P.mds.data(), mds, P.mds.size() * 32);
    const host::PoseidonSchedule S = host::derive_schedule(F, P);
    const PoseidonDev D = to_dev(S);
    const u32* cs = reinterpret_cast<const u32*>(S.consts.data());
    if (kind == kAbsorbBytes) count = duplex_byte_elems(len);
    const DuplexPlan p = duplex_plan(kind >= kSqueeze, DuplexMode{*squeezing, *index}, rate, count);
    if (!p.noop) {
        const DuplexOp op{kind, p.permute_first ? 1 : 0, p.start, p.boundaries, count, reinterpret_cast<const u32*>(in), bytes, len,
                          stride, reinterpret_cast<u32*>(out)};
        u32* st = reinterpret_cast<u32*>(states);
        int rc = 1;
        switch (field) {
            case 0: rc = run_t<Bls12_381_Fr>(st, op, n, D, cs); break;
            case 1: rc = run_t<Bn254_Fr>(st, op, n, D, cs); break;
            case 2: rc = run_t<Jubjub_Fr>(st, op, n, D, cs); break;
            case 3: rc = run_t<Bls12_377_Fr>(st, op, n, D, cs); break;
        }
        if (rc) return -1;
    }
    *squeezing = p.mode.squeezing;
    *index = p.mode.index;
    return S.sparse;
}
