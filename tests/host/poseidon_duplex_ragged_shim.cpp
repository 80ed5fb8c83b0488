// CPU build of the ragged duplex's host/device-shared code (crypto_primitives_b200/csrc/poseidon_duplex.cuh: duplex_ragged_step,
// duplex_ragged_key and the per-sponge body pos_duplex_ragged on the product's own schedule; PTX primitives emulated) for
// tests/test_poseidon_duplex_ragged_host.py.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon_duplex.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
#include <vector>
using namespace cpb;

static unsigned char g_base[1 << 16];   // stands for the data buffers: the step's pointers are reported as offsets from it

// Sponge i's step of a ragged call of kind `kind` over modes (n x 2 words) and offsets (n + 1).  out: valid, noop, first, start,
// boundaries, count, squeezing', index', perms, key, span length, data offset (elements, or bytes for kAbsorbBytes, from vbase).
extern "C" void host_duplex_ragged_step(int kind, const uint64_t* modes, const uint64_t* offsets, long i, long n, uint64_t vbase, long rate,
                                        long* out) {
    const DuplexRagged R{kind, const_cast<u64*>(modes), offsets, vbase, (const u32*)g_base, g_base, (u32*)g_base, n};
    const DuplexStep s = duplex_ragged_step(R, i, rate);
    const RaggedSpan sp = ragged_span(offsets, i, n);
    const unsigned char* p = kind == kAbsorb ? (const unsigned char*)s.op.in : kind == kAbsorbBytes ? s.op.bytes : (const unsigned char*)s.op.out;
    const long unit = kind == kAbsorbBytes ? 1 : 32;
    long v[12] = {s.valid, s.noop, s.op.first, s.op.start, s.op.boundaries, s.op.count, s.mode.squeezing, s.mode.index, s.perms,
                  duplex_ragged_key(R, i, rate), sp.len, (long)(p - g_base) / unit};
    memcpy(out, v, sizeof v);
}

static PoseidonDev to_dev(const host::PoseidonSchedule& S) {
    PoseidonDev D;
    D.t = S.t; D.rate = S.rate; D.cap = S.capacity; D.rf = S.rf; D.rp = S.rp; D.sparse = S.sparse; D.alpha = S.alpha;
    D.off_c = S.off_c; D.off_m = S.off_m; D.off_mpre = S.off_mpre; D.off_cp0 = S.off_cp0; D.off_pc = S.off_pc;
    D.off_sp = S.off_sp; D.off_arkp = S.off_arkp; D.off_mod = S.off_mod; D.off_sc0 = S.off_sc0; D.n_elems = S.n_elems; D.zero = 0;
    return D;
}

template <class F, int T>
static void run(u32* states, const DuplexRagged& R, const unsigned* order, const PoseidonDev& D, const u32* cs) {
    u32 pm[8];
    ld_elem(pm, cs + 8 * D.off_mod);
    for (long j = 0; j < R.n; j++) pos_duplex_ragged<F, T>(states, R, order[j], D, cs, pm);
}
template <class F> static int run_t(u32* states, const DuplexRagged& R, const unsigned* order, const PoseidonDev& D, const u32* cs) {
    switch (D.t) {
        case 2: run<F, 2>(states, R, order, D, cs); return 0;
        case 3: run<F, 3>(states, R, order, D, cs); return 0;
        case 4: run<F, 4>(states, R, order, D, cs); return 0;
        case 5: run<F, 5>(states, R, order, D, cs); return 0;
    }
    return 1;
}

// One ragged call as the library makes it: the order (order_kind 0: input order; 1: the counting sort by duplex_ragged_key, as
// k_ragged_hist / k_ragged_scan / k_ragged_scatter produce it up to the order inside a bucket; 2: reversed), then pos_duplex_ragged for
// every sponge in that order (what k_poseidon_duplex_ragged runs per thread).  data: the elements, the bytes or the output.
// order_out (n) receives the order.  Returns -1 on a bad field or width, else the schedule's sparse flag.
extern "C" int host_duplex_ragged_run(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                      const uint64_t* mds, uint64_t* states, uint64_t* modes, long n, int kind, void* data,
                                      const uint64_t* offsets, uint64_t vbase, int order_kind, unsigned* order_out) {
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
    const DuplexRagged R{kind, modes, offsets, vbase, (const u32*)data, (const unsigned char*)data, (u32*)data, n};
    if (order_kind == 1) {
        unsigned hist[kRaggedBuckets] = {}, starts[kRaggedBuckets + 1];
        for (long i = 0; i < n; i++) hist[duplex_ragged_key(R, i, rate)]++;
        ragged_scan(hist, starts);
        for (long i = 0; i < n; i++) order_out[starts[duplex_ragged_key(R, i, rate)]++] = (unsigned)i;
    } else {
        for (long j = 0; j < n; j++) order_out[j] = (unsigned)(order_kind == 2 ? n - 1 - j : j);
    }
    u32* st = reinterpret_cast<u32*>(states);
    int rc = 1;
    switch (field) {
        case 0: rc = run_t<Bls12_381_Fr>(st, R, order_out, D, cs); break;
        case 1: rc = run_t<Bn254_Fr>(st, R, order_out, D, cs); break;
        case 2: rc = run_t<Jubjub_Fr>(st, R, order_out, D, cs); break;
        case 3: rc = run_t<Bls12_377_Fr>(st, R, order_out, D, cs); break;
    }
    return rc ? -1 : S.sparse;
}
