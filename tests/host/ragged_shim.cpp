// CPU build of the ragged-batch device code (crypto_primitives_b200/csrc/poseidon.cuh: ragged_span, ragged_key, ragged_scan,
// ragged_ranges; PTX primitives emulated) for tests/test_ragged_host.py.  host_ragged_order is the device's counting sort done
// sequentially with the same helpers; host_ragged_sponge_any_width then hashes slot by slot as k_poseidon_crh_ragged does (the
// one-permutation range through pos_hash_single, the rest through pos_sponge).  Not part of the product.
#include "../../crypto_primitives_b200/csrc/poseidon.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
#include <cstring>
#include <vector>
using namespace cpb;

extern "C" int host_ragged_buckets() { return kRaggedBuckets; }

extern "C" long host_ragged_span(const uint64_t* offsets, long i, long n, uint64_t* lo) {
    const RaggedSpan s = ragged_span(offsets, i, n);
    *lo = s.lo;
    return s.len;
}

extern "C" int host_ragged_key(long len, int rate) { return ragged_key(len, rate); }

// order[n], starts[kRaggedBuckets + 1], range[4] as the device's histogram / scan / scatter leave them (scatter in input order).
extern "C" void host_ragged_order(const uint64_t* offsets, long n, int rate, int single, unsigned* order, unsigned* starts, unsigned* range) {
    unsigned hist[kRaggedBuckets] = {};
    for (long i = 0; i < n; i++) hist[ragged_key(ragged_span(offsets, i, n).len, rate)]++;
    ragged_scan(hist, starts);
    ragged_ranges(starts, single != 0, range);
    unsigned cursor[kRaggedBuckets];
    for (int b = 0; b < kRaggedBuckets; b++) cursor[b] = starts[b];
    for (long i = 0; i < n; i++) order[cursor[ragged_key(ragged_span(offsets, i, n).len, rate)]++] = (unsigned)i;
}

static PoseidonDev to_dev(const host::PoseidonSchedule& S) {
    PoseidonDev D;
    D.t = S.t; D.rate = S.rate; D.cap = S.capacity; D.rf = S.rf; D.rp = S.rp; D.sparse = S.sparse; D.alpha = S.alpha;
    D.off_c = S.off_c; D.off_m = S.off_m; D.off_mpre = S.off_mpre; D.off_cp0 = S.off_cp0; D.off_pc = S.off_pc;
    D.off_sp = S.off_sp; D.off_arkp = S.off_arkp; D.off_mod = S.off_mod; D.off_sc0 = S.off_sc0; D.n_elems = S.n_elems; D.zero = 0;
    return D;
}

template <class F, int T>
static void run(const PoseidonDev& D, const u32* cs, const u32* values, u64 vbase, const uint64_t* offsets, long n, long n_out, u32* out) {
    u32 pm[8];
    ld_elem(pm, cs + 8 * D.off_mod);
    const bool single = n_out <= D.rate && D.cap >= 1;
    std::vector<unsigned> order(n), starts(kRaggedBuckets + 1), range(4);
    host_ragged_order(offsets, n, D.rate, single, order.data(), starts.data(), range.data());
    for (int launch = 0; launch < 2; launch++)
        for (long j = range[2 * launch]; j < (long)range[2 * launch + 1]; j++) {
            const long i = order[j];
            const RaggedSpan sp = ragged_span(offsets, i, n);
            const u32* in = values + 8 * (sp.lo - vbase);
            if (launch == 0) pos_hash_single<F, T>(out + 8 * n_out * i, (int)n_out, in, (int)sp.len, D, cs, pm);
            else pos_sponge<F, T>(out + 8 * n_out * i, n_out, in, sp.len, D, cs, pm);
        }
}

template <class F>
static int run_t(const PoseidonDev& D, const u32* cs, const u32* v, u64 vb, const uint64_t* off, long n, long n_out, u32* out) {
    switch (D.t) {
        case 2: run<F, 2>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 3: run<F, 3>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 4: run<F, 4>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 5: run<F, 5>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 6: run<F, 6>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 7: run<F, 7>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 8: run<F, 8>(D, cs, v, vb, off, n, n_out, out); return 0;
        case 9: run<F, 9>(D, cs, v, vb, off, n, n_out, out); return 0;
    }
    return 1;
}

// values: the elements from index vbase on (Montgomery limbs); offsets: n + 1 absolute element indices.  Returns 0, or -1 on a
// bad field / width.
extern "C" int host_ragged_sponge_any_width(int field, int rate, int cap, int rf, int rp, unsigned long long alpha, const uint64_t* ark,
                                            const uint64_t* mds, const uint64_t* values, uint64_t vbase, const uint64_t* offsets, long n,
                                            long n_out, uint64_t* out) {
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
    const u32* v32 = reinterpret_cast<const u32*>(values);
    u32* o32 = reinterpret_cast<u32*>(out);
    int rc = 1;
    switch (field) {
        case 0: rc = run_t<Bls12_381_Fr>(D, cs, v32, vbase, offsets, n, n_out, o32); break;
        case 1: rc = run_t<Bn254_Fr>(D, cs, v32, vbase, offsets, n, n_out, o32); break;
        case 2: rc = run_t<Jubjub_Fr>(D, cs, v32, vbase, offsets, n, n_out, o32); break;
        case 3: rc = run_t<Bls12_377_Fr>(D, cs, v32, vbase, offsets, n, n_out, o32); break;
    }
    return rc ? -1 : 0;
}
