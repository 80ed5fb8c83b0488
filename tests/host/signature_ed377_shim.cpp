// CPU build of the device code behind signatures over ed-on-BLS12-377 (crypto_primitives_b200/csrc/fp.cuh, te_ops.cuh,
// PTX primitives emulated) for tests/test_signature_ed377_host.py: the arithmetic of the scalar-field tag Ed_On_Bls12_377_Fr,
// and the curve operations over the base field BLS12-377 Fr (a = -1, d = 3021) with from_random_bytes at 251 bits.
// Not part of the product.
#include "../../crypto_primitives_b200/csrc/curve_desc.hpp"
#include "../../crypto_primitives_b200/csrc/te_ops.cuh"

#include <cstring>
using namespace cpb;

typedef Bls12_377_Fr Fq;
typedef Ed_On_Bls12_377_Fr Fr;

namespace {
struct Consts {
    u32 pm[8], d2[8], sm[8];
    Consts() {
        host::CurveDesc cd;
        host::curve_desc(1, cd);                         // CPB_ED_ON_BLS12_377
        host::Field F(host::field_modulus(cd.field_id));
        host::Fe d = cd.d(F);
        host::Fe d2 = F.add(d, d);
        memcpy(pm, F.p, 32);
        memcpy(this->d2, d2.l, 32);
        memcpy(sm, cd.order(), 32);
    }
};
const Consts& K() {
    static Consts c;
    return c;
}
void load(TePoint& p, const uint64_t* xy) {
    u32 x[8], y[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    te_from_affine<Fq>(p, x, y, K().pm);
}
void store(uint64_t* xy, const TePoint& p) {
    u32 x[8], y[8];
    te_to_affine<Fq>(x, y, p, K().pm);
    memcpy(xy, x, 32);
    memcpy(xy + 4, y, 32);
}
}  // namespace

// scalar-field arithmetic, n items: 0 mul, 1 add, 2 sub, 3 sqr, 4 inv, 5 to_canonical (operands: 8 LE words each)
extern "C" void host_fr_op(int which, const u32* a, const u32* b, u32* r, long n) {
    u32 pm[8];
    fp_modulus<Fr>(pm);
    for (long i = 0; i < n; i++) {
        u32 x[8], y[8], z[8];
        memcpy(x, a + 8 * i, 32);
        memcpy(y, b + 8 * i, 32);
        switch (which) {
            case 0: fp_mul<Fr>(z, x, y, pm); break;
            case 1: fp_add<Fr>(z, x, y); break;
            case 2: fp_sub<Fr>(z, x, y); break;
            case 3: fp_sqr<Fr>(z, x, pm); break;
            case 4: fp_inv<Fr>(z, x, pm); break;
            case 5: fp_to_canonical<Fr>(z, x, pm); break;
            default: memset(z, 0, 32);
        }
        memcpy(r + 8 * i, z, 32);
    }
}

// the tag's constants, for the test to recompute: P, ONE, R2 (8 words each), NINV, BITS
extern "C" void host_fr_consts(u32* p, u32* one, u32* r2, u32* ninv, int* bits) {
    for (int i = 0; i < 8; i++) {
        p[i] = Fr::P(i);
        one[i] = Fr::ONE(i);
        r2[i] = Fr::R2(i);
    }
    *ninv = Fr::NINV;
    *bits = Fr::BITS;
}

extern "C" void host_compress(const uint64_t* xy, uint8_t* out) {
    u32 x[8], y[8], o[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    te_compress<Fq>(o, x, y, K().pm);
    memcpy(out, o, 32);
}

extern "C" int host_from_random_bytes(const uint8_t* digest, uint64_t* mont) {
    u32 d[8], m[8];
    memcpy(d, digest, 32);
    fp_zero(m);
    const bool ok = fr_from_random_bytes<Fr>(m, d, K().sm);
    memcpy(mont, m, 32);
    return ok ? 1 : 0;
}

extern "C" void host_dbl(const uint64_t* xy, uint64_t* out) {
    TePoint p;
    load(p, xy);
    te_dbl<Fq>(p, K().pm);
    store(out, p);
}

extern "C" void host_add(const uint64_t* a, const uint64_t* b, uint64_t* out) {
    TePoint p, q;
    load(p, a);
    load(q, b);
    te_add<Fq>(p, q, K().d2, K().pm);
    store(out, p);
}

extern "C" void host_neg(const uint64_t* a, uint64_t* out) {
    TePoint p;
    load(p, a);
    te_neg<Fq>(p);
    store(out, p);
}

// scalar: 8 LE words (canonical integer), `nibbles` of them used
extern "C" void host_mul_words(const uint64_t* xy, const uint64_t* scalar, int nibbles, uint64_t* out) {
    u32 x[8], y[8], w[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    memcpy(w, scalar, 32);
    TePoint acc;
    te_mul_var<Fq>(acc, x, y, ScalarWords{w, nibbles}, K().d2, K().pm);
    store(out, acc);
}

extern "C" void host_mul_bitrev_bytes(const uint64_t* xy, const uint8_t* bytes, uint64_t len, uint64_t* out) {
    u32 x[8], y[8];
    memcpy(x, xy, 32);
    memcpy(y, xy + 4, 32);
    TePoint acc;
    te_mul_var<Fq>(acc, x, y, ScalarBitrevBytes{bytes, len}, K().d2, K().pm);
    store(out, acc);
}
