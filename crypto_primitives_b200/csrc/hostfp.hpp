// hostfp.hpp -- host-side 256-bit prime field with a run-time modulus.
//
// Used ONLY for one-off, per-context set-up work that the reference also does on the host:
// Poseidon parameter generation (R/sponge/poseidon/traits.rs:105-146), derivation of the
// device round schedule (sparse partial rounds), Montgomery conversion of integer constants,
// curve-parameter checks.  It is never on the batched evaluation path: every hash is computed
// by the CUDA kernels, and the library has no CPU fallback.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

namespace cpb {
namespace host {

typedef unsigned __int128 u128;
typedef uint64_t u64;

struct Fe {
    u64 l[4];
    bool operator==(const Fe& o) const { return !memcmp(l, o.l, 32); }
    bool operator!=(const Fe& o) const { return !(*this == o); }
    bool is_zero() const { return (l[0] | l[1] | l[2] | l[3]) == 0; }
};

class Field {
public:
    u64 p[4];
    u64 ninv;
    Fe one_, r2_;
    int bits;

    explicit Field(const u64 mod[4]) {
        memcpy(p, mod, 32);
        u64 inv = 1;
        for (int i = 0; i < 6; i++) inv *= 2 - p[0] * inv;
        ninv = 0 - inv;
        bits = 0;
        for (int i = 255; i >= 0; i--)
            if ((p[i / 64] >> (i % 64)) & 1) { bits = i + 1; break; }
        Fe x{{1, 0, 0, 0}};
        for (int i = 0; i < 512; i++) {
            x = add_raw(x, x);
            if (i == 255) one_ = x;
        }
        r2_ = x;
    }

    static bool geq(const u64 a[4], const u64 b[4]) {
        for (int i = 3; i >= 0; i--) {
            if (a[i] > b[i]) return true;
            if (a[i] < b[i]) return false;
        }
        return true;
    }
    bool is_canonical(const Fe& a) const { return !geq(a.l, p); }

    Fe zero() const { return Fe{{0, 0, 0, 0}}; }
    Fe one() const { return one_; }

    Fe add(const Fe& a, const Fe& b) const { return add_raw(a, b); }
    Fe sub(const Fe& a, const Fe& b) const {
        Fe r;
        u64 borrow = 0;
        for (int i = 0; i < 4; i++) {
            u128 d = (u128)a.l[i] - b.l[i] - borrow;
            r.l[i] = (u64)d;
            borrow = (u64)(d >> 64) & 1;
        }
        if (borrow) {
            u64 c = 0;
            for (int i = 0; i < 4; i++) {
                u128 s = (u128)r.l[i] + p[i] + c;
                r.l[i] = (u64)s;
                c = (u64)(s >> 64);
            }
        }
        return r;
    }
    Fe neg(const Fe& a) const { return sub(zero(), a); }

    // Montgomery product
    Fe mul(const Fe& a, const Fe& b) const {
        u64 t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 4; i++) {
            u64 c = 0;
            for (int j = 0; j < 4; j++) {
                u128 s = (u128)a.l[j] * b.l[i] + t[j] + c;
                t[j] = (u64)s;
                c = (u64)(s >> 64);
            }
            u128 s = (u128)t[4] + c;
            t[4] = (u64)s;
            t[5] = (u64)(s >> 64);
            u64 m = t[0] * ninv;
            s = (u128)m * p[0] + t[0];
            c = (u64)(s >> 64);
            for (int j = 1; j < 4; j++) {
                s = (u128)m * p[j] + t[j] + c;
                t[j - 1] = (u64)s;
                c = (u64)(s >> 64);
            }
            s = (u128)t[4] + c;
            t[3] = (u64)s;
            t[4] = t[5] + (u64)(s >> 64);
        }
        Fe r;
        memcpy(r.l, t, 32);
        if (t[4] || geq(r.l, p)) sub_p(r);
        return r;
    }

    Fe inv(const Fe& a) const {   // a^(p-2)
        u64 e[4];
        memcpy(e, p, 32);
        u64 borrow = 2;
        for (int i = 0; i < 4 && borrow; i++) {
            u64 old = e[i];
            e[i] -= borrow;
            borrow = old < borrow ? 1 : 0;
        }
        Fe acc = one_, base = a;
        for (int i = 0; i < 256; i++) {
            if ((e[i / 64] >> (i % 64)) & 1) acc = mul(acc, base);
            base = mul(base, base);
        }
        return acc;
    }

    // canonical little-endian integer (< 2^256, reduced mod p here) -> Montgomery
    Fe from_canonical(const u64 v[4]) const {
        Fe a;
        memcpy(a.l, v, 32);
        while (geq(a.l, p)) sub_p(a);
        return mul(a, r2_);
    }
    Fe from_u64(u64 v) const {
        u64 x[4] = {v, 0, 0, 0};
        return from_canonical(x);
    }
    void to_canonical(const Fe& a, u64 out[4]) const {
        Fe o{{1, 0, 0, 0}};
        Fe r = mul(a, o);
        memcpy(out, r.l, 32);
    }

private:
    void sub_p(Fe& a) const {
        u64 borrow = 0;
        for (int i = 0; i < 4; i++) {
            u128 d = (u128)a.l[i] - p[i] - borrow;
            a.l[i] = (u64)d;
            borrow = (u64)(d >> 64) & 1;
        }
    }
    Fe add_raw(const Fe& a, const Fe& b) const {
        Fe r;
        u64 c = 0;
        for (int i = 0; i < 4; i++) {
            u128 s = (u128)a.l[i] + b.l[i] + c;
            r.l[i] = (u64)s;
            c = (u64)(s >> 64);
        }
        if (c || geq(r.l, p)) sub_p(r);
        return r;
    }
};

// Every field with device arithmetic, indexed by the C-ABI field id (include/cpb200.h).  The field-level entry points
// (modulus, Montgomery conversion, element serialisation) accept all of them.
inline const u64* element_field_modulus(int field_id) {
    static const u64 M[5][4] = {
        {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull},  // BLS12-381 Fr
        {0x43e1f593f0000001ull, 0x2833e84879b97091ull, 0xb85045b68181585dull, 0x30644e72e131a029ull},  // BN254 Fr
        {0xd0970e5ed6f72cb7ull, 0xa6682093ccc81082ull, 0x06673b0101343b00ull, 0x0e7db4ea6533afa9ull},  // Jubjub Fr
        {0x0a11800000000001ull, 0x59aa76fed0000001ull, 0x60b44d1e5c37b001ull, 0x12ab655e9a2ca556ull},  // BLS12-377 Fr
        {0xb95aee9ac33fd9ffull, 0x5293a3afc43c8afeull, 0x982d1347970dec00ull, 0x04aad957a68b2955ull},  // ed-on-BLS12-377 Fr
    };
    if (field_id < 0 || field_id > 4) return nullptr;
    return M[field_id];
}

// The hash fields (ids 0..3): the fields of Poseidon parameters, contexts and Merkle digests.  Every entry point that
// builds or reads hashes validates its field id here, so the scalar field of ed-on-BLS12-377 stays unknown to them.
inline const u64* field_modulus(int field_id) { return field_id <= 3 ? element_field_modulus(field_id) : nullptr; }

typedef std::vector<Fe> FeVec;

}  // namespace host
}  // namespace cpb
