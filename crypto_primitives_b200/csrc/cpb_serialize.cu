// cpb_serialize.cu -- wire formats behind the C-ABI (include/cpb200.h, "wire formats"): the `CanonicalSerialize` /
// `CanonicalDeserialize` images of the types that cross the boundary -- PoseidonConfig (R/sponge/poseidon/mod.rs:25-45),
// pedersen::Parameters (R/crh/pedersen/mod.rs:28-31), merkle_tree::Path and MultiPath (R/merkle_tree/mod.rs:139-152,
// 239-254) -- so that a non-Rust host and an arkworks process can exchange parameters and proofs as bytes.
// HOST code only (one-off conversions, nothing batched, no GPU): compiled with the library for one build recipe.
//
// The derive macros write the struct fields in declaration order; the leaf encodings are ark-serialize / ark-ff / ark-ec 0.4
// conventions (dependencies, absent from /root/reference), restated from their published behaviour -- NOT pinned by any
// vector the reference holds:
//   usize, u64        8 bytes little-endian
//   Vec<T>            u64 length, then the elements
//   Fp (n bits)       ceil(n/8) bytes little-endian of the canonical (non-Montgomery) value; >= p is "invalid data"
//   TE affine point   compressed: y, bit 7 of the last byte set when x > -x;  uncompressed: x then y
//                     (validated on request: on the curve and in the prime-order subgroup)
#include <cstring>
#include <memory>
#include <vector>

#include "common.cuh"
#include "curve_desc.hpp"
#include "hostfp.hpp"

using namespace cpb;
using host::Fe;
using host::Field;
typedef host::u64 hu64;

namespace {

using host::CurveDesc;
using host::curve_desc;

size_t fbytes(const Field& F) { return (size_t)(F.bits + 7) / 8; }

void put_u64(std::vector<uint8_t>& o, hu64 v) {
    for (int i = 0; i < 8; i++) o.push_back((uint8_t)(v >> (8 * i)));
}
void put_field(const Field& F, std::vector<uint8_t>& o, const hu64* mont) {
    Fe a;
    memcpy(a.l, mont, 32);
    hu64 c[4];
    F.to_canonical(a, c);
    uint8_t b[32];
    memcpy(b, c, 32);                                   // little-endian host
    o.insert(o.end(), b, b + fbytes(F));
}

struct Reader {
    const uint8_t* p;
    size_t len, pos = 0;
    bool ok = true;
    const uint8_t* take(size_t n) {
        if (!ok || pos + n > len) { ok = false; return nullptr; }
        const uint8_t* r = p + pos;
        pos += n;
        return r;
    }
    hu64 u64() {
        const uint8_t* b = take(8);
        hu64 v = 0;
        if (b) for (int i = 0; i < 8; i++) v |= (hu64)b[i] << (8 * i);
        return v;
    }
};
// 0 ok, 1 eof, 2 invalid data
int get_field(const Field& F, Reader& r, hu64* mont_out, uint8_t clear_top_mask = 0, uint8_t* top_out = nullptr) {
    const uint8_t* b = r.take(fbytes(F));
    if (!b) return 1;
    uint8_t buf[32] = {0};
    memcpy(buf, b, fbytes(F));
    if (top_out) *top_out = buf[fbytes(F) - 1];
    buf[fbytes(F) - 1] &= (uint8_t)~clear_top_mask;
    hu64 c[4];
    memcpy(c, buf, 32);
    if (Field::geq(c, F.p)) return 2;
    Fe m = F.from_canonical(c);
    memcpy(mont_out, m.l, 32);
    return 0;
}

// ---- field helpers for point decompression
Fe fpow(const Field& F, const Fe& a, const hu64 e[4]) {
    Fe acc = F.one(), base = a;
    for (int i = 0; i < 256; i++) {
        if ((e[i / 64] >> (i % 64)) & 1) acc = F.mul(acc, base);
        base = F.mul(base, base);
    }
    return acc;
}
bool fsqrt(const Field& F, const Fe& n, Fe& out) {       // Tonelli-Shanks
    if (n.is_zero()) { out = n; return true; }
    hu64 e[4], t[4];
    memcpy(e, F.p, 32);
    e[0] -= 1;                                           // p - 1 (p odd)
    hu64 half[4];
    for (int i = 0; i < 4; i++) half[i] = (e[i] >> 1) | (i < 3 ? e[i + 1] << 63 : 0);
    if (fpow(F, n, half) != F.one()) return false;
    int s = 0;
    memcpy(t, e, 32);
    while (!(t[0] & 1)) {
        for (int i = 0; i < 4; i++) t[i] = (t[i] >> 1) | (i < 3 ? t[i + 1] << 63 : 0);
        s++;
    }
    Fe z = F.from_u64(2);
    while (fpow(F, z, half) == F.one()) z = F.add(z, F.one());
    hu64 t1[4];                                          // (t + 1) / 2
    memcpy(t1, t, 32);
    t1[0] += 1;                                          // t odd: no carry beyond bit 0
    for (int i = 0; i < 4; i++) t1[i] = (t1[i] >> 1) | (i < 3 ? t1[i + 1] << 63 : 0);
    int m = s;
    Fe c = fpow(F, z, t), tt = fpow(F, n, t), r = fpow(F, n, t1);
    while (tt != F.one()) {
        int i = 0;
        Fe x = tt;
        while (x != F.one()) { x = F.mul(x, x); i++; }
        Fe b = c;
        for (int k = 0; k < m - i - 1; k++) b = F.mul(b, b);
        m = i;
        c = F.mul(b, b);
        tt = F.mul(tt, c);
        r = F.mul(r, b);
    }
    out = r;
    return true;
}
bool canonical_greater(const Field& F, const Fe& a, const Fe& b) {     // compare canonical integers
    hu64 x[4], y[4];
    F.to_canonical(a, x);
    F.to_canonical(b, y);
    for (int i = 3; i >= 0; i--) {
        if (x[i] > y[i]) return true;
        if (x[i] < y[i]) return false;
    }
    return false;
}

struct Curve {
    Field F;
    Fe d;
    CurveDesc desc;
    explicit Curve(const CurveDesc& c) : F(host::field_modulus(c.field_id)), desc(c) {
        d = c.d(F);
    }
    bool on_curve(const Fe& x, const Fe& y) const {
        Fe xx = F.mul(x, x), yy = F.mul(y, y);
        return F.sub(yy, xx) == F.add(F.one(), F.mul(d, F.mul(xx, yy)));
    }
    // extended coordinates (X:Y:Z:T), a = -1 unified addition (complete for these curves)
    struct Pt { Fe X, Y, Z, T; };
    Pt add(const Pt& p, const Pt& q) const {
        Fe A = F.mul(F.sub(p.Y, p.X), F.sub(q.Y, q.X)), B = F.mul(F.add(p.Y, p.X), F.add(q.Y, q.X));
        Fe C = F.mul(F.mul(p.T, q.T), F.add(d, d)), D = F.mul(F.add(p.Z, p.Z), q.Z);
        Fe E = F.sub(B, A), Fv = F.sub(D, C), G = F.add(D, C), H = F.add(B, A);
        return Pt{F.mul(E, Fv), F.mul(G, H), F.mul(Fv, G), F.mul(E, H)};
    }
    bool in_subgroup(const Fe& x, const Fe& y) const {
        Pt acc{F.zero(), F.one(), F.one(), F.zero()}, base{x, y, F.one(), F.mul(x, y)};
        const hu64* order = desc.order();
        for (int i = 0; i < 256; i++) {
            if ((order[i / 64] >> (i % 64)) & 1) acc = add(acc, base);
            base = add(base, base);
        }
        return acc.X.is_zero() && acc.Y == acc.Z;        // (0 : 1 : 1)
    }
};

void put_point(const Curve& C, std::vector<uint8_t>& o, const hu64* xy, bool compress) {
    if (!compress) {
        put_field(C.F, o, xy);
        put_field(C.F, o, xy + 4);
        return;
    }
    Fe x;
    memcpy(x.l, xy, 32);
    size_t at = o.size();
    put_field(C.F, o, xy + 4);
    if (canonical_greater(C.F, x, C.F.neg(x))) o[at + fbytes(C.F) - 1] |= 0x80;
}
int get_point(const Curve& C, Reader& r, hu64* xy_out, bool compress, bool validate) {
    Fe x, y;
    if (!compress) {
        int e = get_field(C.F, r, x.l);
        if (e) return e;
        e = get_field(C.F, r, y.l);
        if (e) return e;
        if (!C.on_curve(x, y)) return 2;
    } else {
        uint8_t top = 0;
        int e = get_field(C.F, r, y.l, 0x80, &top);
        if (e) return e;
        const bool neg = (top & 0x80) != 0;
        Fe yy = C.F.mul(y, y);
        Fe den = C.F.sub(C.F.neg(C.F.one()), C.F.mul(C.d, yy));        // a - d y^2, a = -1
        if (den.is_zero()) return 2;
        Fe x2 = C.F.mul(C.F.sub(C.F.one(), yy), C.F.inv(den));
        if (!fsqrt(C.F, x2, x)) return 2;
        if (canonical_greater(C.F, x, C.F.neg(x)) != neg) x = C.F.neg(x);
    }
    if (validate && !C.in_subgroup(x, y)) return 2;
    memcpy(xy_out, x.l, 32);
    memcpy(xy_out + 4, y.l, 32);
    return 0;
}

cpb_status finish(const std::vector<uint8_t>& o, uint8_t* out, size_t cap, size_t* written) {
    if (written) *written = o.size();
    if (!out) return CPB_OK;                               // size query
    if (cap < o.size()) return fail(CPB_BAD_LENGTH, "output buffer too small: need %zu bytes", o.size());
    memcpy(out, o.data(), o.size());
    return CPB_OK;
}
cpb_status rd_error(int e) {
    return e == 1 ? fail(CPB_BAD_LENGTH, "unexpected end of input") : fail(CPB_BAD_PARAMS, "invalid data");
}

// digest codec: kind 0 = field element (id = field id), 1 = compressed point, 2 = uncompressed point (id = curve id)
struct Codec {
    int kind, words;
    const Field* F = nullptr;
    const Curve* C = nullptr;
    bool validate;
    void put(std::vector<uint8_t>& o, const hu64* d) const {
        if (kind == 0) put_field(*F, o, d);
        else put_point(*C, o, d, kind == 1);
    }
    int get(Reader& r, hu64* d) const { return kind == 0 ? get_field(*F, r, d) : get_point(*C, r, d, kind == 1, validate); }
};

}  // namespace

extern "C" {

size_t cpb_field_serialized_size(int field_id) {
    const hu64* m = host::element_field_modulus(field_id);
    if (!m) return 0;
    return fbytes(Field(m));
}

cpb_status cpb_field_serialize(int field_id, const uint64_t* mont, size_t n, uint8_t* out) {
    return cpb::guarded([&]() -> cpb_status {
    const hu64* m = host::element_field_modulus(field_id);
    if (!m) return fail(CPB_BAD_PARAMS, "unknown field id %d", field_id);
    if (n && (!mont || !out)) return fail(CPB_NULL_POINTER, "null buffer");
    Field F(m);
    std::vector<uint8_t> o;
    for (size_t i = 0; i < n; i++) put_field(F, o, mont + 4 * i);
    memcpy(out, o.data(), o.size());
    return CPB_OK;
    });
}
cpb_status cpb_field_deserialize(int field_id, const uint8_t* in, size_t n, uint64_t* mont_out) {
    return cpb::guarded([&]() -> cpb_status {
    const hu64* m = host::element_field_modulus(field_id);
    if (!m) return fail(CPB_BAD_PARAMS, "unknown field id %d", field_id);
    if (n && (!in || !mont_out)) return fail(CPB_NULL_POINTER, "null buffer");
    Field F(m);
    Reader r{in, n * fbytes(F)};
    for (size_t i = 0; i < n; i++) {
        int e = get_field(F, r, mont_out + 4 * i);
        if (e) return rd_error(e);
    }
    return CPB_OK;
    });
}
size_t cpb_point_serialized_size(int curve_id, int compress) {
    CurveDesc c;
    if (!curve_desc(curve_id, c)) return 0;
    size_t b = fbytes(Field(host::field_modulus(c.field_id)));
    return compress ? b : 2 * b;
}
cpb_status cpb_point_serialize(int curve_id, const uint64_t* xy, size_t n, int compress, uint8_t* out) {
    return cpb::guarded([&]() -> cpb_status {
    CurveDesc c;
    if (!curve_desc(curve_id, c)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", curve_id);
    if (n && (!xy || !out)) return fail(CPB_NULL_POINTER, "null buffer");
    Curve C(c);
    std::vector<uint8_t> o;
    for (size_t i = 0; i < n; i++) put_point(C, o, xy + 8 * i, compress != 0);
    memcpy(out, o.data(), o.size());
    return CPB_OK;
    });
}
cpb_status cpb_point_deserialize(int curve_id, const uint8_t* in, size_t n, int compress, int validate, uint64_t* xy_out) {
    return cpb::guarded([&]() -> cpb_status {
    CurveDesc c;
    if (!curve_desc(curve_id, c)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", curve_id);
    if (n && (!in || !xy_out)) return fail(CPB_NULL_POINTER, "null buffer");
    Curve C(c);
    Reader r{in, n * cpb_point_serialized_size(curve_id, compress)};
    for (size_t i = 0; i < n; i++) {
        int e = get_point(C, r, xy_out + 8 * i, compress != 0, validate != 0);
        if (e) return rd_error(e);
    }
    return CPB_OK;
    });
}

// PoseidonConfig { full_rounds, partial_rounds, alpha, ark: Vec<Vec<F>>, mds: Vec<Vec<F>>, rate, capacity }
cpb_status cpb_poseidon_config_serialize(int field_id, int rate, int capacity, int full_rounds, int partial_rounds, uint64_t alpha,
                                         const uint64_t* ark, const uint64_t* mds, uint8_t* out, size_t out_cap, size_t* written) {
    return cpb::guarded([&]() -> cpb_status {
    const hu64* m = host::field_modulus(field_id);
    if (!m) return fail(CPB_BAD_PARAMS, "unknown field id %d", field_id);
    if (rate < 1 || capacity < 1 || full_rounds < 0 || partial_rounds < 0) return fail(CPB_BAD_PARAMS, "bad shape");
    if (!ark || !mds) return fail(CPB_NULL_POINTER, "null ark/mds");
    Field F(m);
    const size_t t = (size_t)rate + capacity, rounds = (size_t)full_rounds + partial_rounds;
    std::vector<uint8_t> o;
    put_u64(o, (hu64)full_rounds); put_u64(o, (hu64)partial_rounds); put_u64(o, alpha);
    put_u64(o, rounds);
    for (size_t r = 0; r < rounds; r++) {
        put_u64(o, t);
        for (size_t i = 0; i < t; i++) put_field(F, o, ark + 4 * (r * t + i));
    }
    put_u64(o, t);
    for (size_t r = 0; r < t; r++) {
        put_u64(o, t);
        for (size_t i = 0; i < t; i++) put_field(F, o, mds + 4 * (r * t + i));
    }
    put_u64(o, (hu64)rate); put_u64(o, (hu64)capacity);
    return finish(o, out, out_cap, written);
    });
}
// ark_out / mds_out may be NULL for a shape query (the shape fields are written first).
cpb_status cpb_poseidon_config_deserialize(int field_id, const uint8_t* in, size_t len, int* rate, int* capacity, int* full_rounds,
                                           int* partial_rounds, uint64_t* alpha, uint64_t* ark_out, size_t ark_cap_elems,
                                           uint64_t* mds_out, size_t mds_cap_elems) {
    return cpb::guarded([&]() -> cpb_status {
    const hu64* m = host::field_modulus(field_id);
    if (!m) return fail(CPB_BAD_PARAMS, "unknown field id %d", field_id);
    if (!in) return fail(CPB_NULL_POINTER, "null input");
    Field F(m);
    Reader r{in, len};
    const hu64 rf = r.u64(), rp = r.u64(), al = r.u64(), rows = r.u64();
    if (!r.ok) return rd_error(1);
    if (rf > 4096 || rp > 4096 || rows != rf + rp) return fail(CPB_BAD_PARAMS, "invalid data: ark has %llu rows for %llu rounds", (unsigned long long)rows, (unsigned long long)(rf + rp));
    std::vector<hu64> ark, mds;
    size_t t = 0;
    for (hu64 i = 0; i < rows; i++) {
        hu64 w = r.u64();
        if (!r.ok) return rd_error(1);
        if (i == 0) t = (size_t)w;
        if (w != t || t < 2 || t > 64) return fail(CPB_BAD_PARAMS, "invalid data: ragged ark");
        for (size_t k = 0; k < t; k++) {
            hu64 e[4];
            int er = get_field(F, r, e);
            if (er) return rd_error(er);
            ark.insert(ark.end(), e, e + 4);
        }
    }
    const hu64 mrows = r.u64();
    if (!r.ok) return rd_error(1);
    if (rows == 0) t = (size_t)mrows;
    if (mrows != t) return fail(CPB_BAD_PARAMS, "invalid data: mds shape");
    for (hu64 i = 0; i < mrows; i++) {
        if (r.u64() != t || !r.ok) return r.ok ? fail(CPB_BAD_PARAMS, "invalid data: mds shape") : rd_error(1);
        for (size_t k = 0; k < t; k++) {
            hu64 e[4];
            int er = get_field(F, r, e);
            if (er) return rd_error(er);
            mds.insert(mds.end(), e, e + 4);
        }
    }
    const hu64 ra = r.u64(), ca = r.u64();
    if (!r.ok) return rd_error(1);
    if (r.pos != len) return fail(CPB_BAD_LENGTH, "trailing bytes");
    if (ra + ca != t) return fail(CPB_BAD_PARAMS, "invalid data: rate + capacity != width");
    if (rate) *rate = (int)ra;
    if (capacity) *capacity = (int)ca;
    if (full_rounds) *full_rounds = (int)rf;
    if (partial_rounds) *partial_rounds = (int)rp;
    if (alpha) *alpha = al;
    if (ark_out) {
        if (ark_cap_elems * 4 < ark.size()) return fail(CPB_BAD_LENGTH, "ark buffer too small");
        memcpy(ark_out, ark.data(), ark.size() * 8);
    }
    if (mds_out) {
        if (mds_cap_elems * 4 < mds.size()) return fail(CPB_BAD_LENGTH, "mds buffer too small");
        memcpy(mds_out, mds.data(), mds.size() * 8);
    }
    return CPB_OK;
    });
}

// crh::pedersen::Parameters { generators: Vec<Vec<C>> }
cpb_status cpb_pedersen_parameters_serialize(int curve_id, int window_size, int num_windows, const uint64_t* generators_xy, int compress,
                                             uint8_t* out, size_t out_cap, size_t* written) {
    return cpb::guarded([&]() -> cpb_status {
    CurveDesc c;
    if (!curve_desc(curve_id, c)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", curve_id);
    if (window_size < 0 || num_windows < 0) return fail(CPB_BAD_PARAMS, "bad window");
    if (!generators_xy && window_size * num_windows) return fail(CPB_NULL_POINTER, "null generators");
    Curve C(c);
    std::vector<uint8_t> o;
    put_u64(o, (hu64)num_windows);
    for (int w = 0; w < num_windows; w++) {
        put_u64(o, (hu64)window_size);
        for (int j = 0; j < window_size; j++) put_point(C, o, generators_xy + 8 * ((size_t)w * window_size + j), compress != 0);
    }
    return finish(o, out, out_cap, written);
    });
}
cpb_status cpb_pedersen_parameters_deserialize(int curve_id, const uint8_t* in, size_t len, int compress, int validate, int* window_size,
                                               int* num_windows, uint64_t* generators_xy_out, size_t cap_points) {
    return cpb::guarded([&]() -> cpb_status {
    CurveDesc c;
    if (!curve_desc(curve_id, c)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", curve_id);
    if (!in) return fail(CPB_NULL_POINTER, "null input");
    Curve C(c);
    Reader r{in, len};
    const hu64 nw = r.u64();
    if (!r.ok) return rd_error(1);
    if (nw > (1u << 20)) return fail(CPB_BAD_PARAMS, "invalid data: too many windows");
    std::vector<hu64> pts;
    hu64 ws = 0;
    for (hu64 w = 0; w < nw; w++) {
        hu64 k = r.u64();
        if (!r.ok) return rd_error(1);
        if (w == 0) ws = k;
        if (k != ws || k > (1u << 20)) return fail(CPB_BAD_PARAMS, "invalid data: ragged generator table");
        for (hu64 j = 0; j < k; j++) {
            hu64 xy[8];
            int e = get_point(C, r, xy, compress != 0, validate != 0);
            if (e) return rd_error(e);
            pts.insert(pts.end(), xy, xy + 8);
        }
    }
    if (r.pos != len) return fail(CPB_BAD_LENGTH, "trailing bytes");
    if (window_size) *window_size = (int)ws;
    if (num_windows) *num_windows = (int)nw;
    if (generators_xy_out) {
        if (cap_points * 8 < pts.size()) return fail(CPB_BAD_LENGTH, "generator buffer too small");
        memcpy(generators_xy_out, pts.data(), pts.size() * 8);
    }
    return CPB_OK;
    });
}

static cpb_status make_codec(int kind, int id, int validate, Codec& K, std::unique_ptr<Field>& F, std::unique_ptr<Curve>& C) {
    K.kind = kind; K.validate = validate != 0;
    if (kind == 0) {
        const hu64* m = host::field_modulus(id);
        if (!m) return fail(CPB_BAD_PARAMS, "unknown field id %d", id);
        F.reset(new Field(m));
        K.F = F.get(); K.words = 4;
    } else if (kind == 1 || kind == 2) {
        CurveDesc c;
        if (!curve_desc(id, c)) return fail(CPB_BAD_PARAMS, "unknown curve id %d", id);
        C.reset(new Curve(c));
        K.C = C.get(); K.words = 8;
    } else {
        return fail(CPB_BAD_PARAMS, "digest kind must be 0 (field), 1 (compressed point) or 2 (uncompressed point)");
    }
    return CPB_OK;
}

// Path { leaf_sibling_hash, auth_path: Vec<InnerDigest>, leaf_index: usize }
cpb_status cpb_path_serialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, const uint64_t* leaf_sibling_hash, const uint64_t* auth_path,
                              size_t path_len, uint64_t leaf_index, uint8_t* out, size_t out_cap, size_t* written) {
    return cpb::guarded([&]() -> cpb_status {
    Codec L, I;
    std::unique_ptr<Field> f1, f2;
    std::unique_ptr<Curve> c1, c2;
    CPB_TRY(make_codec(leaf_kind, leaf_id, 0, L, f1, c1));
    CPB_TRY(make_codec(inner_kind, inner_id, 0, I, f2, c2));
    if (!leaf_sibling_hash || (path_len && !auth_path)) return fail(CPB_NULL_POINTER, "null digest");
    std::vector<uint8_t> o;
    L.put(o, leaf_sibling_hash);
    put_u64(o, path_len);
    for (size_t i = 0; i < path_len; i++) I.put(o, auth_path + (size_t)I.words * i);
    put_u64(o, leaf_index);
    return finish(o, out, out_cap, written);
    });
}
cpb_status cpb_path_deserialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, int validate, const uint8_t* in, size_t len,
                                uint64_t* leaf_sibling_hash, uint64_t* auth_path, size_t path_cap, size_t* path_len, uint64_t* leaf_index) {
    return cpb::guarded([&]() -> cpb_status {
    Codec L, I;
    std::unique_ptr<Field> f1, f2;
    std::unique_ptr<Curve> c1, c2;
    CPB_TRY(make_codec(leaf_kind, leaf_id, validate, L, f1, c1));
    CPB_TRY(make_codec(inner_kind, inner_id, validate, I, f2, c2));
    if (!in || !leaf_sibling_hash) return fail(CPB_NULL_POINTER, "null buffer");
    Reader r{in, len};
    int e = L.get(r, leaf_sibling_hash);
    if (e) return rd_error(e);
    const hu64 n = r.u64();
    if (!r.ok) return rd_error(1);
    if (n > 64) return fail(CPB_BAD_PARAMS, "invalid data: path of %llu nodes", (unsigned long long)n);
    if (path_len) *path_len = (size_t)n;
    if (n > path_cap || (n && !auth_path)) return fail(CPB_BAD_LENGTH, "auth path buffer too small: need %llu digests", (unsigned long long)n);
    for (hu64 i = 0; i < n; i++) {
        e = I.get(r, auth_path + (size_t)I.words * i);
        if (e) return rd_error(e);
    }
    const hu64 idx = r.u64();
    if (!r.ok) return rd_error(1);
    if (r.pos != len) return fail(CPB_BAD_LENGTH, "trailing bytes");
    if (leaf_index) *leaf_index = idx;
    return CPB_OK;
    });
}

// MultiPath { leaf_siblings_hashes: Vec<LeafDigest>, auth_paths_prefix_lenghts: Vec<usize>, auth_paths_suffixes: Vec<Vec<InnerDigest>>,
//             leaf_indexes: Vec<usize> } -- flattened: n paths, suffix_lens[n], suffixes = concatenated digests
cpb_status cpb_multipath_serialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, size_t n, const uint64_t* leaf_siblings_hashes,
                                   const uint64_t* prefix_lengths, const uint64_t* suffix_lengths, const uint64_t* suffixes,
                                   const uint64_t* leaf_indexes, uint8_t* out, size_t out_cap, size_t* written) {
    return cpb::guarded([&]() -> cpb_status {
    Codec L, I;
    std::unique_ptr<Field> f1, f2;
    std::unique_ptr<Curve> c1, c2;
    CPB_TRY(make_codec(leaf_kind, leaf_id, 0, L, f1, c1));
    CPB_TRY(make_codec(inner_kind, inner_id, 0, I, f2, c2));
    if (n && (!leaf_siblings_hashes || !prefix_lengths || !suffix_lengths || !leaf_indexes)) return fail(CPB_NULL_POINTER, "null buffer");
    std::vector<uint8_t> o;
    put_u64(o, n);
    for (size_t i = 0; i < n; i++) L.put(o, leaf_siblings_hashes + (size_t)L.words * i);
    put_u64(o, n);
    for (size_t i = 0; i < n; i++) put_u64(o, prefix_lengths[i]);
    put_u64(o, n);
    size_t at = 0;
    for (size_t i = 0; i < n; i++) {
        put_u64(o, suffix_lengths[i]);
        for (hu64 k = 0; k < suffix_lengths[i]; k++, at++) I.put(o, suffixes + (size_t)I.words * at);
    }
    put_u64(o, n);
    for (size_t i = 0; i < n; i++) put_u64(o, leaf_indexes[i]);
    return finish(o, out, out_cap, written);
    });
}
// Two-pass friendly: with NULL outputs only *n_paths and *n_suffix_digests are written.
cpb_status cpb_multipath_deserialize(int leaf_kind, int leaf_id, int inner_kind, int inner_id, int validate, const uint8_t* in, size_t len,
                                     size_t* n_paths, size_t* n_suffix_digests, uint64_t* leaf_siblings_hashes, uint64_t* prefix_lengths,
                                     uint64_t* suffix_lengths, uint64_t* suffixes, uint64_t* leaf_indexes, size_t cap_paths, size_t cap_suffix_digests) {
    return cpb::guarded([&]() -> cpb_status {
    Codec L, I;
    std::unique_ptr<Field> f1, f2;
    std::unique_ptr<Curve> c1, c2;
    CPB_TRY(make_codec(leaf_kind, leaf_id, validate, L, f1, c1));
    CPB_TRY(make_codec(inner_kind, inner_id, validate, I, f2, c2));
    if (!in) return fail(CPB_NULL_POINTER, "null input");
    Reader r{in, len};
    const hu64 n = r.u64();
    if (!r.ok) return rd_error(1);
    if (n > ((hu64)1 << 32)) return fail(CPB_BAD_PARAMS, "invalid data: too many paths");
    std::vector<hu64> sib((size_t)n * L.words), pre((size_t)n), slen((size_t)n), suf, idx((size_t)n);
    for (hu64 i = 0; i < n; i++) {
        int e = L.get(r, sib.data() + (size_t)L.words * i);
        if (e) return rd_error(e);
    }
    if (r.u64() != n || !r.ok) return r.ok ? fail(CPB_BAD_PARAMS, "invalid data: vector lengths differ") : rd_error(1);
    for (hu64 i = 0; i < n; i++) pre[i] = r.u64();
    if (r.u64() != n || !r.ok) return r.ok ? fail(CPB_BAD_PARAMS, "invalid data: vector lengths differ") : rd_error(1);
    for (hu64 i = 0; i < n; i++) {
        slen[i] = r.u64();
        if (!r.ok) return rd_error(1);
        if (slen[i] > 64) return fail(CPB_BAD_PARAMS, "invalid data: suffix of %llu nodes", (unsigned long long)slen[i]);
        for (hu64 k = 0; k < slen[i]; k++) {
            hu64 d[8];
            int e = I.get(r, d);
            if (e) return rd_error(e);
            suf.insert(suf.end(), d, d + I.words);
        }
    }
    if (r.u64() != n || !r.ok) return r.ok ? fail(CPB_BAD_PARAMS, "invalid data: vector lengths differ") : rd_error(1);
    for (hu64 i = 0; i < n; i++) idx[i] = r.u64();
    if (!r.ok) return rd_error(1);
    if (r.pos != len) return fail(CPB_BAD_LENGTH, "trailing bytes");
    if (n_paths) *n_paths = (size_t)n;
    if (n_suffix_digests) *n_suffix_digests = suf.size() / I.words;
    if (!leaf_siblings_hashes) return CPB_OK;                    // size query
    if (cap_paths < n || cap_suffix_digests * I.words < suf.size()) return fail(CPB_BAD_LENGTH, "output buffers too small");
    if (!prefix_lengths || !suffix_lengths || !leaf_indexes || (suf.size() && !suffixes)) return fail(CPB_NULL_POINTER, "null buffer");
    memcpy(leaf_siblings_hashes, sib.data(), sib.size() * 8);
    memcpy(prefix_lengths, pre.data(), pre.size() * 8);
    memcpy(suffix_lengths, slen.data(), slen.size() * 8);
    if (suf.size()) memcpy(suffixes, suf.data(), suf.size() * 8);
    memcpy(leaf_indexes, idx.data(), idx.size() * 8);
    return CPB_OK;
    });
}

}  // extern "C"
