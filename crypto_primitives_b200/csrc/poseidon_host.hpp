// poseidon_host.hpp -- host-side Poseidon parameter work (once per context).
//
//  * PoseidonGrainLFSR + find_poseidon_ark_and_mds: the reference's parameter generator,
//    R/sponge/poseidon/grain_lfsr.rs:16-181 and R/sponge/poseidon/traits.rs:105-146
//    (same bit stream; state kept as an 80-entry byte ring).
//  * derive_schedule: turns a PoseidonConfig (R/sponge/poseidon/mod.rs:26-45) into the round
//    schedule the CUDA kernels execute.  The reference's permute (mod.rs:98-121) applies a
//    dense t x t MDS in all RF+RP rounds; here the RP partial rounds use the equivalent
//    sparse form (1 row + 1 column per round) with round constants folded so that only lane 0
//    receives a constant.  The rewrite is exact field algebra, so outputs are bit-identical;
//    when a required (t-1)x(t-1) minor is singular, M[0][0] = 0, or a row's w_hat[1] is zero (the
//    split loop carries lane 1 as w_hat . s and divides by it), the schedule falls back to the dense form.
#pragma once
#include "hostfp.hpp"

namespace cpb {
namespace host {

// ------------------------------------------------------------------------- Grain LFSR
class GrainLFSR {
public:
    GrainLFSR(bool sbox_inverse, u64 prime_bits, u64 state_len, u64 rf, u64 rp) : prime_bits_(prime_bits) {
        for (int i = 0; i < 80; i++) st_[i] = 0;
        st_[1] = 1;                       // b0,b1: prime field          grain_lfsr.rs:25
        st_[5] = sbox_inverse ? 1 : 0;    // b2..b5: s-box               :28-32
        put(6, 17, prime_bits);           // :35-41
        put(18, 29, state_len);           // :44-50
        put(30, 39, rf);                  // :53-59
        put(40, 49, rp);                  // :62-68
        for (int i = 50; i < 80; i++) st_[i] = 1;   // :71-73
        head_ = 0;
        for (int i = 0; i < 160; i++) update();     // :177-181
    }

    // n bits, first drawn = most significant (grain_lfsr.rs:117-121,144-156), as 4 LE words.
    void draw(u64 out[4]) {
        out[0] = out[1] = out[2] = out[3] = 0;
        for (u64 i = 0; i < prime_bits_; i++) {
            u64 bitpos = prime_bits_ - 1 - i;
            if (next_filtered_bit()) out[bitpos / 64] |= 1ull << (bitpos % 64);
        }
    }

    FeVec rejection_sampling(const Field& F, size_t n) {     // :109-134
        FeVec r;
        while (r.size() < n) {
            u64 v[4];
            draw(v);
            if (!Field::geq(v, F.p)) r.push_back(F.from_canonical(v));
        }
        return r;
    }
    FeVec mod_p(const Field& F, size_t n) {                  // :136-160
        FeVec r;
        for (size_t i = 0; i < n; i++) {
            u64 v[4];
            draw(v);
            r.push_back(F.from_canonical(v));   // reduces mod p
        }
        return r;
    }

private:
    void put(int lo, int hi, u64 v) {
        for (int i = hi; i >= lo; i--) { st_[i] = v & 1; v >>= 1; }
    }
    int update() {                                            // :162-175
        int nb = st_[(head_ + 62) % 80] ^ st_[(head_ + 51) % 80] ^ st_[(head_ + 38) % 80] ^
                 st_[(head_ + 23) % 80] ^ st_[(head_ + 13) % 80] ^ st_[head_];
        st_[head_] = (unsigned char)nb;
        head_ = (head_ + 1) % 80;
        return nb;
    }
    int next_filtered_bit() {                                 // get_bits :87-107
        int b = update();
        while (!b) { update(); b = update(); }
        return update();
    }
    unsigned char st_[80];
    int head_;
    u64 prime_bits_;
};

struct PoseidonParams {
    int rate = 0, capacity = 0, full_rounds = 0, partial_rounds = 0;
    u64 alpha = 0;
    FeVec ark;   // (RF+RP) x t, Montgomery
    FeVec mds;   // t x t row-major, Montgomery
    int t() const { return rate + capacity; }
};

// traits.rs:105-146
inline void find_poseidon_ark_and_mds(const Field& F, u64 prime_bits, int rate, int rf, int rp, int skip,
                                      FeVec& ark, FeVec& mds) {
    int t = rate + 1;
    GrainLFSR lfsr(false, prime_bits, (u64)t, (u64)rf, (u64)rp);
    ark.clear();
    for (int r = 0; r < rf + rp; r++) {
        FeVec row = lfsr.rejection_sampling(F, (size_t)t);
        ark.insert(ark.end(), row.begin(), row.end());
    }
    for (int s = 0; s < skip; s++) (void)lfsr.mod_p(F, (size_t)(2 * t));
    FeVec xs = lfsr.mod_p(F, (size_t)t), ys = lfsr.mod_p(F, (size_t)t);
    mds.assign((size_t)t * t, F.zero());
    for (int i = 0; i < t; i++)
        for (int j = 0; j < t; j++) mds[(size_t)i * t + j] = F.inv(F.add(xs[i], ys[j]));
}

// Default-parameter entry tables of the reference's BLS12-381 test field (R/sponge/test.rs:13-32):
// (rate, alpha, full, partial, skip).  Other fields carry no table in the reference.
struct DefaultEntry { int rate; u64 alpha; int rf, rp, skip; };
inline bool default_entry(int field_id, int rate, bool optimized_for_weights, DefaultEntry& e) {
    if (field_id != 0) return false;   // PoseidonDefaultConfig is implemented per field; the reference does so for its BLS12-381 Fr test field only
    static const DefaultEntry C[7] = {{2, 17, 8, 31, 0}, {3, 5, 8, 56, 0}, {4, 5, 8, 56, 0}, {5, 5, 8, 57, 0},
                                      {6, 5, 8, 57, 0},  {7, 5, 8, 57, 0}, {8, 5, 8, 57, 0}};
    if (rate < 2 || rate > 8) return false;
    if (optimized_for_weights) e = DefaultEntry{rate, 257, 8, 13, 0};
    else e = C[rate - 2];
    return true;
}

// ------------------------------------------------------------------------- device schedule
// All offsets are in field elements into `consts` (8 x u32 / 4 x u64 Montgomery limbs each).
struct PoseidonSchedule {
    int t = 0, rate = 0, capacity = 0, rf = 0, rp = 0, sparse = 0;
    u64 alpha = 0;
    int off_c = 0;     // rf x t   constants added before the s-box of full round fr (0..rf-1)
    int off_m = 0;     // t x t    MDS
    int off_mpre = 0;  // 2 x t x t: Mpre, the matrix of the last first-half full round (= D0*M; M when dense), then
                       //          Mpost, that of the first second-half full round (M with column 0 scaled; M when dense)
    int off_cp0 = 0;   // t        constant vector added before the first partial round
    int off_pc = 0;    // rp       lane-0 constant added after partial round k-1 (entry k; entry 0 unused)
    int off_sp = 0;    // rp x (2t-1): per round the row [one, w_hat[1..t-1]] then v[1..t-1]  (sparse; lane 0 scaled)
    int off_arkp = 0;  // rp x t   original partial-round constants                     (dense schedules only; empty when sparse)
    int off_mod = 0;   // 1        the modulus limbs (plain integer): the kernels load them from here into registers
    int off_sc0 = 0;   // 1        S(C[0][0]): lane 0 after the first S-box when it entered the permutation as zero (fresh sponge)
                       // then, at off_sc0 + 1 (sparse only): rp x (2t-2) per round [gamma, alpha, beta[2..t-1] | v[2..t-1]], then
                       //          Mpre's row 1 (t) and Cp0's entry 1 for lane 1 carried as w_hat . s (pos_permute_split only)
    int n_elems = 0;
    std::vector<u64> consts;
    // Digit tables of fp_dot_tab (sparse only; empty when dense), placed right after the n_elems staged elements of the device
    // buffer and read from global memory: 8 elements K_0(c) .. K_7(c) per constant c that pos_permute_split multiplies by, for
    // M, Mpre, Mpost (t x t each, row-major) and then the off_sc0 + 1 region up to (not including) Cp0's entry 1.
    std::vector<u64> tabs;
};

// The elements K_i(c) = c * 2^(32 i) * 2^64 mod p (c plain, i.e. c_mont * 2^(32 i + 64) / R) fp_dot_tab multiplies the limbs of
// its variable operand by, each stored as the 32-bit limbs 1, 3, 5, 7, 0, 2, 4, 6 (detail::ld_tab_row, fp.cuh).
inline void push_digit_table(const Field& F, const Fe& c, std::vector<u64>& out) {
    Fe z{{0, 1, 0, 0}};                                   // 2^64 < p
    for (int i = 0; i < 8; i++) {
        const Fe k = F.mul(c, z);                         // c_mont * z / R
        u64 w[4];
        for (int j = 0; j < 2; j++) {
            w[j] = (k.l[2 * j] >> 32) | (k.l[2 * j + 1] & 0xffffffff00000000ull);       // limbs 4j+1, 4j+3
            w[2 + j] = (k.l[2 * j] & 0xffffffffull) | (k.l[2 * j + 1] << 32);          // limbs 4j, 4j+2
        }
        out.insert(out.end(), w, w + 4);
        for (int b = 0; b < 32; b++) z = F.add(z, z);
    }
}

namespace detail {
inline FeVec matmul(const Field& F, const FeVec& A, const FeVec& B, int n) {
    FeVec C((size_t)n * n, F.zero());
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) {
            Fe acc = F.zero();
            for (int k = 0; k < n; k++) acc = F.add(acc, F.mul(A[(size_t)i * n + k], B[(size_t)k * n + j]));
            C[(size_t)i * n + j] = acc;
        }
    return C;
}
inline FeVec matvec(const Field& F, const FeVec& A, const FeVec& x, int n) {
    FeVec y((size_t)n, F.zero());
    for (int i = 0; i < n; i++) {
        Fe acc = F.zero();
        for (int k = 0; k < n; k++) acc = F.add(acc, F.mul(A[(size_t)i * n + k], x[k]));
        y[i] = acc;
    }
    return y;
}
// Gauss-Jordan inverse of an m x m matrix; false when singular.
inline bool invert(const Field& F, FeVec A, int m, FeVec& out) {
    FeVec I((size_t)m * m, F.zero());
    for (int i = 0; i < m; i++) I[(size_t)i * m + i] = F.one();
    for (int c = 0; c < m; c++) {
        int piv = -1;
        for (int r = c; r < m; r++)
            if (!A[(size_t)r * m + c].is_zero()) { piv = r; break; }
        if (piv < 0) return false;
        if (piv != c)
            for (int k = 0; k < m; k++) {
                std::swap(A[(size_t)piv * m + k], A[(size_t)c * m + k]);
                std::swap(I[(size_t)piv * m + k], I[(size_t)c * m + k]);
            }
        Fe inv = F.inv(A[(size_t)c * m + c]);
        for (int k = 0; k < m; k++) {
            A[(size_t)c * m + k] = F.mul(A[(size_t)c * m + k], inv);
            I[(size_t)c * m + k] = F.mul(I[(size_t)c * m + k], inv);
        }
        for (int r = 0; r < m; r++) {
            if (r == c) continue;
            Fe f = A[(size_t)r * m + c];
            if (f.is_zero()) continue;
            for (int k = 0; k < m; k++) {
                A[(size_t)r * m + k] = F.sub(A[(size_t)r * m + k], F.mul(f, A[(size_t)c * m + k]));
                I[(size_t)r * m + k] = F.sub(I[(size_t)r * m + k], F.mul(f, I[(size_t)c * m + k]));
            }
        }
    }
    out = I;
    return true;
}
}  // namespace detail

inline PoseidonSchedule derive_schedule(const Field& F, const PoseidonParams& P, bool allow_sparse = true) {
    const int t = P.t(), rf = P.full_rounds, rp = P.partial_rounds, half = rf / 2;
    PoseidonSchedule S;
    S.t = t; S.rate = P.rate; S.capacity = P.capacity; S.rf = rf; S.rp = rp; S.alpha = P.alpha;

    const FeVec& M = P.mds;
    FeVec C((size_t)rf * t), Mpre = M, Mpost = M, Cp0((size_t)t, F.zero()), pc((size_t)(rp > 0 ? rp : 1), F.zero());
    FeVec sp((size_t)(rp > 0 ? rp : 1) * (2 * t - 1), F.zero()), arkp, lp;
    auto ark = [&](int r, int i) -> const Fe& { return P.ark[(size_t)r * t + i]; };
    for (int fr = 0; fr < rf; fr++) {
        int r = fr < half ? fr : half + rp + (fr - half);
        for (int i = 0; i < t; i++) C[(size_t)fr * t + i] = ark(r, i);
    }
    for (int k = 0; k < rp; k++)
        for (int i = 0; i < t; i++) arkp.push_back(ark(half + k, i));

    // m00 = M[0][0] != 0: the lane-0 scale below divides by products of it
    bool sparse = allow_sparse && rp > 0 && t >= 2 && half >= 1 && rf > half && !M[0].is_zero();
    if (sparse) {
        // backward factorisation  N_k = D_{k+1} * M = Sp_k * D_k,  D_rp = I
        FeVec D((size_t)t * t, F.zero());
        for (int i = 0; i < t; i++) D[(size_t)i * t + i] = F.one();
        const int m = t - 1;
        for (int k = rp - 1; k >= 0 && sparse; k--) {
            FeVec N = detail::matmul(F, D, M, t);
            FeVec Mhat((size_t)m * m), Minv;
            for (int i = 0; i < m; i++)
                for (int j = 0; j < m; j++) Mhat[(size_t)i * m + j] = N[(size_t)(i + 1) * t + (j + 1)];
            if (!detail::invert(F, Mhat, m, Minv)) { sparse = false; break; }
            for (int j = 0; j < m; j++) {   // w_hat^T = w^T * Mhat^-1
                Fe acc = F.zero();
                for (int i = 0; i < m; i++) acc = F.add(acc, F.mul(N[(size_t)0 * t + (i + 1)], Minv[(size_t)i * m + j]));
                sp[(size_t)k * (2 * t - 1) + 1 + j] = acc;
            }
            if (sp[(size_t)k * (2 * t - 1) + 1].is_zero()) { sparse = false; break; }   // lane 1's basis change divides by w_hat[1]
            sp[(size_t)k * (2 * t - 1)] = N[0];   // m00 (row 0 of N equals row 0 of M)
            for (int i = 0; i < m; i++) sp[(size_t)k * (2 * t - 1) + t + i] = N[(size_t)(i + 1) * t + 0];
            for (auto& e : D) e = F.zero();
            D[0] = F.one();
            for (int i = 0; i < m; i++)
                for (int j = 0; j < m; j++) D[(size_t)(i + 1) * t + (j + 1)] = Mhat[(size_t)i * m + j];
        }
        if (sparse) {
            Mpre = detail::matmul(F, D, M, t);
            FeVec c0((size_t)t);
            for (int i = 0; i < t; i++) c0[i] = ark(half, i);
            Cp0 = detail::matvec(F, D, c0, t);
            // forward constant folding: lanes 1.. of each later partial constant move one round on
            FeVec d((size_t)t, F.zero());
            for (int k = 1; k < rp; k++) {
                FeVec md = detail::matvec(F, M, d, t);
                FeVec cp((size_t)t);
                for (int i = 0; i < t; i++) cp[i] = F.add(ark(half + k, i), md[i]);
                pc[k] = cp[0];
                d = cp;
                d[0] = F.zero();
            }
            FeVec post = detail::matvec(F, M, d, t);
            for (int i = 0; i < t; i++) C[(size_t)half * t + i] = F.add(C[(size_t)half * t + i], post[i]);
            // Lane 0 is carried as L = lane0 / lam_k through the partial rounds: lam_0 = 1, lam_{k+1} = m00 * lam_k^alpha.  As
            // S(lam*y) = lam^alpha * S(y), round k becomes L' = xi + (w_hat / lam_{k+1}) . s, s' = s + (v * lam_k^alpha) * xi with
            // xi = S(L): the row's lane-0 coefficient is exactly one, which the kernels add instead of multiplying.  The constant
            // entering lane 0 at round k is divided by lam_k; the first second-half full round takes lam_rp out again through its
            // lane-0 constant and column 0 of its matrix (Mpost = M * diag(lam_rp^alpha, 1, ..., 1)).  Exact field algebra.
            auto pow_alpha = [&](Fe b) {
                Fe y = F.one();
                for (u64 e = P.alpha; e; e >>= 1) {
                    if (e & 1) y = F.mul(y, b);
                    b = F.mul(b, b);
                }
                return y;
            };
            Fe lam = F.one();
            for (int k = 0; k < rp; k++) {
                Fe* row = &sp[(size_t)k * (2 * t - 1)];
                const Fe la = pow_alpha(lam), next = F.mul(row[0], la), inv_next = F.inv(next);
                row[0] = F.one();
                for (int j = 1; j < t; j++) row[j] = F.mul(row[j], inv_next);
                for (int j = 0; j < t - 1; j++) row[t + j] = F.mul(row[t + j], la);
                if (k > 0) pc[k] = F.mul(pc[k], F.inv(lam));
                lam = next;
            }
            C[(size_t)half * t] = F.mul(C[(size_t)half * t], F.inv(lam));
            const Fe la = pow_alpha(lam);
            for (int i = 0; i < t; i++) Mpost[(size_t)i * t] = F.mul(M[(size_t)i * t], la);

            // The split loop (pos_permute_split) carries lane 1 as a_k = w_hat_k . s (s = lanes 1..t-1, w_hat as scaled above) and
            // lanes 2.. as they are.  With w_hat_k[1] != 0, s_1 = (a_k - sum_{j>=2} w_hat_k[j]*s_j) / w_hat_k[1], so partial round k
            // (xi = S(L), L' = xi + a_k, s' = s + v_k*xi) needs no row product and updates lane 1 with one t-term dot:
            //   a_{k+1} = w_hat_{k+1} . s' = gamma_k*xi + alpha_k*a_k + sum_{j>=2} beta_kj*s_j,
            //   alpha_k = w_hat_{k+1}[1] / w_hat_k[1],  beta_kj = w_hat_{k+1}[j] - alpha_k*w_hat_k[j],  gamma_k = w_hat_{k+1} . v_k.
            // w_hat_rp := e_1 makes a_rp = s_1: the state leaves the loop in the plain basis.  Entry: a_0 = w_hat_0 . (Mpre*y + Cp0)
            // is folded into row 1 of Mpre and entry 1 of Cp0, stored separately because the merged loop and the team kernel
            // still read the plain ones.  Per round [gamma, alpha, beta_2..t-1 | v_k[2..t-1]] (the dot's coefficients in the
            // state's lane order), then the split form's Mpre row 1 (t) and Cp0 entry 1.  Exact field algebra.
            const int q = 2 * t - 2;
            lp.assign((size_t)rp * q + t + 1, F.zero());
            for (int k = 0; k < rp; k++) {
                const Fe* w = &sp[(size_t)k * (2 * t - 1)];                    // w[j] = w_hat_k[j] (j >= 1), v_k[j] = w[t - 1 + j]
                FeVec wn((size_t)t, F.zero());
                if (k + 1 < rp) for (int j = 1; j < t; j++) wn[j] = sp[(size_t)(k + 1) * (2 * t - 1) + j];
                else wn[1] = F.one();
                Fe* o = &lp[(size_t)k * q];
                o[1] = F.mul(wn[1], F.inv(w[1]));
                for (int j = 1; j < t; j++) o[0] = F.add(o[0], F.mul(wn[j], w[t - 1 + j]));
                for (int j = 2; j < t; j++) {
                    o[j] = F.sub(wn[j], F.mul(o[1], w[j]));
                    o[t + j - 2] = w[t - 1 + j];
                }
            }
            Fe* entry = &lp[(size_t)rp * q];
            for (int j = 1; j < t; j++) {
                const Fe w0 = sp[j];
                for (int i = 0; i < t; i++) entry[i] = F.add(entry[i], F.mul(w0, Mpre[(size_t)j * t + i]));
                entry[t] = F.add(entry[t], F.mul(w0, Cp0[j]));
            }
        }
    }
    if (!sparse) {
        // dense fallback: partial rounds exactly as written in the reference
        for (int fr = 0; fr < rf; fr++) {
            int r = fr < half ? fr : half + rp + (fr - half);
            for (int i = 0; i < t; i++) C[(size_t)fr * t + i] = ark(r, i);
        }
        Mpre = M;
        Mpost = M;
    }
    S.sparse = sparse ? 1 : 0;

    auto push = [&](const FeVec& v) {
        int off = (int)(S.consts.size() / 4);
        for (const Fe& e : v) S.consts.insert(S.consts.end(), e.l, e.l + 4);
        return off;
    };
    S.off_c = push(C);
    S.off_m = push(M);
    S.off_mpre = push(Mpre);
    push(Mpost);                   // at off_mpre + t*t (pos_full_matrix)
    S.off_cp0 = push(Cp0);
    S.off_pc = push(pc);
    S.off_sp = push(sp);
    if (sparse) arkp.clear();      // the original partial-round constants are read by the dense form only
    S.off_arkp = push(arkp);
    {
        Fe pm;
        memcpy(pm.l, F.p, 32);
        S.off_mod = push(FeVec(1, pm));
    }
    {
        Fe y = F.one(), b = C.empty() ? F.zero() : C[0];                       // C[0][0]^alpha (alpha = 0: the constant one, as the kernels' S-box)
        for (u64 e = P.alpha; e; e >>= 1) {
            if (e & 1) y = F.mul(y, b);
            b = F.mul(b, b);
        }
        S.off_sc0 = push(FeVec(1, y));
    }
    push(lp);                      // at off_sc0 + 1 (pos_permute_split); empty when dense
    S.n_elems = (int)(S.consts.size() / 4);
    if (sparse) {
        const FeVec* mats[3] = {&M, &Mpre, &Mpost};
        for (const FeVec* m : mats)
            for (const Fe& c : *m) push_digit_table(F, c, S.tabs);
        for (size_t i = 0; i + 1 < lp.size(); i++) push_digit_table(F, lp[i], S.tabs);
    }
    return S;
}

}  // namespace host
}  // namespace cpb
