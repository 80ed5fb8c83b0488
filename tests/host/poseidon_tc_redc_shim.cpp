// CPU build of the pieces of the S-box's tensor-core reduction (crypto_primitives_b200/csrc/poseidon_tc.cuh: tc_redc) that run
// on the host or outside the IMMA: the 512-bit products fp_sqr_wide and fp_mul_wide (fp.cuh), the R^-1 table
// (poseidon_host.hpp: tc_rinv_table) and its word map, PTX primitives emulated, for tests/test_poseidon_tc_redc.py.  Not part of
// the product.
#include "../../crypto_primitives_b200/csrc/poseidon.cuh"
#include "../../crypto_primitives_b200/csrc/poseidon_host.hpp"
using namespace cpb;

// T[16] = a*a (sq != 0) or a*b.
extern "C" void host_mul_wide(const uint32_t* a, const uint32_t* b, int sq, uint32_t* T) {
    u32 t[16];
    if (sq) fp_sqr_wide(t, a);
    else fp_mul_wide(t, a, b);
    for (int i = 0; i < 16; i++) T[i] = t[i];
}

// The BN254 Fr R^-1 table (kTcRinvWords words); returns the word count.
extern "C" long host_tc_rinv_table(uint32_t* out) {
    const std::vector<u32> t = host::tc_rinv_table(host::Field(host::field_modulus(Bn254_Fr::ID)));
    for (size_t i = 0; i < t.size(); i++) out[i] = t[i];
    return (long)t.size();
}

// tc_tab_word(nt, 0, lane, r, 1) for nt, lane, r in that order: where tc_output reads the R^-1 table.
extern "C" void host_tc_rinv_words(int* out) {
    for (int nt = 0; nt < 4; nt++)
        for (int lane = 0; lane < 32; lane++)
            for (int r = 0; r < 2; r++) *out++ = tc_tab_word(nt, 0, lane, r, 1);
}
