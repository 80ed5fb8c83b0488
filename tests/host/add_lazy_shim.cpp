// CPU build of fp_add_lazy (crypto_primitives_b200/csrc/fp.cuh, PTX primitives emulated) for BN254 Fr, the field whose lazy
// partial rounds use it.  Driven by tests/test_poseidon_lane1_basis.py.  Not part of the product library.
#include "../../crypto_primitives_b200/csrc/fp.cuh"
using namespace cpb;

// r[i] = a[i] + b[i] mod p for a[i] < 2p, b[i] < p; 8 little-endian 32-bit limbs per value.  r may alias a or b.
extern "C" void host_add_lazy_bn254(const u32* a, const u32* b, u32* r, long n) {
    for (long i = 0; i < n; i++) fp_add_lazy<Bn254_Fr>(r + 8 * i, a + 8 * i, b + 8 * i);
}
