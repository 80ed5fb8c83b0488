// Explicit instantiation of the Poseidon digest-fold verification kernel for one field (all state widths t = 2..9).
#include "poseidon_kernels.cuh"
namespace cpb {
CPB_POS_WIDTHS(CPB_POS_INSTANTIATE_DIGESTS, Bls12_377_Fr)
}
