// Explicit instantiation of the batched duplex-sponge kernels for one field (all state widths t = 2..9).
#include "poseidon_kernels.cuh"
namespace cpb {
CPB_POS_WIDTHS(CPB_POS_INSTANTIATE_DUPLEX, Jubjub_Fr)
}
