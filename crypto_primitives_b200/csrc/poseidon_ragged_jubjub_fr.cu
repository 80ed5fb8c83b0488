// Explicit instantiation of the ragged-batch Poseidon kernels for one field (all state widths t = 2..9).
#include "poseidon_kernels.cuh"
namespace cpb {
CPB_POS_WIDTHS(CPB_POS_INSTANTIATE_RAGGED, Jubjub_Fr)
}
