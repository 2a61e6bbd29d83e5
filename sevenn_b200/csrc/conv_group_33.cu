// Tensor-product kinds with lmax_filter = 3, lmax_out = 3 (see conv_dispatch.cuh): the kernels specialised
// for the widths of SevenNet-0 / SevenNet-l3i5 and the runtime-width kernels.
#include "conv_dispatch.cuh"
S7B_DEFINE_CONV_GROUP(3, 3, 1)
