// Tensor-product kinds with lmax_filter = 2, lmax_out = 0 (see conv_dispatch.cuh): the kernels specialised
// for the widths of SevenNet-0 / SevenNet-l3i5 and the runtime-width kernels.
#include "conv_dispatch.cuh"
S7B_DEFINE_CONV_GROUP(2, 0, 1)
