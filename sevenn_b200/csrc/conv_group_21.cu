// Tensor-product kinds with lmax_filter = 2, lmax_out = 1 (see conv_dispatch.cuh): runtime-width kernels only.
#include "conv_dispatch.cuh"
S7B_DEFINE_CONV_GROUP(2, 1, 0)
