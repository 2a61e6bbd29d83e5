// Tensor-product kinds with lmax_filter = 1, lmax_out = 1 (see conv_dispatch.cuh): runtime-width kernels only.
#include "conv_dispatch.cuh"
S7B_DEFINE_CONV_GROUP(1, 1, 0)
