// Top-level dispatch of the fused convolution launches over (lmax_filter, lmax_out) groups.
#include "common.cuh"

namespace s7b {

// One group's dispatch over l1 (conv_dispatch.cuh), instantiated in its translation unit conv_group_<LF><LO>.cu
template <int LF, int LO, class F>
int launch_conv_group(int l1, const F& f, const ConvArgs& a, const ConvRole& role, cudaStream_t st);

extern int64_t g_conv_launches;
int64_t g_conv_launches = 0;

// Return code of a group launch -> 0 (launched, counted, or nothing to launch) or 1 with the error set
static int conv_status(int rc) {
  if (rc == kConvNoPath) return 0;
  if (rc == 2) { set_error(__FILE__, __LINE__, "no tensor-product kind compiled for this (lmax_filter, lmax_out)"); return 1; }
  if (rc == kConvWrongMul) { set_error(__FILE__, __LINE__, "convolution multiplicities must be positive multiples of 32"); return 1; }
  if (rc) { set_error(__FILE__, __LINE__, cudaGetErrorString(cudaGetLastError())); return 1; }
  ++g_conv_launches;
  return 0;
}

// every (lmax_filter, lmax_out) with lmax_filter = 1..3 and lmax_out = 0..3 has a group
template <class F>
int launch_conv(int l1, int lf, int lo, const F& f, const ConvArgs& a, const ConvRole& role, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  switch (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3 ? lf * 10 + lo : 0) {
    case 10: rc = launch_conv_group<1, 0>(l1, f, a, role, st); break;
    case 11: rc = launch_conv_group<1, 1>(l1, f, a, role, st); break;
    case 12: rc = launch_conv_group<1, 2>(l1, f, a, role, st); break;
    case 13: rc = launch_conv_group<1, 3>(l1, f, a, role, st); break;
    case 20: rc = launch_conv_group<2, 0>(l1, f, a, role, st); break;
    case 21: rc = launch_conv_group<2, 1>(l1, f, a, role, st); break;
    case 22: rc = launch_conv_group<2, 2>(l1, f, a, role, st); break;
    case 23: rc = launch_conv_group<2, 3>(l1, f, a, role, st); break;
    case 30: rc = launch_conv_group<3, 0>(l1, f, a, role, st); break;
    case 31: rc = launch_conv_group<3, 1>(l1, f, a, role, st); break;
    case 32: rc = launch_conv_group<3, 2>(l1, f, a, role, st); break;
    case 33: rc = launch_conv_group<3, 3>(l1, f, a, role, st); break;
  }
  return conv_status(rc);
}

#define S7B_CONV_INSTANTIATE(F, ...) \
  struct F;                          \
  template int launch_conv<F>(int, int, int, const F&, const ConvArgs&, const ConvRole&, cudaStream_t);
S7B_CONV_FAMILIES(S7B_CONV_INSTANTIATE)

}  // namespace s7b
