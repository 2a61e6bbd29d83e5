// Top-level dispatch of the fused convolution launches over (lmax_filter, lmax_out) groups.
#include "common.cuh"

namespace s7b {

#define S7B_DECL_GROUP(LF, LO)                                                                      \
  int launch_conv_fwd_##LF##_##LO(int, bool, const ConvArgs&, const ConvRole&, float*, cudaStream_t); \
  int launch_conv_bwd_##LF##_##LO(int, bool, bool, const ConvArgs&, const ConvRole&, const float*,  \
                                  float*, float*, float*, float*, cudaStream_t);
S7B_DECL_GROUP(2, 2)
S7B_DECL_GROUP(2, 0)
S7B_DECL_GROUP(3, 3)
S7B_DECL_GROUP(3, 0)

extern int64_t g_conv_launches;
int64_t g_conv_launches = 0;

int launch_conv_fwd(int l1, int lf, int lo, bool table, const ConvArgs& a, const ConvRole& role,
                    float* out, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf == 2 && lo == 2) rc = launch_conv_fwd_2_2(l1, table, a, role, out, st);
  else if (lf == 2 && lo == 0) rc = launch_conv_fwd_2_0(l1, table, a, role, out, st);
  else if (lf == 3 && lo == 3) rc = launch_conv_fwd_3_3(l1, table, a, role, out, st);
  else if (lf == 3 && lo == 0) rc = launch_conv_fwd_3_0(l1, table, a, role, out, st);
  if (rc == 2) { set_error(__FILE__, __LINE__, "no tensor-product kind compiled for this (lmax_filter, lmax_out)"); return 1; }
  if (rc == kConvWrongMul) { set_error(__FILE__, __LINE__, "no convolution kernel compiled for this l1 multiplicity"); return 1; }
  if (rc) { set_error(__FILE__, __LINE__, cudaGetErrorString(cudaGetLastError())); return 1; }
  ++g_conv_launches;
  return 0;
}

int launch_conv_bwd(int l1, int lf, int lo, bool table, bool need_dx, const ConvArgs& a,
                    const ConvRole& role, const float* gout, float* dx, float* dY_acc,
                    float* dEdr_acc, float* dw, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf == 2 && lo == 2) rc = launch_conv_bwd_2_2(l1, table, need_dx, a, role, gout, dx, dY_acc, dEdr_acc, dw, st);
  else if (lf == 2 && lo == 0) rc = launch_conv_bwd_2_0(l1, table, need_dx, a, role, gout, dx, dY_acc, dEdr_acc, dw, st);
  else if (lf == 3 && lo == 3) rc = launch_conv_bwd_3_3(l1, table, need_dx, a, role, gout, dx, dY_acc, dEdr_acc, dw, st);
  else if (lf == 3 && lo == 0) rc = launch_conv_bwd_3_0(l1, table, need_dx, a, role, gout, dx, dY_acc, dEdr_acc, dw, st);
  if (rc == 2) { set_error(__FILE__, __LINE__, "no tensor-product kind compiled for this (lmax_filter, lmax_out)"); return 1; }
  if (rc == kConvWrongMul) { set_error(__FILE__, __LINE__, "no convolution kernel compiled for this l1 multiplicity"); return 1; }
  if (rc) { set_error(__FILE__, __LINE__, cudaGetErrorString(cudaGetLastError())); return 1; }
  ++g_conv_launches;
  return 0;
}

}  // namespace s7b
