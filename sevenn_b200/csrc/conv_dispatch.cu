// Top-level dispatch of the fused convolution launches over (lmax_filter, lmax_out) groups.
#include "common.cuh"

namespace s7b {

#define S7B_DECL_GROUP(LF, LO)                                                                      \
  int launch_conv_fwd_##LF##_##LO(int, bool, const ConvArgs&, const ConvRole&, float*, cudaStream_t); \
  int launch_conv_bwd_##LF##_##LO(int, bool, bool, const ConvArgs&, const ConvRole&, const float*,  \
                                  float*, float*, float*, float*, cudaStream_t);             \
  int launch_conv_jvp_##LF##_##LO(int, const ConvArgs&, const ConvRole&, const ConvTangents&, float*, cudaStream_t); \
  int launch_conv_bwdt_##LF##_##LO(int, const ConvArgs&, const ConvRole&, const ConvTangents&, const float*, \
                                   float*, float*, float*, cudaStream_t); \
  int launch_conv_flux_##LF##_##LO(int, const ConvArgs&, const ConvRole&, const FluxTangents&, int, int*, float*, \
                                   cudaStream_t); \
  int launch_conv_centroid_##LF##_##LO(int, const ConvArgs&, const ConvRole&, const CentroidAdjoints&, int, int*, \
                                       cudaStream_t);
S7B_DECL_GROUP(1, 0) S7B_DECL_GROUP(1, 1) S7B_DECL_GROUP(1, 2) S7B_DECL_GROUP(1, 3)
S7B_DECL_GROUP(2, 0) S7B_DECL_GROUP(2, 1) S7B_DECL_GROUP(2, 2) S7B_DECL_GROUP(2, 3)
S7B_DECL_GROUP(3, 0) S7B_DECL_GROUP(3, 1) S7B_DECL_GROUP(3, 2) S7B_DECL_GROUP(3, 3)

// every (lmax_filter, lmax_out) with lmax_filter = 1..3 and lmax_out = 0..3 has a group
#define S7B_GROUP_SWITCH(DIR, ...)                                                                  \
  switch (lf * 10 + lo) {                                                                           \
    case 10: rc = launch_conv_##DIR##_1_0(__VA_ARGS__); break;                                      \
    case 11: rc = launch_conv_##DIR##_1_1(__VA_ARGS__); break;                                      \
    case 12: rc = launch_conv_##DIR##_1_2(__VA_ARGS__); break;                                      \
    case 13: rc = launch_conv_##DIR##_1_3(__VA_ARGS__); break;                                      \
    case 20: rc = launch_conv_##DIR##_2_0(__VA_ARGS__); break;                                      \
    case 21: rc = launch_conv_##DIR##_2_1(__VA_ARGS__); break;                                      \
    case 22: rc = launch_conv_##DIR##_2_2(__VA_ARGS__); break;                                      \
    case 23: rc = launch_conv_##DIR##_2_3(__VA_ARGS__); break;                                      \
    case 30: rc = launch_conv_##DIR##_3_0(__VA_ARGS__); break;                                      \
    case 31: rc = launch_conv_##DIR##_3_1(__VA_ARGS__); break;                                      \
    case 32: rc = launch_conv_##DIR##_3_2(__VA_ARGS__); break;                                      \
    case 33: rc = launch_conv_##DIR##_3_3(__VA_ARGS__); break;                                      \
  }

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

int launch_conv_fwd(int l1, int lf, int lo, bool table, const ConvArgs& a, const ConvRole& role,
                    float* out, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3) S7B_GROUP_SWITCH(fwd, l1, table, a, role, out, st)
  return conv_status(rc);
}

int launch_conv_bwd(int l1, int lf, int lo, bool table, bool need_dx, const ConvArgs& a,
                    const ConvRole& role, const float* gout, float* dx, float* dY_acc,
                    float* dEdr_acc, float* dw, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3)
    S7B_GROUP_SWITCH(bwd, l1, table, need_dx, a, role, gout, dx, dY_acc, dEdr_acc, dw, st)
  return conv_status(rc);
}

int launch_conv_jvp(int l1, int lf, int lo, const ConvArgs& a, const ConvRole& role, const ConvTangents& tan,
                    float* out, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3) S7B_GROUP_SWITCH(jvp, l1, a, role, tan, out, st)
  return conv_status(rc);
}

int launch_conv_bwd_tangent(int l1, int lf, int lo, const ConvArgs& a, const ConvRole& role, const ConvTangents& tan,
                            const float* gout, float* dx, float* dY_acc, float* dw, cudaStream_t st) {
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3) S7B_GROUP_SWITCH(bwdt, l1, a, role, tan, gout, dx, dY_acc, dw, st)
  return conv_status(rc);
}

// One walk of the heat flux's convolution JVP over the channels c0 .. c0 + *nch - 1 (*nch set from the kind)
int launch_conv_flux(int l1, int lf, int lo, const ConvArgs& a, const ConvRole& role, const FluxTangents& f, int c0,
                     int* nch, float* out, cudaStream_t st) {
  *nch = 4;
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3) S7B_GROUP_SWITCH(flux, l1, a, role, f, c0, nch, out, st)
  return conv_status(rc);
}

// One walk of the centroid virial's convolution backward over the channels c0 .. c0 + *nch - 1 (*nch set from the
// kind)
int launch_conv_centroid(int l1, int lf, int lo, const ConvArgs& a, const ConvRole& role, const CentroidAdjoints& g,
                         int c0, int* nch, cudaStream_t st) {
  *nch = 4;
  if (a.n_dst <= a.n_begin) return 0;      // empty centre range
  int rc = 2;
  if (lf >= 1 && lf <= 3 && lo >= 0 && lo <= 3) S7B_GROUP_SWITCH(centroid, l1, a, role, g, c0, nch, st)
  return conv_status(rc);
}

}  // namespace s7b
