// Host-side harness: exposes the per-lane arithmetic of the convolution's second-order kernels (tp_tangent.cuh) through
// a C interface so that tests/test_tp_tangent_cpu.py can check it against numpy on the CPU.
// (Test infrastructure only; compiled with g++ by the test.)
#include "../../sevenn_b200/csrc/tp_tangent.cuh"

using namespace s7b;

#define FOR_KINDS(X) \
  X(0,1,1) X(1,1,1) X(0,1,0) X(1,1,0) X(2,1,3) X(3,1,3) \
  X(0,2,2) X(1,2,2) X(2,2,2) X(0,2,0) X(1,2,0) X(2,2,0) X(3,2,3) \
  X(0,3,3) X(1,3,3) X(2,3,3) X(3,3,3) X(0,3,0) X(1,3,0) X(2,3,0) X(3,3,0) X(2,3,1)

template <class K>
static int bwd_out(int out, int has, const float* x, const float* Y, const float* w, const float* ga, const float* tx,
                   const float* tY, const float* tw, float* dw, float* dx, float* dY) {
  const bool hx = has & 1, hY = has & 2, hw = has & 4;
  switch (out) {
    case 7: TPTangent<K>::template bwd<true, true, true>(x, Y, w, ga, tx, tY, tw, hx, hY, hw, dw, dx, dY); return 0;
    case 1: TPTangent<K>::template bwd<true, false, false>(x, Y, w, ga, tx, tY, tw, hx, hY, hw, dw, dx, dY); return 0;
    case 2: TPTangent<K>::template bwd<false, true, false>(x, Y, w, ga, tx, tY, tw, hx, hY, hw, dw, dx, dY); return 0;
    case 4: TPTangent<K>::template bwd<false, false, true>(x, Y, w, ga, tx, tY, tw, hx, hY, hw, dw, dx, dY); return 0;
  }
  return 1;
}

extern "C" {

// has = bit 0: tx, bit 1: tY, bit 2: tw;  out = bit 0: dw, bit 1: dx, bit 2: dY (TPTangent::bwd<DW, DX, DY>)
int tt_jvp(int l1, int lf, int lo, int has, const float* x, const float* Y, const float* w, const float* tx,
           const float* tY, const float* tw, float* acc) {
#define X(a,b,c) if (l1==a && lf==b && lo==c) { TPTangent<TPKind<a,b,c>>::jvp(x, Y, w, tx, tY, tw, has & 1, has & 2, has & 4, acc); return 0; }
  FOR_KINDS(X)
#undef X
  return 1;
}

int tt_bwd(int l1, int lf, int lo, int has, int out, const float* x, const float* Y, const float* w, const float* ga,
           const float* tx, const float* tY, const float* tw, float* dw, float* dx, float* dY) {
#define X(a,b,c) if (l1==a && lf==b && lo==c) return bwd_out<TPKind<a,b,c>>(out, has, x, Y, w, ga, tx, tY, tw, dw, dx, dY);
  FOR_KINDS(X)
#undef X
  return 1;
}

}  // extern "C"
