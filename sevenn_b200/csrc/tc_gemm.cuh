// Block-diagonal irreps linear on the Hopper tensor cores (wgmma + TMA + mbarrier, sm_90a):
//   C[(n,i), :N] (+)= A[(n,i), :K] * W[K, N]        fp32 in / fp32 out
// Same operand addressing as blocklin_gemm_kernel (node_kernels.cuh); replaces e3nn o3.Linear
// (sevenn/nn/linear.py:94-100) for self_interaction_1/2 and the self connection, forward and backward.
//
// Arithmetic: error-free tensor-core accumulation.  The tensor core adds into its fp32 accumulator with
// truncation, which biases long fp32/TF32 accumulations.
// Here every operand is first brought to 24-bit fixed point relative to a power-of-two bound of its row
// (A: per (node, component) row over all K, from row_exponent_kernel; W: per output column, on the host)
// and cut into three signed 8-bit slices  q = q0*2^16 + q1*2^8 + q2,  |q_i| <= 128, each exactly
// representable in bf16.  Then
//     a*b*2^-(Ea+Eb-14) = (A0+A1+A2)(B0+B1+B2),   A0 = q0, A1 = q1*2^-8, A2 = q2*2^-16 (same for B)
//   ACC0 = sum_k A0*B0                 integers < 2^23: EXACT in the fp32 accumulator, nothing to truncate
//   ACC1 = sum_k A0*B1+A1*B0+A0*B2+A1*B1+A2*B0     2^-8 of ACC0: its truncation is 2^-32 relative
//   C    = 2^(Ea-7) * 2^(Eb-7) * (ACC0 + ACC1)     one round-to-nearest fp32 add in the epilogue
// (the dropped A1*B2, A2*B1, A2*B2 are < 2^-24 relative).  Six bf16 MMAs per K = 16 step cost the same
// tensor time as 3xTF32.  Emulated bit for bit on the CPU by tests/test_tc_pack_cpu.py.
//
// Structure (persistent, one CTA per SM, 320 threads = 10 warps, tiles of 64 rows x NT <= 128 columns):
//   warp 8   TMA producer A: per 32-wide K chunk one cp.async.bulk.tensor (3-D map over (k, component,
//            node); 128B swizzle) for the raw fp32 A tile into an 8-deep ring (the HBM/L2 round trip of
//            these loads is what has to be hidden: 64 KB in flight per SM)
//   warp 9   producer W: one cp.async.bulk per chunk for the pre-sliced, pre-arranged W chunk (3-deep ring)
//   warps 0-3 transform: two threads per row of a raw chunk (16 of its 32 k each) pull it into registers
//            (freeing the raw slot), cut it into the three bf16 slices and write them in the canonical
//            K-major no-swizzle core-matrix layout (8-row x 16-byte core matrices) into a 3-deep operand ring
//   warps 4-7 one warpgroup: issues 12 wgmma.mma_async m64nNTk16 per chunk into its two register
//            accumulators (64 x NT each, NT/2 + NT/2 registers per thread), releases a chunk's operand slots
//            once the next chunk's MMAs are in flight (wgmma.wait_group 1), and after the tile's last chunk
//            scales the accumulators and writes C straight from the fragments (8-byte stores per thread, a
//            quad of lanes covers one 32-byte row segment), or RED.ADD.F32x2 when accumulating.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include <type_traits>

#include "common.cuh"
#include "node_kernels.cuh"

namespace s7b {

constexpr int kTcBM = 64;           // rows (nodes) per tile: the M of one wgmma
constexpr int kTcKC = 32;           // K elements per pipeline stage
constexpr int kTcMaxNT = 128;       // columns per tile
constexpr int kTcAccRegs = kTcMaxNT / 2;   // fp32 registers per thread of one m64nNTk16 accumulator at NT = 128
constexpr int kTcThreads = 320;     // 4 transform warps, one MMA + epilogue warpgroup, A producer, W producer
constexpr int kTcXformThreads = 128; // two threads per row of a chunk (16 of its 32 k each)
constexpr int kTcMmaWarps = 4;
constexpr int kTcRawBytes = kTcBM * kTcKC * 4;            // 8 KB raw fp32 A chunk
constexpr int kTcASliceBytes = kTcBM * kTcKC * 2;         // 4 KB per bf16 slice
constexpr int kTcBSliceBytes = kTcMaxNT * kTcKC * 2;      // 8 KB per bf16 slice (NT = 128)
// three decoupled rings: raw A chunks (deep: the HBM/L2 round trip of the TMA loads is what has to be
// hidden), sliced A operands and sliced W operands (both released by the MMA warpgroup)
constexpr int kTcRawStages = 8, kTcOpsStages = 3, kTcWStages = 3;
constexpr int kTcOpsBytes = 3 * kTcASliceBytes, kTcWBytes = 3 * kTcBSliceBytes;
constexpr int kTcRawOff = 0;
constexpr int kTcOpsOff = kTcRawOff + kTcRawStages * kTcRawBytes;
constexpr int kTcWOff = kTcOpsOff + kTcOpsStages * kTcOpsBytes;
constexpr int kTcSmemBytes = kTcWOff + kTcWStages * kTcWBytes + 1024 /*alignment slack*/;
constexpr int kTcZeroRow = -1000;   // row exponent of an all-zero row

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive that carries a REAL data dependency on `dep`: the arrival is predicated on a comparison of the
// value with a bit pattern no fp32 addition can produce, so neither nvcc nor ptxas can drop the dependency
// (a dead `mov` was dropped: the SASS then issued SYNCS.ARRIVE right behind the still outstanding loads and
// the TMA refill overtook them).  The warp therefore waits for the shared-memory loads that produced
// `dep` before it releases the slot they read.
__device__ __forceinline__ void mbar_arrive_after(uint64_t* bar, float dep) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %1, 0x7fc12345;\n"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(__float_as_uint(dep)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// TMA: 3-D tiled tensor load (coordinates innermost first) completing on an mbarrier
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
// TMA engine, linear form: contiguous global -> shared bulk copy completing on an mbarrier
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle: the two 8-row x 16-byte core matrices of one
// K = 16 step lie 128 bytes apart (leading byte offset), 8-row groups 512 bytes apart (stride byte offset).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(512 >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across a wgmma fence / wait
__device__ __forceinline__ void acc_fence(float (&d)[kTcAccRegs]) {
#pragma unroll
  for (int i = 0; i < kTcAccRegs; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64, N] (+)= A[64, 16] * B[16, N]: bf16 operands from shared memory, fp32 accumulator fragment in the
// first N/2 registers of d; scale_d = 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_bf16<16>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<32>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<48>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<80>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %42, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<96>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<112>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %58, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[kTcAccRegs], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

// 2^e as a float (e clamped to the normal range)
__device__ __forceinline__ float exp2i(int e) {
  e = e < -126 ? -126 : (e > 127 ? 127 : e);
  return __int_as_float((e + 127) << 23);
}

// ---- row exponents --------------------------------------------------------------------------------
// E(n, i) with max_k |A[(n,i), k]| < 2^E  (kTcZeroRow for an all-zero / denormal row); one warp per row.
struct RowExpArgs {
  const float* A;
  int* E;                 // [n_nodes, rows_per_node]
  int lda, n_nodes, rows_per_node, nblocks;
  int d[kMaxL], K[kMaxL], a_off[kMaxL], row_base[kMaxL];
};

__global__ void row_exponent_kernel(const RowExpArgs a) {
  // one warp per node: the node's row is read once, coalesced (float4 per lane); every float4 lies inside one
  // (block, component) row (K is a multiple of 4).  Lanes that hold quads of the same row combine their maxima
  // with one warp reduction (match.any + redux.sync), its leader updates the row's slot in shared memory.
  __shared__ unsigned int smax[8][16];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + wib;
  if (lane < 16) smax[wib][lane] = 0u;
  __syncwarp();
  if (n < a.n_nodes) {
    for (int b = 0; b < a.nblocks; ++b) {
      const int K = a.K[b], quads = (a.d[b] * K) >> 2;
      const float4* row = reinterpret_cast<const float4*>(a.A + (size_t)n * a.lda + a.a_off[b]);
      for (int q0 = 0; q0 < quads; q0 += 32) {
        const int q = q0 + lane;
        unsigned int m = 0u;
        int r = -1;
        if (q < quads) {
          const float4 v = __ldg(row + q);
          m = __float_as_uint(v.x) & 0x7fffffffu;
          m = max(m, __float_as_uint(v.y) & 0x7fffffffu);
          m = max(m, __float_as_uint(v.z) & 0x7fffffffu);
          m = max(m, __float_as_uint(v.w) & 0x7fffffffu);
          r = a.row_base[b] + (4 * q) / K;
        }
        const unsigned int peers = __match_any_sync(0xffffffffu, r);
        const unsigned int mm = __reduce_max_sync(peers, m);
        if (r >= 0 && lane == __ffs(peers) - 1) smax[wib][r] = max(smax[wib][r], mm);
        __syncwarp();
      }
    }
  }
  __syncwarp();
  if (n < a.n_nodes && lane < a.rows_per_node) {
    const int ex = (int)(smax[wib][lane] >> 23);
    a.E[(size_t)n * a.rows_per_node + lane] = (ex < 30 || ex == 255) ? kTcZeroRow : ex - 126;     // |a| < 2^(ex-126)
  }
}

// ---- the GEMM --------------------------------------------------------------------------------------
struct TcLinBlock {
  const uint16_t* Wq;   // pre-sliced weights: [nnt][K/32][3 slices][canonical NT x 32 bf16]
  const float* fb;      // [N] column scales 2^(Eb-7)
  int d, K, N, NT, nnt;  // nnt column tiles of NT columns each (nnt * NT >= N; the pad columns carry zero weights)
  int c_off, c_cs;
  int row_base;         // first row of this block in the row-exponent array
  int tile0;            // index of the block's first tile; tiles ordered [node tile][component][n tile]
};
struct TcLinArgs {
  float* C;
  const int* E;         // row exponents of A, [n_nodes, rows_per_node]
  int ldc, n_nodes, rows_per_node, accumulate, nblocks, n_tiles, swizzle;
  int e_bits;           // E holds the raw maxima (|a| bits, written by the producer kernel) instead of exponents
  long long* trace;     // optional timeline of CTA 0 (tools/tc_trace.py): records {role, event, index, clock64}
  int trace_cap;
  TcLinBlock blk[kMaxL];
};
// timeline events of CTA 0 (a.trace != nullptr): five roles, each traced by ONE thread that keeps its own
// record counter in a register and stores {event, index, clock64} with plain stores (no atomics: an atomic's
// round trip would cost more than the stages being measured).  Layout: role r owns records
// [r * trace_cap / 5, (r + 1) * trace_cap / 5); word 0 of the buffer is unused, counts are in words 1..5.
#define TC_TRACE(role, ev, idx)                                                                   \
  do {                                                                                            \
    if (a.trace != nullptr && blockIdx.x == 0) {                                                  \
      const int per = a.trace_cap / 5;                                                            \
      if (trace_n < per) {                                                                        \
        long long* rec = a.trace + 8 + 3 * ((size_t)(role) * per + trace_n);                      \
        rec[0] = (ev);                                                                            \
        rec[1] = (long long)(idx);                                                                \
        rec[2] = clock64();                                                                       \
        ++trace_n;                                                                                \
        a.trace[1 + (role)] = trace_n;                                                            \
      }                                                                                           \
    }                                                                                             \
  } while (0)
struct TcMaps { CUtensorMap m[kMaxL]; };   // per block: A viewed as (k, component, node), fp32

// explicit shared-space accesses (the ring pointers are computed from an aligned base, which makes the compiler
// fall back to generic LD/ST otherwise)
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ void sts128(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

// The 12 MMAs of one 32-wide K chunk (tile width N): ACC0 += A0*B0, ACC1 += the five cross terms
template <int N>
__device__ __forceinline__ void tc_mma_chunk(float (&acc0)[kTcAccRegs], float (&acc1)[kTcAccRegs], uint32_t sa,
                                             uint32_t sb, bool first) {
  constexpr uint32_t b_slice = (uint32_t)N * kTcKC * 2u;
#pragma unroll
  for (int j = 0; j < kTcKC / 16; ++j) {
    const uint32_t ko = (uint32_t)j * 256u;     // two 16-byte K core matrices per MMA
    const uint64_t dA0 = gmma_desc(sa + ko);
    const uint64_t dA1 = gmma_desc(sa + kTcASliceBytes + ko);
    const uint64_t dA2 = gmma_desc(sa + 2 * kTcASliceBytes + ko);
    const uint64_t dB0 = gmma_desc(sb + ko);
    const uint64_t dB1 = gmma_desc(sb + b_slice + ko);
    const uint64_t dB2 = gmma_desc(sb + 2 * b_slice + ko);
    const uint32_t acc = (!first || j > 0) ? 1u : 0u;
    wgmma_bf16<N>(acc0, dA0, dB0, acc);
    wgmma_bf16<N>(acc1, dA0, dB1, acc);
    wgmma_bf16<N>(acc1, dA1, dB0, 1u);
    wgmma_bf16<N>(acc1, dA0, dB2, 1u);
    wgmma_bf16<N>(acc1, dA1, dB1, 1u);
    wgmma_bf16<N>(acc1, dA2, dB0, 1u);
  }
}

__global__ void __launch_bounds__(kTcThreads, 1)
blocklin_tc_kernel(const TcLinArgs a, const __grid_constant__ TcMaps maps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t bar_raw_full[kTcRawStages], bar_raw_empty[kTcRawStages];
  __shared__ uint64_t bar_ops_full[kTcOpsStages], bar_ops_empty[kTcOpsStages];
  __shared__ uint64_t bar_w_full[kTcWStages], bar_w_empty[kTcWStages];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int trace_n = 0;

  if (tid == 0) {
    for (int s = 0; s < kTcRawStages; ++s) { mbar_init(&bar_raw_full[s], 1); mbar_init(&bar_raw_empty[s], kTcXformThreads); }
    for (int s = 0; s < kTcOpsStages; ++s) { mbar_init(&bar_ops_full[s], kTcXformThreads); mbar_init(&bar_ops_empty[s], kTcMmaWarps); }
    for (int s = 0; s < kTcWStages; ++s) { mbar_init(&bar_w_full[s], 1); mbar_init(&bar_w_empty[s], kTcMmaWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // tile t -> (block, node tile, component, n tile)
  auto decode = [&](int t, int& b, int& mt, int& ci, int& nt) {
    b = 0;
    while (b + 1 < a.nblocks && t >= a.blk[b + 1].tile0) ++b;
    const int rel = t - a.blk[b].tile0;
    const int nnt = a.blk[b].nnt;
    nt = rel % nnt;
    const int r2 = rel / nnt;
    ci = r2 % a.blk[b].d;
    mt = r2 / a.blk[b].d;
  };
  auto row_exp = [&](int t, int row) -> int {           // row exponent of tile t's row (kTcZeroRow beyond the nodes)
    if (t >= a.n_tiles) return kTcZeroRow;
    int b, mt, ci, nt;
    decode(t, b, mt, ci, nt);
    const int node = mt * kTcBM + row;
    if (node >= a.n_nodes) return kTcZeroRow;
    int v = __ldg(a.E + (size_t)node * a.rows_per_node + a.blk[b].row_base + ci);
    if (a.e_bits) {
      const int ex = v >> 23;
      v = (ex < 30 || ex == 255) ? kTcZeroRow : ex - 126;          // |a| < 2^(ex-126)
    }
    return v;
  };

  if (warp == 8) {
    // =================== TMA producer, A: raw fp32 chunks ===================
    if (lane == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        int b, mt, ci, nt;
        decode(t, b, mt, ci, nt);
        const int n_kc = a.blk[b].K / kTcKC;
        for (int kc = 0; kc < n_kc; ++kc, ++it) {
          const int s = it % kTcRawStages;
          mbar_wait(&bar_raw_empty[s], ((it / kTcRawStages) & 1) ^ 1);
          TC_TRACE(0, 0, it);      // A producer: slot free, issuing chunk `it`
          mbar_expect_tx(&bar_raw_full[s], (uint32_t)kTcRawBytes);
          tma_load_3d(smem + kTcRawOff + (size_t)s * kTcRawBytes, &maps.m[b], kc * kTcKC, ci, mt * kTcBM, &bar_raw_full[s]);
        }
      }
    }
  } else if (warp == 9) {
    // =================== TMA producer, W: pre-sliced bf16 chunks ===================
    if (lane == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        int b, mt, ci, nt;
        decode(t, b, mt, ci, nt);
        const TcLinBlock& B = a.blk[b];
        const int n_kc = B.K / kTcKC;
        const uint32_t b_bytes = 3u * (uint32_t)B.NT * kTcKC * 2u;
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(B.Wq) + (size_t)nt * n_kc * b_bytes;
        for (int kc = 0; kc < n_kc; ++kc, ++it) {
          const int s = it % kTcWStages;
          mbar_wait(&bar_w_empty[s], ((it / kTcWStages) & 1) ^ 1);
          TC_TRACE(4, 0, it);      // W producer: slot free, issuing
          mbar_expect_tx(&bar_w_full[s], b_bytes);
          bulk_load(smem + kTcWOff + (size_t)s * kTcWBytes, wsrc + (size_t)kc * b_bytes, b_bytes, &bar_w_full[s]);
        }
      }
    }
  } else if (warp < 4) {
    // =================== transform: raw fp32 row -> three bf16 slices ===================
    // thread (r, h): row r of the tile, k = 16 h .. 16 h + 15 of the chunk
    const int r = tid & (kTcBM - 1), h = tid / kTcBM;
    const uint32_t swz = a.swizzle ? (uint32_t)(r & 7) : 0u;
    const uint32_t row_off = (uint32_t)((r & 7) * 16 + (r >> 3) * 512);
    const V2 M2 = splat2(12582912.0f), nM2 = splat2(-12582912.0f);     // 1.5 * 2^23: (x + M) - M = rint(x)
    uint32_t it = 0;
    int Ea_next = row_exp(blockIdx.x, r);
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
      int b, mt, ci, nt;
      decode(t, b, mt, ci, nt);
      const int n_kc = a.blk[b].K / kTcKC;
      const int Ea = Ea_next;
      Ea_next = row_exp(t + gridDim.x, r);              // in flight while this tile is converted
      const float sc = (Ea == kTcZeroRow) ? 0.0f : exp2i(23 - Ea);     // t = a * sc, |t| < 2^23
      for (int kc = 0; kc < n_kc; ++kc, ++it) {
        const int s = it % kTcRawStages, o = it % kTcOpsStages;
        mbar_wait(&bar_raw_full[s], (it / kTcRawStages) & 1);
        if (tid == 0) TC_TRACE(1, 0, it);    // transform: raw chunk landed
        const uint32_t raw = smem_u32(smem + kTcRawOff + (size_t)s * kTcRawBytes + (size_t)r * 128);
        float4 v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = lds128(raw + (((uint32_t)(4 * h + q) ^ swz) << 4));
        const float dep = (v[0].x + v[1].x) + (v[2].x + v[3].x);   // touches every load: all four have returned
        mbar_arrive_after(&bar_raw_empty[s], dep);                  // the raw chunk is in registers: its slot can be refilled
        mbar_wait(&bar_ops_empty[o], ((it / kTcOpsStages) & 1) ^ 1);
        if (tid == 0) TC_TRACE(1, 1, it);    // transform: operand slot free
        const uint32_t a0 = smem_u32(smem + kTcOpsOff + (size_t)o * kTcOpsBytes);
        const uint32_t a1 = a0 + kTcASliceBytes, a2 = a1 + kTcASliceBytes;
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {                // 8 consecutive k = one 16-byte core-matrix row
          const V2 x[4] = {make_float2(v[2 * kk].x, v[2 * kk].y), make_float2(v[2 * kk].z, v[2 * kk].w),
                           make_float2(v[2 * kk + 1].x, v[2 * kk + 1].y), make_float2(v[2 * kk + 1].z, v[2 * kk + 1].w)};
          uint32_t p0[4], p1[4], p2[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const V2 tt = mul_(x[j], sc);
            const V2 q0 = add_(fma_(tt, splat2(1.52587890625e-05f), M2), nM2);        // rint(t / 2^16)
            const V2 r1 = fma_(q0, splat2(-65536.0f), tt);                            // exact
            const V2 q1 = add_(fma_(r1, splat2(0.00390625f), M2), nM2);               // rint(r1 / 2^8)
            const V2 r2 = fma_(q1, splat2(-256.0f), r1);                              // exact
            const V2 q2 = add_(add_(r2, M2), nM2);                                    // rint(r2)
            const V2 s1 = mul_(q1, 0.00390625f), s2 = mul_(q2, 1.52587890625e-05f);
            p0[j] = pack_bf16(q0.x, q0.y);
            p1[j] = pack_bf16(s1.x, s1.y);
            p2[j] = pack_bf16(s2.x, s2.y);
          }
          const uint32_t off = row_off + (uint32_t)(2 * h + kk) * 128u;
          sts128(a0 + off, p0[0], p0[1], p0[2], p0[3]);
          sts128(a1 + off, p1[0], p1[1], p1[2], p1[3]);
          sts128(a2 + off, p2[0], p2[1], p2[2], p2[3]);
        }
        fence_async_smem();          // generic-proxy smem writes -> visible to the tensor-core (async) proxy
        if (tid == 0) TC_TRACE(1, 2, it);    // transform: slices written
        mbar_arrive(&bar_ops_full[o]);
      }
    }
  } else if (warp < 8) {
    // =================== MMA + epilogue warpgroup (warps 4..7) ===================
    // accumulator fragment of m64nNk16: warp w of the group holds rows 16 w + lane/4 (registers 4j, 4j+1) and
    // 16 w + lane/4 + 8 (4j+2, 4j+3), columns 8 j + 2 (lane % 4) + {0, 1}
    const int mw = warp - 4, q4 = lane & 3;
    const int rl = 16 * mw + (lane >> 2);
    float acc0[kTcAccRegs], acc1[kTcAccRegs];
#pragma unroll
    for (int i = 0; i < kTcAccRegs; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
    uint32_t it = 0, tile_it = 0;
    int Ea_next0 = row_exp(blockIdx.x, rl), Ea_next1 = row_exp(blockIdx.x, rl + 8);
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++tile_it) {
      int b, mt, ci, nt;
      decode(t, b, mt, ci, nt);
      const TcLinBlock& B = a.blk[b];
      const int n_kc = B.K / kTcKC;
      const int Ea0 = Ea_next0, Ea1 = Ea_next1;
      Ea_next0 = row_exp(t + gridDim.x, rl);
      Ea_next1 = row_exp(t + gridDim.x, rl + 8);
      // the K loop of one tile, instantiated per tile width: the wgmma shape is an immediate, and a width
      // dispatch inside the loop would make ptxas serialize the MMAs
      auto mainloop = [&](auto width) {
        constexpr int N = decltype(width)::value;
        int prev_o = 0, prev_w = 0;
        for (int kc = 0; kc < n_kc; ++kc, ++it) {
          const int o = it % kTcOpsStages, w = it % kTcWStages;
          mbar_wait(&bar_w_full[w], (it / kTcWStages) & 1);
          if (tid == 128) TC_TRACE(2, 0, it);      // MMA: weights landed
          mbar_wait(&bar_ops_full[o], (it / kTcOpsStages) & 1);
          if (tid == 128) TC_TRACE(2, 1, it);      // MMA: operands ready, issuing
          __syncwarp();
          const uint32_t sa = smem_u32(smem + kTcOpsOff + (size_t)o * kTcOpsBytes);
          const uint32_t sb = smem_u32(smem + kTcWOff + (size_t)w * kTcWBytes);
          acc_fence(acc0);
          acc_fence(acc1);
          wgmma_fence();
          tc_mma_chunk<N>(acc0, acc1, sa, sb, kc == 0);
          wgmma_commit();
          acc_fence(acc0);
          acc_fence(acc1);
          wgmma_wait<1>();             // the previous chunk's MMAs have read their operands: release its slots
          if (kc > 0) {
            __syncwarp();
            if (lane == 0) { mbar_arrive(&bar_ops_empty[prev_o]); mbar_arrive(&bar_w_empty[prev_w]); }
          }
          prev_o = o;
          prev_w = w;
        }
        wgmma_wait<0>();
        acc_fence(acc0);
        acc_fence(acc1);
        __syncwarp();
        if (lane == 0) { mbar_arrive(&bar_ops_empty[prev_o]); mbar_arrive(&bar_w_empty[prev_w]); }
      };
      switch (B.NT) {
        case 16: mainloop(std::integral_constant<int, 16>()); break;
        case 32: mainloop(std::integral_constant<int, 32>()); break;
        case 48: mainloop(std::integral_constant<int, 48>()); break;
        case 64: mainloop(std::integral_constant<int, 64>()); break;
        case 80: mainloop(std::integral_constant<int, 80>()); break;
        case 96: mainloop(std::integral_constant<int, 96>()); break;
        case 112: mainloop(std::integral_constant<int, 112>()); break;
        default: mainloop(std::integral_constant<int, 128>()); break;
      }
      if (tid == 160) TC_TRACE(3, 0, tile_it);    // epilogue: accumulators complete

      // every element of C belongs to exactly one tile, so the single add per element is deterministic
      const float fa0 = (Ea0 == kTcZeroRow) ? 0.0f : exp2i(Ea0 - 7);
      const float fa1 = (Ea1 == kTcZeroRow) ? 0.0f : exp2i(Ea1 - 7);
      const int col0 = nt * B.NT;
      const int node0 = mt * kTcBM + rl;
      const bool ok0 = node0 < a.n_nodes, ok1 = node0 + 8 < a.n_nodes;
      float* c0 = a.C + (size_t)node0 * a.ldc + B.c_off + (size_t)ci * B.c_cs + col0 + 2 * q4;
      float* c1 = c0 + (size_t)8 * a.ldc;
      const float* fbp = B.fb + col0 + 2 * q4;
#pragma unroll
      for (int j = 0; j < kTcMaxNT / 8; ++j) {
        // column pairs are all-in or all-out (N a multiple of 4)
        if (8 * j < B.NT && col0 + 8 * j + 2 * q4 < B.N) {
          const float2 fb2 = __ldg(reinterpret_cast<const float2*>(fbp + 8 * j));
          const float2 v0 = make_float2((acc0[4 * j + 0] + acc1[4 * j + 0]) * fa0 * fb2.x,
                                        (acc0[4 * j + 1] + acc1[4 * j + 1]) * fa0 * fb2.y);
          const float2 v1 = make_float2((acc0[4 * j + 2] + acc1[4 * j + 2]) * fa1 * fb2.x,
                                        (acc0[4 * j + 3] + acc1[4 * j + 3]) * fa1 * fb2.y);
          if (a.accumulate) {
            if (ok0) atomicAdd(reinterpret_cast<float2*>(c0 + 8 * j), v0);
            if (ok1) atomicAdd(reinterpret_cast<float2*>(c1 + 8 * j), v1);
          } else {
            if (ok0) *reinterpret_cast<float2*>(c0 + 8 * j) = v0;
            if (ok1) *reinterpret_cast<float2*>(c1 + 8 * j) = v1;
          }
        }
      }
      if (tid == 160) TC_TRACE(3, 1, tile_it);        // epilogue: tile written
    }
  }
}

}  // namespace s7b
