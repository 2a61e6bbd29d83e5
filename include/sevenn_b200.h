/* sevenn_b200 -- C ABI of the H100-native SevenNet energy/force engine.
 *
 * Plain pointers and sizes only (no torch / C++ types): this is the boundary a maintainer of
 * the reference binds with ctypes / cgo-style FFI (see INTEGRATION.md).  All device pointers
 * are CUDA device memory on the current device; `stream` is a cudaStream_t passed as void*.
 * Every function returns 0 on success and non-zero on error; s7b_last_error() then returns a
 * human-readable message (thread-local).
 *
 * Reference interfaces replaced (paths relative to the reference tree):
 *   - the TP-accelerator plug-in `convolution_cls`
 *       sevenn/nn/convolution.py:243-247,270-276 (call contract)
 *       sevenn/nn/flash_helper.py:33-48, sevenn/nn/oeq_helper.py:30-70 (existing adapters)
 *       sevenn/pair_e3gnn/pair_e3gnn_oeq_autograd.cpp:23-27,64-133 (C++ fwd/bwd op signatures)
 *     -> s7b_conv_plan_create / s7b_conv_forward / s7b_conv_backward
 *   - the model forward + autograd force path executed per MD step by
 *       sevenn/calculator.py:219-233 (SevenNetCalculator.calculate)
 *       sevenn/pair_e3gnn/pair_e3gnn.cpp:74-289 (PairE3GNN::compute: edges in, E/F/virial out)
 *     -> s7b_engine_* (device-resident graph) and s7b_engine_compute_host (host buffers)
 *   - the per-layer segments + ghost exchange hooks of
 *       sevenn/pair_e3gnn/pair_e3gnn_parallel.cpp:345-441 (segment forward / manual backward)
 *     -> s7b_engine_run_stage + s7b_engine_buffer (the caller exchanges ghost rows between stages)
 */
#ifndef SEVENN_B200_H
#define SEVENN_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define S7B_API __attribute__((visibility("default")))
#else
#define S7B_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define S7B_MAX_LAYERS 8
#define S7B_MAX_L 4 /* l = 0..3 */

typedef struct S7bEngine S7bEngine;
typedef struct S7bConvPlan S7bConvPlan;

/* Model architecture (even-parity NequIP-type SevenNet; sevenn/model_build.py:448-616). */
typedef struct {
  int32_t n_layers;                                   /* interaction layers (5 for SevenNet-0) */
  int32_t lmax_filter;                                /* spherical harmonics up to this l */
  int32_t num_species;
  int32_t n_basis;                                    /* Bessel functions (8) */
  float cutoff;
  int32_t cutoff_fn;                                  /* 0 = XPLOR, 1 = polynomial */
  float cutoff_on;                                    /* XPLOR r_on */
  int32_t poly_p;
  int32_t radial_hidden[2];                           /* radial MLP hidden widths (64, 64) */
  int32_t n_l[S7B_MAX_LAYERS + 1];                    /* number of l's of irreps t (t = n_layers: output) */
  int32_t muls[S7B_MAX_LAYERS + 1][S7B_MAX_L];        /* multiplicity of l in irreps t: positive multiples of 32
                                                         (x of a layer: at most 1024).  The widths of SevenNet-0 /
                                                         SevenNet-l3i5 (128, 64, 32, 32 at l = 0..3, lmax_filter 2 or 3,
                                                         lmax_out = lmax_filter or 0) run convolution kernels
                                                         specialised for them; every other width and lmax combination
                                                         runs the runtime-width convolution kernels. */
  int32_t table_knots;                                /* > 0: radial weights from cubic tables */
} S7bModelDesc;

/* Stages of one energy/force evaluation (single GPU: s7b_engine_compute runs them all).
 * Multi-GPU callers run them one by one and exchange ghost rows in between:
 *   FWD_BEGIN | for t: FWD_LAYER(t) [exchange ghost rows of x(t+1)] | FWD_END |
 *   for t = T-1..0: BWD_LAYER_A(t) [reverse-add ghost rows of dx(t)] BWD_LAYER_B(t) |
 *   BWD_END [reverse-add ghost rows of forces]                                               */
enum {
  S7B_STAGE_FWD_BEGIN = 0,
  S7B_STAGE_FWD_LAYER = 1,
  S7B_STAGE_FWD_END = 2,
  S7B_STAGE_BWD_LAYER_A = 3,
  S7B_STAGE_BWD_LAYER_B = 4,
  S7B_STAGE_BWD_END = 5,
  /* finer split for comm/compute overlap (FWD_LAYER = FWD_LAYER_A + FWD_LAYER_SC, BWD_LAYER_B = B1 + B2):
   * FWD_LAYER_A(t) ends with the local rows of x(t+1); the self-connection GEMM FWD_LAYER_SC(t) does not
   * need the ghost rows and can run while they are exchanged.  BWD_LAYER_B1(t) (self-connection term of
   * dE/dh) does not need the reverse exchange of dx(t); BWD_LAYER_B2(t) adds the dx term afterwards. */
  S7B_STAGE_FWD_LAYER_A = 6,
  S7B_STAGE_FWD_LAYER_SC = 7,
  S7B_STAGE_BWD_LAYER_B1 = 8,
  S7B_STAGE_BWD_LAYER_B2 = 9,
  /* interior / boundary split of the convolutions (s7b_engine_set_interior): owned atoms [0, n_interior)
   * have no ghost neighbour.  FWD_LAYER_A(t) = FWD_CONV_INTERIOR(t) + FWD_LAYER_A2(t): the interior
   * convolution needs no ghost row of x(t) and runs while they are still in flight.
   * BWD_LAYER_A(t) = BWD_LAYER_A1(t) + BWD_LAYER_A2(t): A1 ends with the boundary atoms' backward
   * convolution, after which the ghost rows of dx(t) are final and can travel while A2 (interior) runs. */
  S7B_STAGE_FWD_CONV_INTERIOR = 10,
  S7B_STAGE_FWD_LAYER_A2 = 11,
  S7B_STAGE_BWD_LAYER_A1 = 12,
  S7B_STAGE_BWD_LAYER_A2 = 13
};

S7B_API const char* s7b_last_error(void);
S7B_API int s7b_version(void);

/* Runtime options: "tc_gemm" = 1 (default) runs the node linears on the tensor cores (TMA-fed
 * wgmma, register accumulators, error-free bf16x3 fixed-point slices: sevenn_b200/csrc/tc_gemm.cuh); 0 selects the
 * FP32 SIMT GEMM kernel (IEEE fp32 FMA chain).  "tc_swizzle" (default 1): 128B-swizzled TMA tiles.
 * "atomic_virial" = 1: engines created afterwards also fill the buffer "atomic_virial" [n_nodes, 6]
 * (force_output.py:198-214).  "concurrent_conv" (default 1): co-schedule the per-l1 convolution kernels.
 * "cuda_graph" (default 1): s7b_engine_compute (and the two *_host entry points built on it) replay a
 * captured CUDA graph of the step instead of issuing its ~75 launches; recaptured automatically when
 * sizes, edge capacity, graph pointers or allocations change.  "stage_graphs" (default 0): s7b_engine_run_stage
 * replays one captured graph per (stage, layer) -- see s7b_engine_stage_graph_stats.  "gate_bwd_rows" (default 0):
 * the gate backward also leaves the row maxima of dg for the tensor-core linears (saves one pass per layer).
 * Unknown names return non-zero with s7b_last_error() set. */
S7B_API int s7b_set_option(const char* name, int value);

/* C[rows, N] = A[rows, K] * W[K, N] (row-major, device pointers) through the same GEMM kernels the
 * engine uses for its linears; use_tc selects the tensor-core path (needs K % 32 == 0, N % 16 == 0). */
S7B_API int s7b_dense_linear(const float* A, const float* W, float* C, int64_t rows, int32_t K, int32_t N,
                             int32_t use_tc, void* stream);

/* Ghost-exchange pack / unpack for multi-GPU callers (device pointers; the transfer itself is the caller's:
 * NCCL send/recv in sevenn_b200/parallel.py).  Replaces the pack/unpack loops of
 * sevenn/pair_e3gnn/pair_e3gnn_parallel.cpp:698-799.
 *   gather:      out[i, :width] = src[idx[i], :width]           (out packed [n, width])
 *   scatter_add: dst[idx[i], :width] += in[i, :width]           (idx unique within one call) */
S7B_API int s7b_gather_rows(const float* src, int32_t ld_src, const int32_t* idx, int64_t n, int32_t width,
                            float* out, void* stream);
S7B_API int s7b_scatter_add_rows(float* dst, int32_t ld_dst, const int32_t* idx, int64_t n, int32_t width,
                                 const float* in, void* stream);

/* One block-diagonal irreps linear C_l (+)= A_l W_l, l = 0..n_l-1 (block l: 2l+1 rows per node, component-
 * major rows of K_l / N_l floats at a_off[l] / c_off[l] inside node rows of lda / ldc floats) through the
 * engine's own kernels: use_tc = 1 the tensor-core path, 0 the FP32 SIMT kernel.  A, C device; W host. */
S7B_API int s7b_block_linear(const float* A, int32_t lda, int32_t n_nodes, int32_t n_l, const int32_t* a_off,
                             const int32_t* a_K, const float* W_host, float* C, int32_t ldc, const int32_t* c_off,
                             const int32_t* c_N, int32_t accumulate, int32_t use_tc, void* stream);

/* Test / utility entry: one species-wise block-diagonal linear  C_l[n] (+)= A_l[n] * W_l[species[n]]  (block l has 2l+1
 * rows per node, l < n_l) through the engine's kernels: the counting sort of the rows by species, then the
 * species-segmented GEMM the 'nequip' self-connection runs on.  A, C and species[n_rows] are device pointers, W a host
 * pointer laid out [num_species][l block][K_l][N_l].  Rows whose species lies outside [0, num_species) are not written.
 * K_l, N_l, the offsets and lda / ldc must be multiples of 4. */
S7B_API int s7b_species_linear(const float* A, int32_t lda, int32_t n_rows, const int32_t* species, int32_t num_species,
                               int32_t n_l, const int32_t* a_off, const int32_t* a_K, const float* W_host, float* C,
                               int32_t ldc, const int32_t* c_off, const int32_t* c_N, int32_t accumulate, void* stream);

/* Debug aid: timeline (role, event, index, clock64) of CTA 0 of the following tensor-core linear launches,
 * written to a device buffer of 8 + 3 * cap int64 (words 1..5 = records of each of the five roles, then cap / 5
 * records {event, index, clock64} per role); cap = 0 switches it off. */
S7B_API int s7b_tc_trace_enable(int32_t cap, void** device_buffer);

/* Host-only helper (no GPU needed): the weight packing of the tensor-core linear for one [K, N] block --
 * three signed 8-bit fixed-point slices per weight as bf16, in the shared-memory layout the kernel
 * consumes (sevenn_b200/csrc/tc_gemm.cuh).  q: 3*K*N uint16, fb: N column scales, *NT: tile width. */
S7B_API int s7b_tc_pack_weights(const float* W, int32_t K, int32_t N, uint16_t* q, float* fb, int32_t* NT);

/* ---- engine ---------------------------------------------------------------------------- */
S7B_API int s7b_engine_create(const S7bModelDesc* desc, S7bEngine** out);
S7B_API void s7b_engine_destroy(S7bEngine* eng);

/* Per engine: also fill the buffer "atomic_virial" [n_nodes, 6] (force_output.py:198-214) from the next
 * s7b_engine_set_graph on.  (The process-wide option "atomic_virial" only sets the default of engines
 * created afterwards; this call is the thread-safe way.) */
S7B_API int s7b_engine_set_atomic_virial(S7bEngine* eng, int enable);

/* Upload one named parameter array (host pointer, fp32).  Names: "embed_x0", "embed_g0",
 * "readout" (+ optional "readout_lo", the fp32 residual of the fp64 fold), "scale", "shift", "bessel", and per layer t "si1", "si1T", "sc", "scT", "si2",
 * "si2T", "table", "mlp0".."mlp2", "mlp0T".."mlp2T" (layouts: sevenn_b200/engine.py).  A layer with the species-wise
 * ('nequip') self-connection takes "sc_species" / "scT_species" ([num_species][l block][K][N], the transpose per block)
 * instead of "sc" / "scT"; setting both kinds on one layer is an error. */
S7B_API int s7b_engine_set_param(S7bEngine* eng, const char* name, int layer, const float* host, size_t numel);

/* Describe the graph of this step (device pointers, kept by reference until the next call).
 * Nodes 0..n_local-1 are owned atoms, n_local..n_nodes-1 ghosts; edges are sorted by centre:
 * rowptr[n_local+1] is the CSR over centres, src[e] in [0, n_nodes), edge_vec = r_src - r_centre. */
S7B_API int s7b_engine_set_graph(S7bEngine* eng, int32_t n_nodes, int32_t n_local, int64_t n_edges,
                         const int32_t* d_species, const int32_t* d_rowptr, const int32_t* d_src,
                         const float* d_edge_vec, void* stream);

/* Number of leading owned atoms without ghost neighbours (default: n_local, i.e. no boundary range);
 * call after s7b_engine_set_graph.  Only the split stages 10-13 look at it. */
S7B_API int s7b_engine_set_interior(S7bEngine* eng, int32_t n_interior);

S7B_API int s7b_engine_run_stage(S7bEngine* eng, int stage, int layer, void* stream);
S7B_API int s7b_engine_compute(S7bEngine* eng, void* stream);

/* Device pointer to an engine-owned buffer (valid until the next set_graph that grows it):
 * "x" (layer t input after self_interaction_1, [n_nodes, dim_x(t)]), "dx", "gate_in", "mid",
 * "h", "energy" (double[1]), "atomic_energy" [n_local], "atomic_energy_f64" (double[n_local], the same
 * per-atom energies before their rounding to float), "forces" [n_nodes,3], "edge_force" [E,3],
 * "virial" (double[6], = -sum r (x) f), "edge_Y", "edge_rec".  *numel receives the element count. */
S7B_API void* s7b_engine_buffer(S7bEngine* eng, const char* name, int layer, size_t* numel);

/* Host-buffer entry point, the analogue of PairE3GNN::compute (pair_e3gnn.cpp:74-289):
 * edges as (centre, neighbour, vector) triples sorted by centre, H2D + all stages + D2H.
 * forces: [n_nodes,3]; virial: 6 doubles (xx,yy,zz,xy,yz,zx of -sum r (x) f); atomic_energy may be NULL. */
S7B_API int s7b_engine_compute_host(S7bEngine* eng, int32_t n_nodes, int64_t n_edges,
                            const int32_t* species, const int32_t* edge_centre,
                            const int32_t* edge_neighbour, const float* edge_vec, double* energy,
                            float* atomic_energy, float* forces, double* virial, void* stream);

/* Host-staged stage protocol (a LAMMPS pair style that exchanges ghost rows through MPI host buffers, as
 * PairE3GNNParallel does without CUDA-aware MPI, pair_e3gnn_parallel.cpp:698-799): the graph with ghosts from host
 * arrays (edges as (centre, neighbour, vector) sorted by centre, centres < n_local, neighbours < n_nodes), and
 * rows [row_begin, row_begin + n_rows) of an fp32 engine buffer (names of s7b_engine_buffer; `width` floats per
 * row) copied to / from the host between the stages.  All three synchronise the stream. */
S7B_API int s7b_engine_set_graph_host(S7bEngine* eng, int32_t n_nodes, int32_t n_local, int64_t n_edges,
                                      const int32_t* species, const int32_t* edge_centre, const int32_t* edge_neighbour,
                                      const float* edge_vec, void* stream);
S7B_API int s7b_engine_read_rows_host(S7bEngine* eng, const char* name, int layer, int32_t row_begin, int32_t n_rows,
                                      int32_t width, float* host_out, void* stream);
S7B_API int s7b_engine_write_rows_host(S7bEngine* eng, const char* name, int layer, int32_t row_begin, int32_t n_rows,
                                       int32_t width, const float* host_in, void* stream);
/* energy (1 double) and virial (6 doubles: xx,yy,zz,xy,yz,zx of -sum r (x) f) of the last BWD_END; either may be NULL */
S7B_API int s7b_engine_read_scalars_host(S7bEngine* eng, double* energy, double* virial6, void* stream);

/* Positions in (SURVEY 8(f).1): builds the neighbour list / CSR graph on the device (cell list over the
 * fractional cell, any cell size and shape, per-direction pbc) with the semantics of the reference's
 * graph builder (sevenn/train/dataload.py:32-129: every image pair with |r_j - r_i + S.cell| < cutoff,
 * edge_vec in double -> float) and makes it the engine's current graph.  positions [n,3] and cell
 * [3,3] (rows = lattice vectors) are host doubles, pbc3 host ints.  The compute variant then runs all
 * stages and copies energy / forces [n,3] / virial back; *n_edges_out receives the edge count. */
S7B_API int s7b_engine_set_positions_host(S7bEngine* eng, int32_t n_atoms, const int32_t* species,
                                          const double* positions, const double* cell9, const int32_t* pbc3,
                                          void* stream);
S7B_API int s7b_engine_compute_positions_host(S7bEngine* eng, int32_t n_atoms, const int32_t* species,
                                              const double* positions, const double* cell9,
                                              const int32_t* pbc3, double* energy, float* atomic_energy,
                                              float* forces, double* virial, int64_t* n_edges_out,
                                              void* stream);

/* Multi-GPU front-end: neighbour rows of a subset of centre atoms (a rank's own atoms, `centres` = indices into
 * the n_atoms atoms) against ALL atoms, built on the device with the same semantics as above.  Does not touch
 * the engine's graph: read "nl_rowptr" [n_centres+1], "nl_src" [E] (indices into the n_atoms atoms), "nl_vec"
 * [E,3] with s7b_engine_buffer.  Replaces the per-step ghost / edge build of pair_e3gnn_parallel.cpp:194-340. */
S7B_API int s7b_engine_neighbor_rows_host(S7bEngine* eng, int32_t n_atoms, const int32_t* species, const double* positions,
                                          const double* cell9, const int32_t* pbc3, int32_t n_centres,
                                          const int32_t* centres, int64_t* n_edges_out, void* stream);

/* B independent structures; atoms of structure b are [atom_ptr[b], atom_ptr[b+1]) (host, B+1 entries,
 * atom_ptr[0] = 0, non-decreasing; empty structures are legal).  species [n] and positions [n,3] (double)
 * are DEVICE pointers; cells [B,9] (rows = lattice vectors) and pbc [B,3] are host arrays.
 * Builds every structure's neighbour list in one pass, with the semantics of s7b_engine_set_positions_host
 * per structure, and installs the union graph (no cross-structure edges).  Each structure gets the cell-list
 * grid it would get alone, so its CSR rows are those of s7b_engine_set_positions_host with offsets.  Kernel
 * launches and host synchronisations do not depend on B.  Bad arguments (atom_ptr, a zero lattice vector or
 * singular cell along a periodic direction -- the message names the structure) fail before the device is
 * touched.  The graph lives in engine-owned buffers, so a following call whose edge count stays within
 * their headroom replays the captured step of s7b_engine_compute. */
S7B_API int s7b_engine_set_positions_batch(S7bEngine* eng, int32_t n_systems, const int32_t* atom_ptr,
                                           const int32_t* d_species, const double* d_positions,
                                           const double* cells9, const int32_t* pbc3,
                                           int64_t* n_edges_out, void* stream);

/* After s7b_engine_compute on a graph from s7b_engine_set_positions_batch: per-structure energy [B] and
 * virial [B,6] (xx,yy,zz,xy,yz,zx of -sum r (x) f), fp64, device pointers, deterministic given edge forces.
 * The energy sums the fp64 per-atom energies (engine buffer "atomic_energy_f64").  Fails when the current
 * graph was not installed by s7b_engine_set_positions_batch. */
S7B_API int s7b_engine_system_results(S7bEngine* eng, double* d_energy, double* d_virial, void* stream);

/* Per-kernel timing with CUDA events recorded on the launching stream around every kernel (or
 * kernel group) of the stage sequence; labels like "conv_bwd.t2.l1".  Enable, run steps, then read. */
S7B_API int s7b_engine_set_profiling(S7bEngine* eng, int enable);
S7B_API int s7b_engine_profile_count(S7bEngine* eng);
S7B_API int s7b_engine_profile_entry(S7bEngine* eng, int index, char* name, size_t name_len,
                                     double* total_ms, int64_t* calls);

/* Number of kernels this library launched since the last reset (bench.py's gpu_launches); kernels run
 * by a CUDA-graph replay are counted per replay. */
S7B_API int64_t s7b_launch_count(int reset);

/* How often s7b_engine_compute captured a new CUDA graph / replayed one (either pointer may be NULL). */
S7B_API int s7b_engine_graph_stats(S7bEngine* eng, int64_t* captures, int64_t* replays);

/* With s7b_set_option("stage_graphs", 1), s7b_engine_run_stage captures each (stage, layer) into its own CUDA
 * graph on first use and replays it on the caller's stream afterwards (table radial mode, not under
 * profiling, not while the caller's stream is itself capturing).  Meant for callers that put their own
 * work -- the ghost exchanges of the multi-GPU runner -- between the stages.  Captures / replays so far: */
S7B_API int s7b_engine_stage_graph_stats(S7bEngine* eng, int64_t* captures, int64_t* replays);

/* ---- operator-level plug-in: fused gather -> 'uvu' tensor product -> scatter ------------- */
/* irreps of x as multiplicities per l (even parity; positive multiples of 32, at most 1024), filter lmax 1..3,
 * and lmax of the output 0..3; the instruction set is the complete triangle-allowed one of
 * sevenn/nn/convolution.py:61-82.  Widths other than 128, 64, 32, 32 at l = 0..3, and (lmax_filter, lmax_out)
 * other than (2, 2), (2, 0), (3, 3), (3, 0), run the runtime-width kernels.                                   */
S7B_API int s7b_conv_plan_create(int32_t n_l_x, const int32_t* x_muls, int32_t lmax_filter,
                         int32_t lmax_out, S7bConvPlan** out);
S7B_API void s7b_conv_plan_destroy(S7bConvPlan* plan);
S7B_API int s7b_conv_plan_dims(const S7bConvPlan* plan, int32_t* dim_x, int32_t* dim_mid, int32_t* weight_numel,
                       int32_t* n_sh);

/* All tensors in the engine's component-major layout (sevenn_b200/conv_op.py converts from
 * e3nn mul_ir): x [n_nodes, dim_x], sh [E, n_sh] (incl. Y_0), weight [E, W], edges sorted by
 * centre with rowptr [n_dst+1]; out [n_dst, dim_mid] is overwritten.  E == 0 is legal.          */
S7B_API int s7b_conv_forward(const S7bConvPlan* plan, const float* x, const float* sh, const float* weight,
                     const int32_t* rowptr, const int32_t* src, int32_t n_nodes, int32_t n_dst,
                     int64_t n_edges, float* out, void* stream);
/* grad_x [n_nodes, dim_x] (overwritten), grad_sh [E, n_sh], grad_weight [E, W]. */
S7B_API int s7b_conv_backward(const S7bConvPlan* plan, const float* x, const float* sh, const float* weight,
                      const int32_t* rowptr, const int32_t* src, int32_t n_nodes, int32_t n_dst,
                      int64_t n_edges, const float* grad_out, float* grad_x, float* grad_sh,
                      float* grad_weight, void* stream);

/* ---- D3 dispersion correction (SURVEY 8(f).2) ------------------------------------------------------
 * Cell-list DFT-D3 (zero / Becke-Johnson damping) replacing the reference's all-pairs CUDA code
 * sevenn/pair_e3gnn/pair_d3.cu / pair_d3_for_ase.cu (kernels :765-845, 1004-1058, 1263-1745, 1797-1962).
 * Native interface: tables reduced to the system's atom types (sevenn_b200/d3.py does what
 * PairD3::coeff, :633-845, does), positions / cell rows in Angstrom, types 0-based.  Stages operate on an
 * atom range of the bin-sorted order so that several GPUs can share one system (atom decomposition with
 * replicated positions; the caller all-gathers "cn" after stage 1 and "dc6i" after stage 2):
 *   1 = coordination numbers, 2 = C6 weights of all atoms + pair energy / forces / dE/dCN of the range,
 *   3 = chain-rule forces through the coordination numbers. */
typedef struct S7bD3 S7bD3;
S7B_API int s7b_d3_create(S7bD3** out);
S7B_API void s7b_d3_destroy(S7bD3* d3);
S7B_API int s7b_d3_set_params(S7bD3* d3, int32_t ntypes, const double* rcov, const double* r2r4, const double* r0ab,
                              const double* c6ref, const double* cnref, const int32_t* mxc);
/* damping: 0 = zero, 1 = Becke-Johnson; cutoffs are squared distances in bohr^2 (reference defaults 9000 / 1600) */
S7B_API int s7b_d3_set_damping(S7bD3* d3, int32_t damping, double s6, double s8, double a1, double a2, double alp6,
                               double alp8, double vdw_cutoff_au2, double cn_cutoff_au2);
/* types / positions / cell9 / pbc3 are host arrays; they are copied before the call returns (it synchronises stream) */
S7B_API int s7b_d3_set_system(S7bD3* d3, int32_t n_atoms, const int32_t* types, const double* positions,
                              const double* cell9, const int32_t* pbc3, void* stream);
S7B_API int s7b_d3_run_stage(S7bD3* d3, int32_t stage, int32_t i_begin, int32_t i_end, void* stream);
/* device buffers in bin-sorted order: "cn", "dc6i" double[n]; "force" double[n,3] (hartree/bohr); "energy"
 * double[B]; "sigma" double[B,6]; "order" int32[n] (sorted position -> caller's atom index); "type" int32[n] (after
 * s7b_d3_set_system_batch: Z - 1 | local type << 8, the local type being the rank of Z among the elements of the
 * atom's structure; after s7b_d3_set_system: the type index).  B = 1 after
 * s7b_d3_set_system.  Stage 2 sets energy / sigma to the pair sums of its range, stage 3 adds its virial. */
S7B_API void* s7b_d3_buffer(S7bD3* d3, const char* name, size_t* numel);
/* energy (eV), forces [n,3] (eV/A, caller's atom order), sigma6 (eV: xx,yy,zz,xy,xz,yz of sum f (x) r); one structure */
S7B_API int s7b_d3_results_host(S7bD3* d3, double* energy, double* forces, double* sigma6, void* stream);
S7B_API int s7b_d3_compute_host(S7bD3* d3, double* energy, double* forces, double* sigma6, void* stream);

/* Batches.  The full element tables, rows indexed by Z - 1: rcov [94], r2r4 [94], r0ab [94*94] (Angstrom),
 * c6ref [94*94*25], cnref [94*5], mxc [94].  Uploaded once per handle. */
S7B_API int s7b_d3_set_element_tables(S7bD3* d3, const double* rcov, const double* r2r4, const double* r0ab,
                                      const double* c6ref, const double* cnref, const int32_t* mxc);
/* B structures in one pass: atoms of structure b are [atom_ptr[b], atom_ptr[b+1]) (host, [B+1]); d_numbers (device
 * int32 [n], atomic numbers 1..94) and d_positions (device double [n,3], Angstrom) stay on the device; cells9 (host
 * double [B,9], rows) and pbc3 (host int32 [B,3]).  Every structure has its own cell list, wrap and local element
 * types (at most 16 elements per structure, any number in the batch).  Empty structures are allowed and give zeros.
 * An atomic number outside 1..94, more than 16 elements in a structure, a singular cell or a decreasing atom_ptr is
 * refused with a message naming the structure, before the current system is touched.  One small readback.  Then run
 * the three stages over [0, n). */
S7B_API int s7b_d3_set_system_batch(S7bD3* d3, int32_t n_systems, const int32_t* atom_ptr, const int32_t* d_numbers,
                                    const double* d_positions, const double* cells9, const int32_t* pbc3, void* stream);
/* After the three stages over [0, n): energy [B] (eV), forces [n,3] (eV/A, caller's atom order) and virial [B,6]
 * (eV; xx,yy,zz,xy,yz,zx of -sum r (x) dE/dr, the order and sign of s7b_engine_system_results, so the two add), fp64
 * device pointers, no synchronisation.  Per-structure sums in a fixed order: deterministic, and independent of the
 * other structures of the batch. */
S7B_API int s7b_d3_system_results(S7bD3* d3, double* d_energy, double* d_forces, double* d_virial, void* stream);

/* The reference's own D3 entry points (pair_d3_for_ase.cu:2034-2082; ctypes signatures sevenn/calculator.py:430-483),
 * same names / arguments / call order, so its D3Calculator can load this library in place of pair_d3.so.
 * Tables: weights/d3_params.bin next to the repository's library, or $S7B_D3_PARAMS. */
S7B_API S7bD3* pair_init(void);
S7B_API void pair_set_atom(S7bD3* pair, int natoms, int ntypes, int* type, double* x_flat);
S7B_API void pair_set_domain(S7bD3* pair, int xperiodic, int yperiodic, int zperiodic, double* boxlo, double* boxhi,
                             double xy, double xz, double yz);
S7B_API void pair_run_settings(S7bD3* pair, double rthr, double cnthr, const char* damp_name, const char* func_name);
S7B_API void pair_run_coeff(S7bD3* pair, int* atomic_numbers);
S7B_API void pair_run_compute(S7bD3* pair);
S7B_API double pair_get_energy(S7bD3* pair);
S7B_API double* pair_get_force(S7bD3* pair);
S7B_API double* pair_get_stress(S7bD3* pair);
S7B_API void pair_fin(S7bD3* pair);

#ifdef __cplusplus
}
#endif
#endif /* SEVENN_B200_H */
