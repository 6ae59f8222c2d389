// gw_internal.h -- declarations shared by the translation units of libgwb200.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <string>

#include "gw_ops.h"

namespace gw {

// grid-stride kernels launch a fixed number of blocks per SM of an H100 SXM (132 SMs)
constexpr int GRID_SMS = 132;

void count_launch(int n = 1);
void set_error(const std::string& msg);

// exact-fp32 CUDA-core execution of one row op (gw_simt.cu)
cudaError_t launch_rowop_simt(const GemmOp& op, cudaStream_t stream);
// The LayerNorm of a row op whose rows another kernel left in op.out as the value entering it: out = residual + LN(out) in place
// over op.N columns (eps 1e-5, two passes like torch).  amax (optional, zeroed by the caller): *amax = max(*amax, max |out|), inf
// if a row is not finite.
cudaError_t launch_ln_rows(const GemmOp& op, float* amax, cudaStream_t stream);

cudaError_t launch_pad_rows(const float* src, int ld_src, int width, float* dst, int ld_dst, long long rows, float* amax, cudaStream_t stream);
cudaError_t launch_absmax_flat(const float* p, long long n, float* amax, cudaStream_t stream);
cudaError_t launch_csr_expand(const int32_t* ptr, int n, int32_t* dst, int* stats, cudaStream_t stream);
// backward primitives (gw_simt.cu)
cudaError_t launch_wgrad(const float* dY, int ldy, int N, const RowSrc& a, int K, int rows_per_sample, int batch, float* dW, int ldw, float* db,
                         cudaStream_t st);
cudaError_t launch_ln_bwd(const float* dy, int ld_dy, const float* z, int ld_z, int N, const float* gamma, long long R, float* dz, int ld_dz,
                          float* dgamma, float* dbeta, cudaStream_t st);
constexpr int LN_BWD_MAX_N = 1024;  // widest row launch_ln_bwd takes (rows of more than 256 columns run on a kernel of their own)
// Fixed-order variants of the two (gw_train_set_deterministic): the same per-slab / per-CTA sums, stored as partials in a
// workspace and added in an order that follows from the shapes alone, so that every run gives the same bits.  The workspace
// stays within DET_WS_BYTES: launch_wgrad_det cuts fewer row slabs for wide weights (one slab's tile fits for K < 32767), and
// launch_ln_bwd_det needs 2 x (its grid, at most 8 GRID_SMS) x N floats, 8.7 MB at N = 1024.  ws_floats below the
// *_workspace_floats of the shapes: cudaErrorInvalidValue.
constexpr size_t DET_WS_BYTES = size_t(32) << 20;
size_t wgrad_det_workspace_floats(long long R, int N, int K);
cudaError_t launch_wgrad_det(const float* dY, int ldy, int N, const RowSrc& a, int K, int rows_per_sample, int batch, float* dW, int ldw, float* db,
                             float* ws, size_t ws_floats, cudaStream_t st);
size_t ln_bwd_det_workspace_floats(long long R, int N);
cudaError_t launch_ln_bwd_det(const float* dy, int ld_dy, const float* z, int ld_z, int N, const float* gamma, long long R, float* dz, int ld_dz,
                              float* dgamma, float* dbeta, float* ws, size_t ws_floats, cudaStream_t st);
cudaError_t launch_batch_reduce(const float* in, int ld_in, long long rows, int width, int batch, float* out, int ld_out, bool accumulate,
                                cudaStream_t st);
// idx_base: `in` holds the targets idx_base .. idx_base + src_rows - 1 only (a chunk of the training step's grid-sized stages).
// Any width and strides: float4 where they and both pointers allow it, one float per thread otherwise.
cudaError_t launch_gather_rows(const float* in, int ld_in, int src_rows, const int32_t* idx, long long rows, int width, int batch, float* out,
                               int ld_out, bool accumulate, cudaStream_t st, int idx_base = 0);
// rows through a permutation, per sample: gather (out row j = in row idx[j] of other_rows) or scatter (out row idx[j] of other_rows = in row j)
cudaError_t launch_permute_rows(const float* in, int ld_in, const int32_t* idx, long long rows, int other_rows, int width, int batch, float* out,
                                int ld_out, bool scatter, cudaStream_t st);
cudaError_t launch_strided_add(const float* src, int ld_src, float* dst, int ld_dst, long long rows, int width, cudaStream_t st);
cudaError_t launch_transpose(const float* W, int rows, int cols, float* WT, cudaStream_t st);
int seg_chunk_bound(int n_seg, int n_rows);
cudaError_t launch_seg_chunks(const int32_t* ptr, int n_seg, int32_t* chunk_seg, int32_t* chunk_j0, int32_t* seg_chunk0, cudaStream_t st);
cudaError_t launch_segsum_chunked(const float* base, int ld, const int32_t* ptr, const int32_t* perm, int src_rows, int rows, int batch,
                                  const int32_t* chunk_seg, const int32_t* chunk_j0, const int32_t* seg_chunk0, int max_chunks, float* partial,
                                  float* out, int ldo, cudaStream_t st);
cudaError_t launch_seg_carry(const float* carry, const int32_t* seg_dst, int rows, int seg_rows, int batch, float* out, int ldo,
                             cudaStream_t stream);
// ptr_base: subtracted from every ptr entry (a CSR slice over a range of rows that starts at row ptr_base of the full table);
// accumulate: out += the segment sums (a per-segment sum split over row ranges, added in the order of the calls).  Any width and
// strides: float4 where they and both pointers allow it, one float per thread otherwise, summing each column in the same order.
cudaError_t launch_segsum(const float* base, int ld, int width, const int32_t* ptr, const int32_t* perm, int src_rows,
                          int rows, int batch, float* out, int ldo, cudaStream_t stream, int ptr_base = 0, bool accumulate = false);

// wgmma chain kernel (gw_tc3.cu)
cudaError_t launch_chain_tc3(const TcChain& ch, cudaStream_t stream);
bool tc3_chain_is_lean(const TcChain& ch);  // would the launch take the lean (perm32, 256-bit access) path?
// A one-layer chain computes at most TC_COL_BLOCK output columns.  Wider row ops (the training step's data gradient into the
// features and the decoder's output layer; every layer of a trunk wider than 256 on a layer-by-layer plan) run as column blocks
// (gw_forward.cu, tc_row_op): tc_column_block turns the layer of `ch`, which describes all its
// outputs, into the chain of columns n0 .. n0 + nb - 1 (bias, addends, residual, mask, pre-LayerNorm store and output shifted
// by n0 columns; stage-0 sources and their bounds shared).  The caller sets the block's weight image (W rows n0 .. n0 + nb - 1).
// A layer with a LayerNorm cannot be split: cudaErrorInvalidValue.
constexpr int TC_COL_BLOCK = 256;
cudaError_t tc_column_block(const TcChain& ch, int n0, int nb, TcChain* out);
// The one-layer chain of a training row op (gw_train.cu, train_op): stage 0 = op.a with K0 = K rounded to 64, layer 0 = the op's
// bias, addends, ReLU, LayerNorm, residual, output, pre-LayerNorm store and mask over all N columns -- the `ch` tc_column_block
// cuts into the blocks that run.  It sets no operand bounds, weight image, split or status.  cudaErrorInvalidValue for an op no
// chain runs: an add[2] addend, no a[0], or a LayerNorm wider than TC_COL_BLOCK.
cudaError_t tc_row_op_chain(const GemmOp& op, TcChain* ch);
// fp32-mode bound of a training row op's stage-0 source s: *amax (zeroed by the caller) takes the absmax of the whole tensor s
// reads (batch x src_rows rows of a stream, rows_per_sample rows of a broadcast), and s is bounded by it.  Sources of another
// kind: cudaErrorInvalidValue.
cudaError_t launch_operand_bound(RowSrc& s, int rows_per_sample, int batch, float* amax, cudaStream_t st);
// Packs W[n, k] (n < N_src rows of stride ldw, k < K_src) into the GMMA operand image the chain kernel streams with
// cp.async.bulk (perm32 feature order, gw_pack.cu); `parts` = 2 (fp16 hi, lo) or 1 (bf16).  dst must hold tc_packed_bytes(K_src, N_src, parts).
size_t tc_packed_bytes(int K_src, int N_src, int parts);
int tc_packed_rows(int N_src);  // rows of the packed image: N padded to 64
// amax_dev (optional): device max|W|; the scale is then tc_weight_scale(*amax_dev, parts), taken on the device (training images,
// repacked every step without a host round trip) instead of `wscale`.
cudaError_t launch_pack_weights(const float* W, int ldw, int K_src, int N_src, float wscale, int parts, void* dst, cudaStream_t stream,
                                const float* amax_dev = nullptr);
cudaError_t launch_absmax(const float* W, int ldw, int K_src, int N_src, float* out_max, cudaStream_t stream);
// The training step's image of W, scale taken on the device: *wamax = max|W| (reset first), then the pack.  A chain layer given
// this image takes wamax as its TcLayer::wamax.
cudaError_t launch_pack_image(const float* W, int ldw, int K_src, int N_src, int parts, void* img, float* wamax, cudaStream_t stream);
// A weight image packed with a scale the host chose from max|W| (the inference plans' images, gw_forward.cu): what its chain layer
// needs to know of it.  Pack it with wscale = 1 / winv (a power of two: exact).
struct TcWeights {
  const void* p = nullptr;
  int K = 0, N = 0, N32 = 0, n_valid = 0;  // TcLayer::K (K_src rounded to 64), N (N_src rounded to 16), N32, n_valid (N_src)
  float winv = 1.f;                        // TcLayer::wscale_inv
  float gain = 0.f;                        // K_src * max|W|: |A.W^T| <= gain * max|A|
};
TcWeights tc_weights(const void* img, int K_src, int N_src, float wamax, int parts);
// bound of a LayerNorm'd row of N real columns (n_valid, not the padded width): sqrt(N) max|gamma| + max|beta|, since a
// normalised row has sum x^2 <= N
float tc_ln_bound(int N, float gamma_amax, float beta_amax);
// Power of two a weight image is stored times: fp16 hi|lo images (parts 2) bring max|W| into [2048, 4096) so the lo parts stay
// normal (the host's pack_tc_weights uses the same rule); bf16 images are not scaled.
__host__ __device__ inline float tc_weight_scale(float amax, int parts) {
  if (parts != 2 || !(amax > 0.f) || !(amax < 3.0e38f)) return 1.f;
  int e = 0;  // amax = f * 2^e, f in [0.5, 1)
#ifdef __CUDA_ARCH__
  e = (int)((__float_as_uint(amax) >> 23) & 0xffu) - 126;
#else
  uint32_t u;
  memcpy(&u, &amax, 4);
  e = (int)((u >> 23) & 0xffu) - 126;
#endif
  e = e < -100 ? -100 : e;  // (subnormal max: any scale that keeps the image finite)
  return ldexpf(1.f, 12 - e);
}

// weight gradient on tensor cores (gw_wgrad_tc.cu): dW[o, k] += sum_r dY[r, o] A(r, k), db[o] += sum_r dY[r, o], in a fixed order
// (per-CTA partials in `ws`, then one pass that sums them).  A: SRC_STREAM / SRC_BCAST.  split: fp16 hi/lo operands (3 MMAs per
// product, power-of-two scaled from the operands' absmax), else bf16.  Any N (128-row output blocks); K > 256 runs as blocks of
// 256 columns of A, one after the other through the same workspace.
size_t wgrad_tc_workspace_floats(long long R, int N, int K);
// dW[o, k] += sum_s part[s][o][k] (s ascending, part [S][N][K]), db[o] += sum_s part_b[s][o] (db null: none)
cudaError_t launch_wgrad_sum(const float* part, const float* part_b, int S, int N, int K, float* dW, int ldw, float* db, cudaStream_t st);
cudaError_t launch_wgrad_tc(const float* dY, int ldy, int N, const RowSrc& a, int K, int rows_per_sample, int batch, float* dW, int ldw, float* db,
                            bool split, float* ws, size_t ws_floats, int32_t* status, cudaStream_t st);

// device-side observation graph of the assimilator (gw_graph.cu)
struct H3Tables {
  int res = -1, n_cells = 0, lat_n = 0;  // lattice table covers a, b in [-lat_n, lat_n]
  const double* frames = nullptr;        // [20][9]: face centre c, in-plane unit vectors ex, ey
  const int32_t* cell_of = nullptr;      // [20][(2 lat_n + 1)^2]: canonical cell of lattice point (a, b) on the face, -1 if none
  const int32_t* cell_slot = nullptr;    // [n_cells]: mesh-node slot of the cell in the encoder's numbering (H - 1 - rank)
  const double* cell_lat = nullptr;      // [n_cells] radians (as the host path sees them: through degrees and back)
  const double* cell_lng = nullptr;
  double scale = 0.0, cr = 1.0, sr = 0.0;  // plane -> lattice scale; Class III rotation (cos, sin), identity for even res
};

size_t obs_graph_workspace_bytes(int n);
size_t sort_csr_workspace_bytes(int n);
cudaError_t launch_sort_csr(const int32_t* src, int n, int n_slots, int32_t* perm, int32_t* ptr, void* ws, size_t ws_bytes, cudaStream_t st);
cudaError_t launch_obs_graph(const H3Tables& t, const float* llh, int n, int n_slots, int32_t* slot, int32_t* perm, int32_t* ptr, float* attr,
                             void* ws, size_t ws_bytes, int32_t* status, cudaStream_t st);

}  // namespace gw
