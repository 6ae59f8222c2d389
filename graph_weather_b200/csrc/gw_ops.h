// gw_ops.h -- POD descriptors shared by the host plan and the kernels.
//
// Every stage of the encode-process-decode forward is a chain of "row ops":
//     out[r, :] = residual(r) + LN( relu( A(r, :) . W^T + bias + addends(r) ) )        (each part optional)
// over R = batch * rows_per_sample rows, where the A row and the addends are assembled on the fly from
// "row sources" (stream / broadcast-over-batch / gather by index / CSR segment sum / relu(gather+broadcast)).
// This is what lets the kernels skip the reference's materialised cat([x[row], x[col], e]) (graph_net_block.py:131),
// scatter_sum output (:188) and replicated edge tensors (encoder.py:206-218).
#pragma once
#include <stdint.h>

namespace gw {

enum SrcKind : int32_t {
  SRC_NONE = 0,
  SRC_STREAM = 1,      // base[(b*rows + i)*ld + col0 + k]                       per-sample rows
  SRC_BCAST = 2,       // base[i*ld + col0 + k]                                  same rows for every sample
  SRC_GATHER = 3,      // base[(b*src_rows + idx[i])*ld + col0 + k]              per-sample table, shared index
  SRC_SEGSUM = 4,      // sum_{j in [ptr[i],ptr[i+1])} base[(b*src_rows + eid(j))*ld + col0 + k], eid = perm ? perm[j] : j
  SRC_GATHER_BCAST_RELU = 5,  // relu(GATHER(base, idx) + base2[i*ld2 + k])     decoder edge layer-1, see gw_forward.cu
  SRC_BGATHER = 6,     // base[idx[i]*ld + col0 + k]                             batch-invariant table, gathered
};

struct RowSrc {
  int32_t kind = SRC_NONE;
  int32_t width = 0;     // number of columns this source contributes
  int32_t ld = 0;        // leading dimension of base (floats)
  int32_t col0 = 0;      // first column inside base rows
  const float* base = nullptr;
  const float* base2 = nullptr;  // SRC_GATHER_BCAST_RELU: broadcast table
  int32_t ld2 = 0;
  int32_t src_rows = 0;  // rows per sample of the gathered / summed table
  const int32_t* idx = nullptr;   // [rows_per_sample]
  const int32_t* ptr = nullptr;   // [rows_per_sample+1]
  const int32_t* perm = nullptr;  // optional edge permutation for SEGSUM
  const float* bound2 = nullptr;  // SRC_GATHER_BCAST_RELU: bound of base2
  float bound_mul = 1.f;          // the source's values are bounded by *bound * bound_mul (e.g. sums of up to bound_mul rows)
  const int32_t* bound_mul_i = nullptr;  // ... times this device integer when set (segment lengths known only on the device)
  const float* bound = nullptr;   // device float: |values of this source| <= *bound (null: unknown).  Tensor-core chains use it
                                  // to scale fp16-split operands into range (gw_tc3.cu, "operand range")
};

struct GemmOp {
  int32_t rows_per_sample = 0;
  int32_t batch = 0;
  RowSrc a[2];                 // A row = concat(a[0], a[1]); K = a[0].width + a[1].width
  const float* W = nullptr;    // [N, ldw] row-major (nn.Linear weight, possibly a column slice: pointer offset + ldw)
  int32_t K = 0, N = 0, ldw = 0;
  const float* bias = nullptr; // [N]
  RowSrc add[3];               // epilogue addends, each N wide
  int32_t relu = 0;
  const float* ln_gamma = nullptr;  // LayerNorm over the N outputs (eps 1e-5) if non-null
  const float* ln_beta = nullptr;
  RowSrc residual;             // added after LN
  float* out = nullptr;        // out[(b*rows + i)*ldo + n]
  int32_t ldo = 0;
  float* save_pre = nullptr;   // training: the value entering LayerNorm is also stored here (same ldo) -- LayerNorm's backward needs it
  RowSrc mask;                 // backward of ReLU: the result is kept where mask(row, n) > 0 and zeroed elsewhere (applied last)
};

// ---- tensor-core chain (gw_tc3.cu) -------------------------------------------------------------------------------
// A chain runs up to TC_MAX_LAYERS row ops back to back on one 128-row tile without leaving the SM: the result of a
// layer is split to fp16 hi/lo and written straight into the shared-memory A operand of the next layer.
constexpr int TC_MAX_LAYERS = 8;

struct TcLayer {
  const void* Wp = nullptr;   // packed weights (gw_pack.cu): [K/64][parts][N32 x 64] fp16/bf16, GMMA SW128 K-major, perm32 feature order
  int32_t K = 0, N = 0;       // K multiple of 64 (zero padded), N multiple of 16 (<= 256)
  int32_t N32 = 0;            // rows of the perm32 image (N padded to 64): the N the chain kernel runs this layer with
  int32_t n_valid = 0;        // real output columns (<= N); bias / LN parameters / addends exist only for these
  float wscale_inv = 1.f;     // weights are stored times a power of two; the accumulator is multiplied by this
  const float* bias = nullptr;
  RowSrc add[2];              // epilogue addends (SRC_BCAST / SRC_GATHER / SRC_STREAM), N wide
  int32_t relu = 0;
  const float* ln_g = nullptr;  // LayerNorm over N (eps 1e-5) if non-null
  const float* ln_b = nullptr;
  RowSrc residual;            // added after LN
  float* out = nullptr;       // fp32 result rows -> out[(b*rows+i)*ldo + n], n < out_cols (null: not stored)
  int32_t ldo = 0, out_cols = 0;
  int32_t feeds_next = 0;     // result becomes the A operand of the next layer
  int32_t reuse_a = 0;        // this layer multiplies the same A operand as the previous layer
  int32_t kind = -1;          // gw_tc3 launcher: epilogue feature mask if a specialised instance exists, else -1 (flags read at run time)
  // operand range (gw_tc3.cu): a rigorous magnitude bound travels with every tensor so that each fp16-split operand can be
  // scaled by a power of two into the fp16 range.  |A . W^T| <= gain * max|A| with gain = K * max|W|; off = max|bias|.
  float gain = 0.f, off = 0.f;
  float ln_bound = 0.f;       // LayerNorm layers: sqrt(N) * max|gamma| + max|beta| bounds the normalised row
  float* out_bound = nullptr; // device float the kernel sets to the bound of this layer's result (CTA 0), for `out` consumers
  // fused per-target sum of the result rows (graph_net_block.py:188 scatter_sum): rows are grouped by target (seg_dst
  // non-decreasing, segments of <= 8 rows); each segment sum goes to seg_out, the part of a segment behind a 16-row group
  // boundary (the rows one worker warp reduces) goes to seg_carry and is added by gw_seg_carry_kernel.
  const int32_t* seg_dst = nullptr;  // [rows_per_sample] target of every row
  float* seg_out = nullptr;          // [(b * seg_rows + target) * seg_ld + n]
  float* seg_carry = nullptr;        // [((b * tiles_per_sample + tile) * 8 + row group) * 256 + n]
  int32_t seg_ld = 0, seg_rows = 0;
  float seg_maxdeg = 0.f;            // longest segment (bound of the sums)
  float* seg_bound = nullptr;        // device float set to the bound of the segment sums
  const float* seg_add = nullptr;    // [seg_rows, seg_ld] or null: a per-target constant added to every complete sum (the sum of a
                                     // constant residual over the target's rows, hoisted out of the row loop: gw_forward.cu S_dec)
  const float* seg_add_bound = nullptr;  // device float: magnitude bound of seg_add
  // training step (gw_train.cu), general path only: the value entering LayerNorm is also stored to save_pre (same ldo / out_cols
  // as out; GemmOp::save_pre), and the result is zeroed wherever mask(row, n) <= 0 (the ReLU's backward, applied last; GemmOp::mask)
  float* save_pre = nullptr;
  RowSrc mask;
  const float* wamax = nullptr;  // device max|W| of an image packed with its scale taken on the device (launch_pack_weights with
                                 // amax_dev): the kernel derives wscale_inv and gain from it instead of the host fields
};

struct TcChain {
  int32_t rows_per_sample = 0, batch = 0;
  RowSrc a0[2];               // stage-0 operand = concat(a0[0], a0[1]) zero-padded to K0
  int32_t K0 = 0;             // multiple of 64
  int32_t n_layers = 0;
  int32_t split = 1;          // 1: fp16 hi+lo operands, 3 MMAs per product (fp32-faithful); 0: bf16 single MMA
  int32_t* status = nullptr;  // device word: bit0 = operand exceeded the fp16 range, bit1 = pipeline timeout
  long long* trace = nullptr; // optional debug timeline: [8 roles][1024 events][2] = {clock64, code}; CTA 0 only
  int32_t fast = 0;           // gw_tc3: bit l = layer l takes the lean full-width path, bit 31 = stage 0 does (set by the launcher)
  int32_t ablate = 0;         // diagnostics build only (-DGW_ABLATE): bit mask of pipeline parts to skip, for timing attribution
  // Loss-boundary gather fused into the chain that produces the forecast (multi-GPU; graph_weather_b200/dist.py): the LAST layer's
  // fp32 result rows are stored, tile by tile as they leave the accumulator, into the gather buffers of every GPU of the job --
  // out_mode 1: one multimem.st per value to the NVLink multicast alias of `out` (the switch replicates it to every GPU);
  // out_mode 2: one plain store per peer mapping.  The aliases address the same element as the layer's `out`.
  int32_t out_mode = 0, n_out_peers = 0;
  float* out_mc = nullptr;
  float* out_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  TcLayer layer[TC_MAX_LAYERS];
};

}  // namespace gw
