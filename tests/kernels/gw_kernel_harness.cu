// gw_kernel_harness.cu -- test-only shim over the internal launchers of libgwb200.so (tests/test_gpu_kernels.py,
// tests/test_gpu_wide_training.py, tests/test_gpu_chunk_primitives.py).
//
// Host code only: flat extern "C" wrappers that the kernel tests call through ctypes, so that every CUDA primitive of the
// training step, the forward's CUDA-core row ops and helpers, and the device-built graphs (tests/test_gpu_forward_simt.py,
// tests/test_gpu_graph_kernels.py) can be run on its own and compared with a float64 or host reference.  The row sources cross the boundary as the
// harness's own POD (HSrc / HOp below), never as gw::RowSrc / gw::TcChain, so the tests do not depend on their layout.  Every
// wrapper enqueues on the caller's stream and returns the CUDA error code (cudaErrorInvalidValue from a launcher that does not
// take a shape is passed through unchanged).  Built by the test into a temporary directory and linked against the package's
// libgwb200.so with --no-undefined: a renamed or re-typed launcher fails at link time.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../graph_weather_b200/csrc/gw_internal.h"

using namespace gw;

extern "C" {

struct HSrc {  // one row source: kind = gw::SrcKind (0 none, 1 stream, 2 bcast, 3 gather, 4 segsum, 5 relu(gather + bcast), 6 bgather)
  int32_t kind, width, ld, col0;
  const float* base;
  int32_t src_rows;
  const int32_t* idx;
  const float* base2;  // kind 5: the broadcast table (ld2)
  int32_t ld2;
  const int32_t* bound_mul_i;  // h_chain: the source's bound is multiplied by this device integer (a sum of up to that many rows)
  const int32_t* ptr;          // kind 4: CSR [rows + 1] over the summed table's rows
  const int32_t* perm;         // kind 4: optional row permutation (null: rows in CSR order)
};

struct HOp {  // one training row op: out = mask(residual + LN(relu(concat(a) . W^T + bias + add)))
  int32_t rows, batch;
  HSrc a[2];
  const float* W;
  int32_t K, N, ldw;
  const float* bias;
  HSrc add[2];
  int32_t relu;
  const float* ln_g;
  const float* ln_b;
  HSrc residual;
  float* out;
  int32_t ldo;
  float* save_pre;
  HSrc mask;
};

struct HLayer {  // one forward chain layer: out = residual + LN(relu(A . W^T + bias + add)), fp32 W [N, ldw] with K real inputs
  const float* W;
  int32_t K, N, ldw;
  const float* bias;
  HSrc add[2];
  int32_t relu;
  const float* ln_g;
  const float* ln_b;
  HSrc residual;
  float* out;
  int32_t ldo, out_cols, feeds_next, reuse_a;
  const int32_t* seg_dst;  // fused per-target sums (gw::TcLayer::seg_*)
  float* seg_out;
  int32_t seg_ld, seg_rows, seg_maxdeg;
  const float* seg_add;    // [seg_rows, seg_ld]
  float* out_bound;        // device floats the chain sets (may be null)
  float* seg_bound;
};

struct HChain {  // one inference chain as gw_forward.cu builds it
  int32_t rows, batch, K0, n_layers;
  HSrc a0[2];
  HLayer layer[6];
  int32_t out_mode, n_out_peers;  // out_mode 2: the last layer stores through out_peer[j] instead of its own out
  float* out_peer[3];
};

}  // extern "C"

namespace {

RowSrc row_src(const HSrc& h) {
  RowSrc s;
  s.kind = h.kind, s.width = h.width, s.ld = h.ld, s.col0 = h.col0, s.base = h.base, s.src_rows = h.src_rows, s.idx = h.idx;
  s.base2 = h.base2, s.ld2 = h.ld2, s.ptr = h.ptr, s.perm = h.perm;
  return s;
}

// device temporaries of one wrapper call, freed in stream order when it returns
struct Temps {
  cudaStream_t st;
  std::vector<void*> p;
  explicit Temps(cudaStream_t s) : st(s) {}
  ~Temps() {
    for (void* q : p) cudaFreeAsync(q, st);
  }
  template <class T>
  cudaError_t get(T** out, size_t n) {
    void* q = nullptr;
    const cudaError_t e = cudaMallocAsync(&q, n * sizeof(T) + 16, st);
    if (e != cudaSuccess) return e;
    p.push_back(q);
    *out = static_cast<T*>(q);
    return cudaSuccess;
  }
};

#define H_TRY(expr)                          \
  do {                                       \
    const cudaError_t _e = (expr);           \
    if (_e != cudaSuccess) return (int)_e;   \
  } while (0)

}  // namespace

extern "C" {

int h_sizeof_src() { return (int)sizeof(HSrc); }
int h_sizeof_op() { return (int)sizeof(HOp); }
int h_sizeof_layer() { return (int)sizeof(HLayer); }
int h_sizeof_chain() { return (int)sizeof(HChain); }

// dW[o, k] (ld ldw) += sum_r dY[r, o] A(r, k), db[o] += sum_r dY[r, o] (db may be null), on tensor cores; workspace sized here
int h_wgrad_tc(int split, const float* dY, int ldy, int N, const HSrc* a, int K, int rows, int batch, float* dW, int ldw, float* db, int32_t* status,
               void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  Temps t(st);
  const size_t n = wgrad_tc_workspace_floats((long long)rows * batch, N, K);
  float* ws = nullptr;
  H_TRY(t.get(&ws, n));
  return (int)launch_wgrad_tc(dY, ldy, N, row_src(*a), K, rows, batch, dW, ldw, db, split != 0, ws, n, status, st);
}

// the same on CUDA cores (exact fp32 products, float atomics across row slabs)
int h_wgrad_simt(const float* dY, int ldy, int N, const HSrc* a, int K, int rows, int batch, float* dW, int ldw, float* db, void* stream) {
  return (int)launch_wgrad(dY, ldy, N, row_src(*a), K, rows, batch, dW, ldw, db, (cudaStream_t)stream);
}

// One training row op of any N.  precision 0: fp32_simt (gw_simt.cu); 1: fp32 (fp16 hi/lo, 3 MMAs); 2: bf16.  The tensor-core
// precisions run it as the training step does (gw_train.cu, train_op): the chain of tc_row_op_chain, its stage-0 sources bounded
// by launch_operand_bound (fp32), cut by tc_column_block into blocks of at most TC_COL_BLOCK output columns, each with the image of
// its rows of W from launch_pack_image.  *lean: bit j = column block j takes the lean path (-1 for fp32_simt).
int h_row_op(int precision, const HOp* h, int* lean, int32_t* status, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  GemmOp op;
  op.rows_per_sample = h->rows, op.batch = h->batch;
  op.a[0] = row_src(h->a[0]), op.a[1] = row_src(h->a[1]);
  op.W = h->W, op.K = h->K, op.N = h->N, op.ldw = h->ldw, op.bias = h->bias;
  op.add[0] = row_src(h->add[0]), op.add[1] = row_src(h->add[1]);
  op.relu = h->relu, op.ln_gamma = h->ln_g, op.ln_beta = h->ln_b, op.residual = row_src(h->residual);
  op.out = h->out, op.ldo = h->ldo, op.save_pre = h->save_pre, op.mask = row_src(h->mask);
  if (lean) *lean = -1;
  if (precision == 0) return (int)launch_rowop_simt(op, st);
  if (precision != 1 && precision != 2) return (int)cudaErrorInvalidValue;
  const bool split = precision == 1;
  const int parts = split ? 2 : 1;
  TcChain ch;
  H_TRY(tc_row_op_chain(op, &ch));
  ch.split = split ? 1 : 0, ch.status = status;
  Temps t(st);
  float* bounds = nullptr;
  H_TRY(t.get(&bounds, 2));
  H_TRY(cudaMemsetAsync(bounds, 0, 2 * sizeof(float), st));
  if (split)
    for (int a = 0; a < 2; ++a)
      if (ch.a0[a].kind != SRC_NONE) H_TRY(launch_operand_bound(ch.a0[a], op.rows_per_sample, op.batch, bounds + a, st));
  if (lean) *lean = 0;
  for (int n0 = 0, j = 0; n0 < op.N; n0 += TC_COL_BLOCK, ++j) {
    const int nb = std::min(TC_COL_BLOCK, op.N - n0);
    TcChain blk;
    H_TRY(tc_column_block(ch, n0, nb, &blk));
    unsigned char* img = nullptr;
    float* wamax = nullptr;
    H_TRY(t.get(&img, tc_packed_bytes(op.K, nb, parts)));
    H_TRY(t.get(&wamax, 1));
    H_TRY(launch_pack_image(op.W + (size_t)n0 * op.ldw, op.ldw, op.K, nb, parts, img, wamax, st));
    blk.layer[0].Wp = img, blk.layer[0].wamax = wamax;
    if (lean && tc3_chain_is_lean(blk)) *lean |= 1 << j;
    H_TRY(launch_chain_tc3(blk, st));
  }
  return 0;
}

// One inference chain (precision 1: fp32, 2: bf16), prepared as gw_forward.cu prepares it: every weight image described by tc_weights
// of its device absmax and packed with that scale, off = max|bias|, ln_bound = tc_ln_bound of the LayerNorm parameters' absmax,
// and every source bounded by the absmax of its whole table (launch_absmax_flat).  A layer with fused per-target sums
// gets a carry buffer (prefilled with NaN: a carry row read before it is written poisons the sum), and gw_seg_carry_kernel runs
// after the chain, as in stage_processor / stage_decoder.  *lean: tc3_chain_is_lean.
int h_chain(int precision, const HChain* h, int* lean, int32_t* status, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  if (lean) *lean = -1;
  if ((precision != 1 && precision != 2) || h->n_layers < 1 || h->n_layers > 6 || h->n_out_peers < 0 || h->n_out_peers > 3)
    return (int)cudaErrorInvalidValue;
  const bool split = precision == 1;
  const int parts = split ? 2 : 1, nl = h->n_layers;
  Temps t(st);
  // device maxima: per layer {W, bias, gamma, beta}, then one slot per source
  constexpr int NSLOT = 64;
  float* mx = nullptr;
  H_TRY(t.get(&mx, NSLOT));
  H_TRY(cudaMemsetAsync(mx, 0, NSLOT * sizeof(float), st));
  int next = 24;
  auto vmax = [&](const float* v, int n, float* slot) { return v ? launch_absmax(v, n, n, 1, slot, st) : cudaSuccess; };
  auto bounded = [&](const HSrc& hs, RowSrc& s) -> cudaError_t {
    s = row_src(hs);
    if (s.kind == SRC_NONE) return cudaSuccess;
    const bool per_sample = s.kind == SRC_STREAM || s.kind == SRC_GATHER || s.kind == SRC_GATHER_BCAST_RELU;
    const long long table_rows = per_sample ? (long long)h->batch * s.src_rows : (s.kind == SRC_BGATHER ? s.src_rows : h->rows);
    s.bound = mx + next++, s.bound_mul = 1.f, s.bound_mul_i = hs.bound_mul_i;
    cudaError_t e = launch_absmax_flat(s.base, table_rows * s.ld, mx + next - 1, st);
    if (e == cudaSuccess && s.kind == SRC_GATHER_BCAST_RELU) {
      s.bound2 = mx + next++;
      e = launch_absmax_flat(s.base2, (long long)h->rows * s.ld2, mx + next - 1, st);
    }
    return e;
  };
  TcChain ch;
  ch.rows_per_sample = h->rows, ch.batch = h->batch, ch.K0 = h->K0, ch.n_layers = nl, ch.split = split ? 1 : 0, ch.status = status;
  for (int a = 0; a < 2; ++a) H_TRY(bounded(h->a0[a], ch.a0[a]));
  int seg_layer = -1;
  for (int l = 0; l < nl; ++l) {
    const HLayer& H = h->layer[l];
    TcLayer& L = ch.layer[l];
    H_TRY(launch_absmax(H.W, H.ldw, H.K, H.N, mx + 4 * l, st));
    H_TRY(vmax(H.bias, H.N, mx + 4 * l + 1));
    H_TRY(vmax(H.ln_g, H.N, mx + 4 * l + 2));
    H_TRY(vmax(H.ln_b, H.N, mx + 4 * l + 3));
    for (int a = 0; a < 2; ++a) H_TRY(bounded(H.add[a], L.add[a]));
    H_TRY(bounded(H.residual, L.residual));
    if (H.seg_add) {
      L.seg_add_bound = mx + next++;
      H_TRY(launch_absmax_flat(H.seg_add, (long long)H.seg_rows * H.seg_ld, mx + next - 1, st));
    }
    if (H.seg_dst) seg_layer = l;
  }
  if (next > NSLOT) return (int)cudaErrorInvalidValue;
  float hm[24];
  H_TRY(cudaMemcpyAsync(hm, mx, sizeof(hm), cudaMemcpyDeviceToHost, st));
  H_TRY(cudaStreamSynchronize(st));
  for (int l = 0; l < nl; ++l) {
    const HLayer& H = h->layer[l];
    TcLayer& L = ch.layer[l];
    unsigned char* img = nullptr;
    H_TRY(t.get(&img, tc_packed_bytes(H.K, H.N, parts)));
    const TcWeights w = tc_weights(img, H.K, H.N, hm[4 * l], parts);
    H_TRY(launch_pack_weights(H.W, H.ldw, H.K, H.N, 1.f / w.winv, parts, img, st));
    L.Wp = w.p, L.K = w.K, L.N = w.N, L.N32 = w.N32, L.n_valid = w.n_valid, L.wscale_inv = w.winv, L.gain = w.gain, L.off = hm[4 * l + 1];
    L.bias = H.bias, L.relu = H.relu, L.ln_g = H.ln_g, L.ln_b = H.ln_b;
    if (H.ln_g) L.ln_bound = tc_ln_bound(H.N, hm[4 * l + 2], hm[4 * l + 3]);
    L.out = H.out, L.ldo = H.ldo, L.out_cols = H.out_cols, L.out_bound = H.out_bound;
    L.feeds_next = H.feeds_next, L.reuse_a = H.reuse_a;
    L.seg_dst = H.seg_dst, L.seg_out = H.seg_out, L.seg_ld = H.seg_ld, L.seg_rows = H.seg_rows, L.seg_maxdeg = (float)H.seg_maxdeg;
    L.seg_add = H.seg_add, L.seg_bound = H.seg_bound;
  }
  ch.out_mode = h->out_mode, ch.n_out_peers = h->n_out_peers;
  for (int j = 0; j < h->n_out_peers; ++j) ch.out_peer[j] = h->out_peer[j];
  float* carry = nullptr;
  const int tiles = (h->rows + 127) / 128;
  if (seg_layer >= 0) {
    const size_t n = (size_t)h->batch * tiles * 8 * 256;
    H_TRY(t.get(&carry, n));
    H_TRY(cudaMemsetAsync(carry, 0xff, n * sizeof(float), st));
    ch.layer[seg_layer].seg_carry = carry;
  }
  if (lean) *lean = tc3_chain_is_lean(ch) ? 1 : 0;
  H_TRY(launch_chain_tc3(ch, st));
  if (seg_layer >= 0) {
    const HLayer& H = h->layer[seg_layer];
    H_TRY(launch_seg_carry(carry, H.seg_dst, h->rows, H.seg_rows, h->batch, H.seg_out, H.seg_ld, st));
  }
  return 0;
}

int h_ln_bwd(const float* dy, int ld_dy, const float* z, int ld_z, int N, const float* gamma, long long R, float* dz, int ld_dz, float* dgamma,
             float* dbeta, void* stream) {
  return (int)launch_ln_bwd(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta, (cudaStream_t)stream);
}

int h_segsum(const float* base, int ld, int width, const int32_t* ptr, const int32_t* perm, int src_rows, int rows, int batch, float* out, int ldo,
             void* stream) {
  return (int)launch_segsum(base, ld, width, ptr, perm, src_rows, rows, batch, out, ldo, (cudaStream_t)stream);
}

// the two-level segment sum (256-wide rows): chunk table built on the device from ptr, then the chunk and finish kernels;
// n_src_rows = ptr[rows] (the row count the chunk table is sized for)
int h_segsum_chunked(const float* base, int ld, const int32_t* ptr, const int32_t* perm, int src_rows, int rows, int n_src_rows, int batch,
                     float* out, int ldo, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  Temps t(st);
  const int max_chunks = seg_chunk_bound(rows, n_src_rows);
  int32_t *chunk_seg = nullptr, *chunk_j0 = nullptr, *seg_chunk0 = nullptr;
  float* partial = nullptr;
  H_TRY(t.get(&chunk_seg, max_chunks));
  H_TRY(t.get(&chunk_j0, max_chunks));
  H_TRY(t.get(&seg_chunk0, (size_t)rows + 1));
  H_TRY(t.get(&partial, (size_t)batch * max_chunks * 256));
  H_TRY(launch_seg_chunks(ptr, rows, chunk_seg, chunk_j0, seg_chunk0, st));
  return (int)launch_segsum_chunked(base, ld, ptr, perm, src_rows, rows, batch, chunk_seg, chunk_j0, seg_chunk0, max_chunks, partial, out, ldo, st);
}

int h_batch_reduce(const float* in, int ld_in, long long rows, int width, int batch, float* out, int ld_out, int accumulate, void* stream) {
  return (int)launch_batch_reduce(in, ld_in, rows, width, batch, out, ld_out, accumulate != 0, (cudaStream_t)stream);
}

int h_gather_rows(const float* in, int ld_in, int src_rows, const int32_t* idx, long long rows, int width, int batch, float* out, int ld_out,
                  int accumulate, void* stream) {
  return (int)launch_gather_rows(in, ld_in, src_rows, idx, rows, width, batch, out, ld_out, accumulate != 0, (cudaStream_t)stream);
}

// ---- the bounded-memory step's row movement (gw_train.cu: build_chunks, enc_fwd / enc_bwd / enc_node_bwd, dec_fwd / dec_bwd) ----
// launch_segsum over a CSR slice whose entries start at ptr_base, optionally adding to what out holds (tests/test_gpu_chunk_primitives.py)
int h_segsum_range(const float* base, int ld, int width, const int32_t* ptr, const int32_t* perm, int src_rows, int rows, int batch, float* out,
                   int ldo, int ptr_base, int accumulate, void* stream) {
  return (int)launch_segsum(base, ld, width, ptr, perm, src_rows, rows, batch, out, ldo, (cudaStream_t)stream, ptr_base, accumulate != 0);
}

// launch_gather_rows from a table that holds the targets idx_base .. idx_base + src_rows - 1 only
int h_gather_rows_base(const float* in, int ld_in, int src_rows, const int32_t* idx, long long rows, int width, int batch, float* out, int ld_out,
                       int accumulate, int idx_base, void* stream) {
  return (int)launch_gather_rows(in, ld_in, src_rows, idx, rows, width, batch, out, ld_out, accumulate != 0, (cudaStream_t)stream, idx_base);
}

// scatter 0: out row (b, j) = in row (b, idx[j]) of other_rows per sample; scatter 1: out row (b, idx[j]) = in row (b, j)
int h_permute_rows(const float* in, int ld_in, const int32_t* idx, long long rows, int other_rows, int width, int batch, float* out, int ld_out,
                   int scatter, void* stream) {
  return (int)launch_permute_rows(in, ld_in, idx, rows, other_rows, width, batch, out, ld_out, scatter != 0, (cudaStream_t)stream);
}

// dst[r, c] += src[r, c] for c < width
int h_strided_add(const float* src, int ld_src, float* dst, int ld_dst, long long rows, int width, void* stream) {
  return (int)launch_strided_add(src, ld_src, dst, ld_dst, rows, width, (cudaStream_t)stream);
}

int h_transpose(const float* W, int rows, int cols, float* WT, void* stream) {
  return (int)launch_transpose(W, rows, cols, WT, (cudaStream_t)stream);
}

// ---- the forward's small helpers (gw_simt.cu) and the device-built graphs (gw_graph.cu) ---------------------------------------
// dst[r, :] = [src[r, 0:width], 0 ...] over ld_dst columns; *amax = max(*amax, max |src|) (amax may be null)
int h_pad_rows(const float* src, int ld_src, int width, float* dst, int ld_dst, long long rows, float* amax, void* stream) {
  return (int)launch_pad_rows(src, ld_src, width, dst, ld_dst, rows, amax, (cudaStream_t)stream);
}

// *amax = max(*amax, max |p[0..n)|)
int h_absmax_flat(const float* p, long long n, float* amax, void* stream) { return (int)launch_absmax_flat(p, n, amax, (cudaStream_t)stream); }

// dst[j] = i for ptr[i] <= j < ptr[i + 1] (dst may be null); stats = {max(stats[0], longest segment), min(stats[1], shortest)}
int h_csr_expand(const int32_t* ptr, int n, int32_t* dst, int* stats, void* stream) {
  return (int)launch_csr_expand(ptr, n, dst, stats, (cudaStream_t)stream);
}

// perm = the row ids ordered by src (ties in row order), ptr[s] = first position of slot s (s = 0 .. n_slots); workspace sized here
int h_sort_csr(const int32_t* src, int n, int n_slots, int32_t* perm, int32_t* ptr, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  Temps t(st);
  const size_t nb = sort_csr_workspace_bytes(n);
  unsigned char* ws = nullptr;
  H_TRY(t.get(&ws, nb));
  return (int)launch_sort_csr(src, n, n_slots, perm, ptr, ws, nb, st);
}

// The observation graph of n points llh [n, 3] (lat deg, lon deg, height): the arrays of h3lite.device_tables(res) as device
// pointers (gw_plan_set_h3_tables), cell_slot = H - 1 - rank; slot [n], perm [n], ptr [n_slots + 1], attr [n, 3]; workspace sized here
int h_obs_graph(int res, int n_cells, int lat_n, const double* frames, const int32_t* cell_of, const int32_t* cell_slot, const double* cell_lat,
                const double* cell_lng, double scale, double rot_cos, double rot_sin, const float* llh, int n, int n_slots, int32_t* slot,
                int32_t* perm, int32_t* ptr, float* attr, int32_t* status, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  H3Tables tab;
  tab.res = res, tab.n_cells = n_cells, tab.lat_n = lat_n;
  tab.frames = frames, tab.cell_of = cell_of, tab.cell_slot = cell_slot, tab.cell_lat = cell_lat, tab.cell_lng = cell_lng;
  tab.scale = scale, tab.cr = rot_cos, tab.sr = rot_sin;
  Temps t(st);
  const size_t nb = obs_graph_workspace_bytes(n);
  unsigned char* ws = nullptr;
  H_TRY(t.get(&ws, nb));
  return (int)launch_obs_graph(tab, llh, n, n_slots, slot, perm, ptr, attr, ws, nb, status, st);
}

}  // extern "C"
