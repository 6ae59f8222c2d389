// gw_kernel_harness.cu -- test-only shim over the internal launchers of libgwb200.so (tests/test_gpu_kernels.py).
//
// Host code only: flat extern "C" wrappers that the kernel tests call through ctypes, so that every CUDA primitive of the
// training step can be run on its own and compared with a float64 reference.  The row sources cross the boundary as the
// harness's own POD (HSrc / HOp below), never as gw::RowSrc / gw::TcChain, so the tests do not depend on their layout.  Every
// wrapper enqueues on the caller's stream and returns the CUDA error code (cudaErrorInvalidValue from a launcher that does not
// take a shape is passed through unchanged).  Built by the test into a temporary directory and linked against the package's
// libgwb200.so with --no-undefined: a renamed or re-typed launcher fails at link time.
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "../../graph_weather_b200/csrc/gw_internal.h"

using namespace gw;

extern "C" {

struct HSrc {  // one row source: kind = gw::SrcKind (0 none, 1 stream, 2 bcast, 3 gather, 6 bgather)
  int32_t kind, width, ld, col0;
  const float* base;
  int32_t src_rows;
  const int32_t* idx;
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

}  // extern "C"

namespace {

RowSrc row_src(const HSrc& h) {
  RowSrc s;
  s.kind = h.kind, s.width = h.width, s.ld = h.ld, s.col0 = h.col0, s.base = h.base, s.src_rows = h.src_rows, s.idx = h.idx;
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

// One training row op.  precision 0: fp32_simt (gw_simt.cu); 1: fp32 (fp16 hi/lo, 3 MMAs); 2: bf16.  The tensor-core precisions
// build the one-layer chain the training step builds (gw_train.inl, train_op): weight image packed with its scale taken on the
// device, stage-0 sources bounded by their whole tensor's absmax (fp32), K0 rounded to 64, range_fit.  *lean: whether the chain
// takes the lean path (-1 for fp32_simt).
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
  Temps t(st);
  unsigned char* img = nullptr;
  float* wamax = nullptr;
  float* bounds = nullptr;
  H_TRY(t.get(&img, tc_packed_bytes(op.K, op.N, parts)));
  H_TRY(t.get(&wamax, 1));
  H_TRY(t.get(&bounds, 2));
  H_TRY(cudaMemsetAsync(wamax, 0, sizeof(float), st));
  H_TRY(cudaMemsetAsync(bounds, 0, 2 * sizeof(float), st));
  H_TRY(launch_absmax(op.W, op.ldw, op.K, op.N, wamax, st));
  H_TRY(launch_pack_weights(op.W, op.ldw, op.K, op.N, 1.f, parts, img, st, wamax));
  TcChain ch;
  ch.rows_per_sample = op.rows_per_sample, ch.batch = op.batch;
  ch.a0[0] = op.a[0], ch.a0[1] = op.a[1];
  ch.K0 = (op.K + 63) / 64 * 64, ch.n_layers = 1, ch.range_fit = 1, ch.split = split ? 1 : 0, ch.status = status;
  if (split)
    for (int a = 0; a < 2; ++a) {
      RowSrc& s = ch.a0[a];
      if (s.kind == SRC_NONE) continue;
      if (s.kind != SRC_STREAM && s.kind != SRC_BCAST) return (int)cudaErrorInvalidValue;
      const long long n = (long long)(s.kind == SRC_STREAM ? (long long)op.batch * s.src_rows : (long long)op.rows_per_sample) * s.ld;
      H_TRY(launch_absmax_flat(s.base, n, bounds + a, st));
      s.bound = bounds + a, s.bound_mul = 1.f, s.bound_mul_i = nullptr;
    }
  TcLayer& L = ch.layer[0];
  L.Wp = img, L.K = ch.K0, L.N = (op.N + 15) / 16 * 16, L.N32 = tc_packed_rows(op.N), L.n_valid = op.N, L.wamax = wamax;
  L.bias = op.bias, L.add[0] = op.add[0], L.add[1] = op.add[1], L.relu = op.relu;
  L.ln_g = op.ln_gamma, L.ln_b = op.ln_beta, L.residual = op.residual;
  L.out = op.out, L.ldo = op.ldo, L.out_cols = op.N, L.save_pre = op.save_pre, L.mask = op.mask;
  if (lean) *lean = tc3_chain_is_lean(ch) ? 1 : 0;
  return (int)launch_chain_tc3(ch, st);
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

int h_transpose(const float* W, int rows, int cols, float* WT, void* stream) {
  return (int)launch_transpose(W, rows, cols, WT, (cudaStream_t)stream);
}

}  // extern "C"
