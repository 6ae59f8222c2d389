// gw_det_harness.cu -- test-only shim over the fixed-order launchers of libgwb200.so (tests/test_gpu_deterministic_kernels.py):
// the weight gradient and the LayerNorm backward that gw_train_set_deterministic selects, each with its workspace sized and
// allocated here.
//
// Host code only, like gw_kernel_harness.cu: flat extern "C" wrappers called through ctypes.  The row source crosses the boundary
// as the same POD as that harness's HSrc (test_gpu_kernels.HSrc mirrors it), never as gw::RowSrc.  Every wrapper enqueues on the
// caller's stream and returns the CUDA error code.  Built by the test into a temporary directory and linked against the package's
// libgwb200.so with --no-undefined.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../graph_weather_b200/csrc/gw_internal.h"

using namespace gw;

extern "C" {

struct HSrc {  // one row source (layout of gw_kernel_harness.cu's HSrc)
  int32_t kind, width, ld, col0;
  const float* base;
  int32_t src_rows;
  const int32_t* idx;
  const float* base2;
  int32_t ld2;
  const int32_t* bound_mul_i;
  const int32_t* ptr;
  const int32_t* perm;
};

}  // extern "C"

namespace {

RowSrc row_src(const HSrc& h) {
  RowSrc s;
  s.kind = h.kind, s.width = h.width, s.ld = h.ld, s.col0 = h.col0, s.base = h.base, s.src_rows = h.src_rows, s.idx = h.idx;
  s.base2 = h.base2, s.ld2 = h.ld2, s.ptr = h.ptr, s.perm = h.perm;
  return s;
}

// a device workspace of n floats for one wrapper call, freed in stream order when it returns
struct Workspace {
  cudaStream_t st;
  float* p = nullptr;
  explicit Workspace(cudaStream_t s) : st(s) {}
  ~Workspace() {
    if (p) cudaFreeAsync(p, st);
  }
  cudaError_t get(size_t n) { return cudaMallocAsync(reinterpret_cast<void**>(&p), n * sizeof(float) + 16, st); }
};

}  // namespace

extern "C" {

int h_sizeof_src() { return (int)sizeof(HSrc); }

long long h_det_ws_bytes() { return (long long)DET_WS_BYTES; }

// dW[o, k] (ld ldw) += sum_r dY[r, o] A(r, k), db[o] += sum_r dY[r, o] (db may be null), slab partials added in slab order;
// *ws_floats = the workspace it took
int h_wgrad_det(const float* dY, int ldy, int N, const HSrc* a, int K, int rows, int batch, float* dW, int ldw, float* db, long long* ws_floats,
                void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t n = wgrad_det_workspace_floats((long long)rows * batch, N, K);
  *ws_floats = (long long)n;
  Workspace ws(st);
  const cudaError_t e = ws.get(n);
  if (e != cudaSuccess) return (int)e;
  return (int)launch_wgrad_det(dY, ldy, N, row_src(*a), K, rows, batch, dW, ldw, db, ws.p, n, st);
}

// LayerNorm backward with per-CTA dgamma / dbeta partials added in a fixed order; *ws_floats = the workspace it took
int h_ln_bwd_det(const float* dy, int ld_dy, const float* z, int ld_z, int N, const float* gamma, long long R, float* dz, int ld_dz, float* dgamma,
                 float* dbeta, long long* ws_floats, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t n = ln_bwd_det_workspace_floats(R, N);
  *ws_floats = (long long)n;
  Workspace ws(st);
  const cudaError_t e = ws.get(n);
  if (e != cudaSuccess) return (int)e;
  return (int)launch_ln_bwd_det(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta, ws.p, n, st);
}

}  // extern "C"
