// gw_wide_forward_harness.cu -- test-only shim over the row op of a layer-by-layer tensor-core plan (tests/test_gpu_wide_forward.py):
// gw::run_op on a plan that holds only what a row op reads -- its precision, the bound slots, the assembled-operand scratch, the
// status word and the weight-image cache -- so that one forward row op (column blocks, the LayerNorm finished by gw_ln_rows_kernel
// and the bound it writes) runs on its own and can be compared with float64.
//
// Host code only, like gw_kernel_harness.cu: flat extern "C" wrappers called through ctypes.  The op crosses the boundary as the
// same POD as that harness's HOp (test_gpu_kernels.HOp mirrors it), never as gw::GemmOp.  Every wrapper enqueues on the caller's
// stream.  Built by the test into a temporary directory and linked against the package's libgwb200.so with --no-undefined.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../graph_weather_b200/csrc/gw_plan.h"

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

struct HOp {  // one row op (layout of gw_kernel_harness.cu's HOp)
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

int h_sizeof_op() { return (int)sizeof(HOp); }

static gw::RowSrc row_src(const HSrc& h) {
  gw::RowSrc s;
  s.kind = h.kind, s.width = h.width, s.ld = h.ld, s.col0 = h.col0, s.base = h.base, s.src_rows = h.src_rows, s.idx = h.idx;
  s.base2 = h.base2, s.ld2 = h.ld2, s.ptr = h.ptr, s.perm = h.perm;
  return s;
}

// One forward row op as a plan of `precision` runs it (0: fp32_simt, the CUDA-core kernels; 1: fp32 and 2: bf16, a layer-by-layer
// plan: gw::run_op).  out_bound (LayerNorm'd ops on the tensor cores; zeroed by the caller) receives max |out|; status: the device
// status word the chains write.  Returns 0, or 1 with the library's message in *err (256 bytes).
int h_layered_row_op(int precision, const HOp* h, float* out_bound, int32_t* status, char* err, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  gw::GemmOp op;
  op.rows_per_sample = h->rows, op.batch = h->batch;
  op.a[0] = row_src(h->a[0]), op.a[1] = row_src(h->a[1]);
  op.W = h->W, op.K = h->K, op.N = h->N, op.ldw = h->ldw, op.bias = h->bias;
  op.add[0] = row_src(h->add[0]), op.add[1] = row_src(h->add[1]);
  op.relu = h->relu, op.ln_gamma = h->ln_g, op.ln_beta = h->ln_b, op.residual = row_src(h->residual);
  op.out = h->out, op.ldo = h->ldo, op.save_pre = h->save_pre, op.mask = row_src(h->mask);
  int rc = 1;
  {
    gw_plan p;
    std::memset(&p.d, 0, sizeof(p.d));
    p.d.precision = precision == 1 ? GW_PREC_FP32_TC : precision == 2 ? GW_PREC_BF16_TC : GW_PREC_FP32_SIMT;
    p.layered = precision != 0;
    p.tc_status_dev = status;
    p.row_images.new_weights(op.W);
    const size_t cat = (op.a[1].kind != gw::SRC_NONE || op.a[0].kind == gw::SRC_SEGSUM) ? (size_t)h->rows * h->batch * h->K : 0;
    if (p.bounds.alloc(gw::SL_COUNT) == 0 && p.cat.alloc(cat) == 0 && cudaMemsetAsync(p.bounds.p, 0, p.bounds.bytes(), st) == cudaSuccess)
      rc = gw::run_op(&p, op, st, out_bound);
    if (rc == 0 && cudaStreamSynchronize(st) != cudaSuccess) rc = 1;  // (the plan's buffers are freed below)
  }
  if (rc != 0 && err) {
    const char* m = gw_last_error();
    int i = 0;
    for (; m && m[i] && i < 255; ++i) err[i] = m[i];
    err[i] = 0;
  }
  return rc;
}

}  // extern "C"
