// gw_wide_harness.cu -- test-only shim for tests/test_gpu_wide_training.py: every wrapper of gw_kernel_harness.cu (included
// as it is, so the structs and helpers are the same ones) plus the column-blocked training row op.  Built by the test into a
// temporary directory and linked against the package's libgwb200.so with --no-undefined.
#include "gw_kernel_harness.cu"

extern "C" {

// One training row op of any N, as the training step runs it (gw_train.inl, train_op): precision 0 on CUDA cores; 1 / 2 as one-layer
// chains of at most TC_COL_BLOCK output columns (tc_column_block), each with the image of its rows of W, the stage-0 sources and
// their whole-tensor bounds shared.  *lean_mask: bit j = column block j takes the lean path.
int h_row_op_blocks(int precision, const HOp* h, int* lean_mask, int32_t* status, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  if (lean_mask) *lean_mask = 0;
  if (precision == 0) return h_row_op(0, h, nullptr, status, stream);
  if (precision != 1 && precision != 2) return (int)cudaErrorInvalidValue;
  const bool split = precision == 1;
  const int parts = split ? 2 : 1;
  Temps t(st);
  float* bounds = nullptr;
  H_TRY(t.get(&bounds, 2));
  H_TRY(cudaMemsetAsync(bounds, 0, 2 * sizeof(float), st));
  TcChain ch;
  ch.rows_per_sample = h->rows, ch.batch = h->batch;
  ch.a0[0] = row_src(h->a[0]), ch.a0[1] = row_src(h->a[1]);
  ch.K0 = (h->K + 63) / 64 * 64, ch.n_layers = 1, ch.split = split ? 1 : 0, ch.status = status;
  if (split)
    for (int a = 0; a < 2; ++a) {
      RowSrc& s = ch.a0[a];
      if (s.kind == SRC_NONE) continue;
      if (s.kind != SRC_STREAM && s.kind != SRC_BCAST) return (int)cudaErrorInvalidValue;
      const long long n = (long long)(s.kind == SRC_STREAM ? (long long)h->batch * s.src_rows : (long long)h->rows) * s.ld;
      H_TRY(launch_absmax_flat(s.base, n, bounds + a, st));
      s.bound = bounds + a, s.bound_mul = 1.f, s.bound_mul_i = nullptr;
    }
  TcLayer& L = ch.layer[0];
  L.K = ch.K0, L.N = h->N, L.n_valid = h->N;
  L.bias = h->bias, L.add[0] = row_src(h->add[0]), L.add[1] = row_src(h->add[1]), L.relu = h->relu;
  L.ln_g = h->ln_g, L.ln_b = h->ln_b, L.residual = row_src(h->residual);
  L.out = h->out, L.ldo = h->ldo, L.out_cols = h->N, L.save_pre = h->save_pre, L.mask = row_src(h->mask);
  for (int n0 = 0, j = 0; n0 < h->N; n0 += TC_COL_BLOCK, ++j) {
    const int nb = h->N - n0 < TC_COL_BLOCK ? h->N - n0 : TC_COL_BLOCK;
    TcChain blk;
    H_TRY(tc_column_block(ch, n0, nb, &blk));
    const float* W = h->W + (size_t)n0 * h->ldw;
    unsigned char* img = nullptr;
    float* wamax = nullptr;
    H_TRY(t.get(&img, tc_packed_bytes(h->K, nb, parts)));
    H_TRY(t.get(&wamax, 1));
    H_TRY(cudaMemsetAsync(wamax, 0, sizeof(float), st));
    H_TRY(launch_absmax(W, h->ldw, h->K, nb, wamax, st));
    H_TRY(launch_pack_weights(W, h->ldw, h->K, nb, 1.f, parts, img, st, wamax));
    blk.layer[0].Wp = img, blk.layer[0].wamax = wamax;
    if (lean_mask && tc3_chain_is_lean(blk)) *lean_mask |= 1 << j;
    H_TRY(launch_chain_tc3(blk, st));
  }
  return 0;
}


}  // extern "C"
