// gw_train.cu -- training step of GraphWeatherForecaster: a forward that keeps what the backward needs, and the backward itself (every caller of the reference trains: train/run.py:508-543 calls
// loss.backward() on forecast.py:215-247), and its part of the C ABI (the gw_tape_* and gw_train_* calls of include/gw_b200.h).  It works on
// gw_plan's graphs and weight views and launches through the forward's run_op / run_chain (gw_plan.h).  GraphCast and
// GraphWeatherAssimilator train on the same step: GraphCast is the forecaster with the full input as the residual, the assimilator
// has no residual, a zero (non-parameter) h3_nodes table and an observation graph rebuilt on every call (n_in_cur, enc_graph_gen).
//
// The forward is the factored graph of gw_forward.cu written out with every intermediate kept (h = hidden activations, z = the value
// entering LayerNorm); the backward walks it in reverse with five primitives (gw_simt.cu):
//     data gradient   dX = (dY . W) (.) relu-mask        the forward row-op kernel with the transposed weight and a mask
//     weight gradient dW += dY^T . A,  db += colsum(dY)   gw_wgrad_kernel (A assembled from a row source, like the forward)
//     LayerNorm       gw_ln_bwd_kernel                     dz, dgamma, dbeta
//     gathers         backward of x[src] / x[dst] / per-target sums: per-source / per-target segment sums and row gathers
//     broadcasts      tensors shared by the batch (encoded edge attributes, h3 node rows): gw_batch_reduce_kernel
// The weight gradient and the LayerNorm backward add their CTAs' sums with float atomics; gw_train_set_deterministic swaps in
// their fixed-order variants (gw_wgrad_det_kernel, gw_ln_bwd_det_kernel), and every other sum of the step has a fixed order.
// Gradients of the factored layer 1,  h1 = relu(e W1e^T + P_s[src] + P_d[dst] + b1),  P = x [W1s ; W1d]^T :
//     dP_s = per-source sum of dh1, dP_d = per-target sum of dh1;  dW1s += dP_s^T x, dW1d += dP_d^T x, dW1e += dh1^T e;
//     dx += dP_s W1s + dP_d W1d, de += dh1 W1e   -- two thirds of the K = 768 weight gradient are formed per NODE, not per edge.
// Scope: LayerNorm MLPs, the network up to the forecast (a constraint layer's backward, gw_constraint.cu, runs before this one
// on the gradient of the constrained output; its `lr` term reaches the features through autograd).  fp32_simt: node / edge dims <= 1024
// (LN_BWD_MAX_N), any feature / hidden / decoder width (train/run.py's 1024-wide model); fp32 / bf16: the 256-wide trunk the
// tensor-core plans are built for, any feature / output width (train/run_fulll.py's 597 + 24 features).
//
// Tapes: what a forward saves for its backward is a gw_tape.  Every forward runs on a tape gw_tape_create made -- one per training
// step, or one per forward of a multi-step rollout -- and its own backward consumes it.
//
// Stages: the step is three stage functions (enc_stage_* / proc_stage_* / dec_stage_*) with explicit boundary tensors; the whole
// network's forward and backward compose them, and the reference's standalone Encoder / Processor / Decoder train on one stage
// alone (gw_train_{encoder,processor,decoder}_{forward,backward}_tape).  A standalone encoder or decoder takes the step of its plan,
// taped or chunked, as the whole network does; its plan holds only its own graphs, and build_chunks cuts only their tables.
//
// Memory: the grid-sized phases (the encoder's lat/lon side, the decoder) are written once over a GridRange.  The taped step runs
// each on one whole range and keeps its tape from the forward.  A training-only plan (gw_plan_create_train, use_checkpointing=True)
// runs them chunk by chunk: the forward keeps only agg_m and the output rows, and the backward recomputes each chunk's tape with the
// same ops (and, in fp32 mode, the same per-chunk operand bounds) just before that chunk's backward, then frees it.  A standalone
// stage's chunks read the caller's rows (features; the decoder's x and residual rows) again through the forward's own row sources,
// which the caller keeps alive until the backward.  Processor
// segments (gw_train_set_processor_segments, either step) do the same for the mesh-sized processor: the forward keeps x and e at the
// start of every segment, and the backward recomputes a segment's blocks with block_fwd right before their block_bwd.
//
// Arithmetic (the plan's precision):
//   fp32_simt   every product on CUDA cores in exact fp32 (gw_simt.cu).
//   fp32 / bf16 every row op (forward layer, data gradient) is a one-layer wgmma chain (gw_tc3.cu, general or lean path; the mask
//               and the pre-LayerNorm store are chain epilogue parts) and every weight gradient with K > 16 runs on gw_wgrad_tc.cu.
//               fp32: operands split to fp16 hi/lo, 3 MMAs per product, each operand scaled by a power of two from its measured
//               absmax into [2^14, 2^15) (gradients are ~1e-8); bf16: one MMA per product.  Master weights, gradients and the tape
//               stay fp32.  The weight images (W and W^T, K-major perm32, SWIZZLE_128B) are repacked once per weight upload (the
//               first step after gw_plan_set_weights), their scale taken on the device.  The memory-bound parts (LayerNorm backward, segment sums, gathers, batch reductions) stay on the
//               CUDA-core kernels above.

#include "gw_plan.h"

namespace gw {

struct MlpTape {
  std::vector<float*> h;  // hidden activations h[l] [R, out_l], l < L
  float* z = nullptr;     // [R, out_L] value entering LayerNorm (null: MLP without norm)
  int rows = 0, batch = 0;
};

// Rows of one grid-sized phase of the step.  whole: every row in its natural order (the taped step).  Otherwise a chunk:
//   encoder  positions r0 .. r1 of enc_perm (points sorted by mesh slot), i.e. all points of the mesh slots s0 .. s1
//   decoder  lat/lon points r0 .. r1 and their decoder edges e0 .. e1; c = chunk number (its source-sorted CSR)
struct GridRange {
  bool whole = true;
  int r0 = 0, r1 = 0, s0 = 0, s1 = 0, e0 = 0, e1 = 0, c = 0;
};
// what the backward of the encoder's grid side reads (lat/lon rows of one GridRange)
struct EncTape {
  const float* feat = nullptr;   // node-encoder input rows [B, n, in_dim]
  const float* attr = nullptr;   // edge attributes [n, enc_edge_attr_dim]
  const int32_t* mesh = nullptr; // mesh slot of every row
  float *xg = nullptr, *e_enc = nullptr;
  MlpTape node_g, edge_enc, edge;
};
// ... and of the decoder (lat/lon points and decoder edges of one GridRange)
struct DecTape {
  float *e_dec = nullptr, *agg_g = nullptr, *xg2 = nullptr;
  MlpTape edge_enc, edge, node, out;
};
// the graph a tape's processor runs on: the plan's latent graph (the whole network), or a standalone processor's per-call graph
// copied onto the tape with its source-sorted CSR (gw_train_processor_forward_tape)
struct LatGraph {
  int H = 0, El = 0;                                              // nodes per sample, edges per sample
  const int32_t *src = nullptr, *dst = nullptr, *ptr = nullptr;   // edges sorted by target, CSR over targets
  const int32_t *perm_src = nullptr, *ptr_src = nullptr;          // the same edges grouped by source
  bool e0_bcast = true;  // block 0 reads e[0] as one sample's rows broadcast over the batch (the encoder's e_lat), else per edge
};
// what a tape's forward ran, so that only the matching backward consumes it
enum TapeStage { TAPE_NET = 0, TAPE_ENC, TAPE_PROC, TAPE_DEC };

}  // namespace gw

// One tape: what one training forward saves for its own backward.  A plan has as many as gw_tape_create made, so that several
// forwards of one window (a multi-step rollout) stay differentiable at once; a second forward on a tape replaces the first's
// activations.  Everything a backward reads that its forward wrote lives here; what the plan shares
// between tapes (TrainState) depends on the shapes, the graphs and the weights only -- and a backward refuses to run once the
// weights it would differentiate were replaced (wgen).
struct gw_tape {
  gw_plan* plan = nullptr;  // null: dead (its plan was destroyed, which released its memory)
  std::vector<std::pair<void*, size_t>> allocs;  // stream-ordered allocations (pointer, bytes): the saved tensors, and the backward's temporaries
  size_t bytes = 0;                              // bytes they hold now
  unsigned wgen = 0;                             // gw_plan::wgen of the weights the forward ran with
  int batch = 0;
  int segments = 0;        // processor segments its forward ran with (gw_plan::train_segments; its backward follows them)
  bool have_tape = false;  // a forward's activations, not yet consumed by a backward
  int stage = gw::TAPE_NET;        // the forward that made it: the whole network or one stage
  unsigned enc_gen = 0;            // gw_plan::enc_graph_gen its encoder ran on
  unsigned graph_gen = 0;          // gw_plan::graph_gen of the latent and decoder graphs and h3_nodes rows it ran on
  bool caller_input = false;       // the processor's / decoder's input rows are the caller's: their stage-0 ops bound them (train_op)
  const float* features = nullptr;
  const float* start = nullptr;    // the decoder's residual rows (the features in the whole network), row stride start_ld
  int start_ld = 0;
  const float* xd = nullptr;       // the decoder's input x [B, H, Dn]
  float *xm0 = nullptr, *agg_m = nullptr, *e_lat = nullptr, *Pm = nullptr, *Pd = nullptr;  // (Pm, Pd: the grid phases' mesh-side addends)
  // x[k] k = 0..nb, e[k] k = 0..nb (e[0]: e_lat broadcast, or a standalone processor's per-edge input), agg[k].  With processor
  // segments only x[k], e[k] at the start of each segment and x[nb] are kept; agg, t_pe and t_pn stay empty.
  std::vector<float*> x, e, agg;
  gw::LatGraph g;
  gw::MlpTape t_enc_node_h, t_enc_mnode, t_lat_enc;
  gw::EncTape enc;  // taped step: the grid-sized tapes (the chunked step recomputes them chunk by chunk)
  gw::DecTape dec;
  std::vector<gw::MlpTape> t_pe, t_pn;
};

namespace gw {

// What the tapes of a plan share: the stream, the weights' transposes and gradient buffer, the source-sorted graphs, the chunk
// tables and the tensor-core weight images.
struct TrainState {
  cudaStream_t st = nullptr;
  gw_tape* tp = nullptr;       // the tape the running forward / backward writes and reads (set by each of them)
  std::set<gw_tape*> tapes;    // every tape of the plan that is not dead
  size_t cur_bytes = 0, peak_bytes = 0;  // bytes all tapes hold now / at most since a forward began with no other tape holding any
  DevBuf<float> wT, gbuf;     // transposed weights / gradients, laid out like gw_plan::wbuf
  unsigned wgen = 0;          // gw_plan::wgen that wT and the weight images were made for (per-weight work runs once per upload)
  DevBuf<int32_t> lat_perm_src, lat_ptr_src, dec_perm_src, dec_ptr_src, iota;
  DevBuf<unsigned char> sort_ws;
  bool pool_kept = false;   // the stream-ordered pool keeps its memory between steps
  unsigned graphs_gen = 0;  // gw_plan::graph_gen the source-sorted graphs were built for
  // chunked step (training-only plans): chunk tables for a batch size (and, for the encoder, an encoder graph), built by the forward
  // and, when a tape of another batch size ran since, again by the backward
  int enc_chunks_batch = 0, dec_chunks_batch = 0;
  unsigned enc_chunks_gen = 0, dec_chunks_gen = 0;  // gw_plan::enc_graph_gen / graph_gen the tables were built for
  std::vector<GridRange> enc_chunks, dec_chunks;
  DevBuf<int32_t> enc_slot_sorted;  // mesh slot of every position of enc_perm
  DevBuf<int32_t> dec_cperm, dec_cptr;  // per decoder chunk: its edges sorted by source (chunk-local ids) and the CSR over mesh slots
  RowImages images;      // tensor-core precisions: the weight images of the step's row ops (tc_row_op)
  DevBuf<float> bslots;  // operand magnitude bounds of the current phase (reset at the start of the forward and of the backward)
  size_t bslot_used = 0;
  DevBuf<float> wg_ws;   // gw_wgrad_tc.cu partial sums
  DevBuf<float> det_ws;  // partial sums of the fixed-order CUDA-core weight gradient and LayerNorm backward (gw_plan::train_deterministic)
};

// an allocation of the running tape (stream-ordered on the step's stream)
static float* talloc(TrainState* t, size_t floats) {
  void* q = nullptr;
  const size_t bytes = std::max<size_t>(floats, 1) * sizeof(float);
  if (cudaMallocAsync(&q, bytes, t->st) != cudaSuccess) return nullptr;
  t->tp->allocs.push_back({q, bytes});
  t->tp->bytes += bytes;
  t->cur_bytes += bytes;
  t->peak_bytes = std::max(t->peak_bytes, t->cur_bytes);
  return static_cast<float*>(q);
}
// releases (stream-ordered, on `st`) every allocation tape k made since its allocs.size() was `mark`
static void tape_free_to(TrainState* t, gw_tape* k, size_t mark, cudaStream_t st) {
  while (k->allocs.size() > mark) {
    cudaFreeAsync(k->allocs.back().first, st);
    k->bytes -= k->allocs.back().second;
    t->cur_bytes -= k->allocs.back().second;
    k->allocs.pop_back();
  }
}
static void tfree_to(TrainState* t, size_t mark) { tape_free_to(t, t->tp, mark, t->st); }
// releases every allocation of the running tape made since its allocs.size() was `mark`, except the buffers in `keep` (which stay,
// in their order, at the end of the list)
static void tfree_except(TrainState* t, size_t mark, std::initializer_list<const void*> keep) {
  gw_tape* k = t->tp;
  size_t w = mark;
  for (size_t r = mark; r < k->allocs.size(); ++r) {
    const auto a = k->allocs[r];
    if (std::find(keep.begin(), keep.end(), a.first) != keep.end()) {
      k->allocs[w++] = a;
    } else {
      cudaFreeAsync(a.first, t->st);
      k->bytes -= a.second;
      t->cur_bytes -= a.second;
    }
  }
  k->allocs.resize(w);
}
// releases one allocation of the running tape (null: none).  It may lie below a mark, so no mark may be pending across this call.
static void tfree_one(TrainState* t, const void* q) {
  if (!q) return;
  gw_tape* k = t->tp;
  for (size_t r = k->allocs.size(); r-- > 0;)
    if (k->allocs[r].first == q) {
      cudaFreeAsync(k->allocs[r].first, t->st);
      k->bytes -= k->allocs[r].second;
      t->cur_bytes -= k->allocs[r].second;
      k->allocs.erase(k->allocs.begin() + r);
      return;
    }
}
static void tape_release(TrainState* t, gw_tape* k, cudaStream_t st) {
  tape_free_to(t, k, 0, st);
  k->have_tape = false;
}
#define GW_TALLOC(var, floats)                                          \
  float* var = talloc(T, (floats));                                     \
  GW_CHECK(var != nullptr, "training step: out of device memory")

static float* grad_of(gw_plan* p, TrainState* T, const float* w) { return T->gbuf.p + (w - p->wbuf.p); }

// a memory-bound kernel of the step, timed under train_other
#define GW_OTHER(expr)                     \
  do {                                     \
    p->cur_tag = TAG_TRAIN_OTHER;          \
    TimedLaunch _tl(p, T->st);             \
    GW_CUDA(expr);                         \
  } while (0)

static bool split_of(const gw_plan* p) { return p->d.precision == GW_PREC_FP32_TC; }

// device bound of a chain's stage-0 source (fp32 mode), in the next operand-bound slot
static int operand_bound(gw_plan* p, TrainState* T, RowSrc& s, int rows, int batch) {
  GW_CHECK(T->bslot_used < T->bslots.n, "training step: out of operand-bound slots");
  float* b = T->bslots.p + T->bslot_used++;
  p->cur_tag = TAG_TRAIN_PACK;
  TimedLaunch tl(p, T->st);
  GW_CUDA(launch_operand_bound(s, rows, batch, b, T->st));
  return 0;
}

// One row op of the step: exact fp32 on CUDA cores (fp32_simt plans) or one-layer wgmma chains in column blocks (tensor-core
// plans: tc_row_op; the stage-0 operand and its bound are shared by the blocks).  tag: the phase it is timed under (train_fwd /
// train_dgrad).  reads_input: the op's stage-0 operand is the caller's features; bf16 plans bound it too (fp32 plans bound every
// operand), so that an inf / NaN feature sets status bit 3 in every tensor-core precision instead of passing through the
// epilogue's ReLU as a finite number.
static int train_op(gw_plan* p, TrainState* T, GemmOp op, int tag, bool reads_input = false) {
  if (!is_tc(p)) {
    p->cur_tag = tag;
    return run_op(p, op, T->st);
  }
  GW_CHECK(op.add[2].kind == SRC_NONE && op.a[0].kind != SRC_NONE && !(op.ln_gamma && op.N > TC_COL_BLOCK),
           "training row op: no tensor-core chain for an add[2] addend, a missing a[0] or a LayerNorm wider than 256 columns");
  if (split_of(p) || reads_input)
    for (int a = 0; a < 2; ++a)
      if (op.a[a].kind != SRC_NONE) GW_TRY(operand_bound(p, T, op.a[a], op.rows_per_sample, op.batch));
  return tc_row_op(p, T->images, op, nullptr, tag, T->st);
}

static int det_workspace(TrainState* T, size_t floats) {
  if (T->det_ws.n < floats) GW_TRY(T->det_ws.alloc(floats));
  return 0;
}

// dW += dY^T A, db += colsum(dY): gw_wgrad_tc.cu on tensor-core plans (K > 16), else the CUDA-core kernel (its fixed-order
// variant under gw_train_set_deterministic)
static int train_wgrad(gw_plan* p, TrainState* T, const float* dY, int ldy, int N, const RowSrc& a, int K, int rows, int batch, float* dW, int ldw,
                       float* db) {
  p->cur_tag = TAG_TRAIN_WGRAD;
  TimedLaunch tl(p, T->st);
  if (!is_tc(p) || K <= 16) {  // (the edge encoders' 2- and 3-wide inputs: too narrow for a tensor-core product)
    if (p->train_deterministic) {
      GW_TRY(det_workspace(T, wgrad_det_workspace_floats((long long)rows * batch, N, K)));
      GW_CUDA(launch_wgrad_det(dY, ldy, N, a, K, rows, batch, dW, ldw, db, T->det_ws.p, T->det_ws.n, T->st));
    } else {
      GW_CUDA(launch_wgrad(dY, ldy, N, a, K, rows, batch, dW, ldw, db, T->st));
    }
    return 0;
  }
  const size_t need = wgrad_tc_workspace_floats((long long)rows * batch, N, K);
  if (T->wg_ws.n < need) GW_TRY(T->wg_ws.alloc(need));
  GW_CUDA(launch_wgrad_tc(dY, ldy, N, a, K, rows, batch, dW, ldw, db, split_of(p), T->wg_ws.p, T->wg_ws.n, p->tc_status_dev, T->st));
  return 0;
}
static const float* wT_of(gw_plan* p, TrainState* T, const float* w) { return T->wT.p + (w - p->wbuf.p); }

// MLP forward keeping h and z.  `first` describes Linear 0 (A sources / addends / weight slice / bias may be customised by the
// caller: factored layer 1); the result is out = residual + LN(...) (LN if the MLP has a norm).  reads_input: Linear 0 reads the
// caller's features (train_op).
static int mlp_fwd(gw_plan* p, TrainState* T, const Mlp& m, GemmOp first, const RowSrc& residual, float* out, int ldo, MlpTape* tape,
                   bool reads_input = false) {
  const int rows = first.rows_per_sample, batch = first.batch;
  const size_t R = (size_t)rows * batch;
  tape->rows = rows, tape->batch = batch;
  tape->h.assign(m.L, nullptr);
  for (int l = 0; l < m.L; ++l) {
    tape->h[l] = talloc(T, R * m.out[l]);
    GW_CHECK(tape->h[l] != nullptr, "training step: out of device memory");
  }
  const bool norm = m.ln_g != nullptr;
  if (norm) {
    tape->z = talloc(T, R * m.out[m.L]);
    GW_CHECK(tape->z != nullptr, "training step: out of device memory");
  }
  for (int l = 0; l <= m.L; ++l) {
    GemmOp op;
    if (l == 0) {
      op = first;
    } else {
      op.rows_per_sample = rows, op.batch = batch;
      op.a[0] = src_stream(tape->h[l - 1], m.in[l], m.in[l], rows);
      op.W = m.W[l], op.K = m.in[l], op.ldw = m.in[l], op.bias = m.b[l];
    }
    op.N = m.out[l];
    if (l < m.L) {
      op.relu = 1, op.out = tape->h[l], op.ldo = m.out[l];
    } else {
      op.relu = 0;
      if (norm) op.ln_gamma = m.ln_g, op.ln_beta = m.ln_b, op.save_pre = tape->z;
      op.residual = residual, op.out = out, op.ldo = ldo;
      GW_CHECK(!norm || ldo == m.out[l], "training MLP: LayerNorm output must be dense");
    }
    GW_TRY(train_op(p, T, op, TAG_TRAIN_FWD, reads_input && l == 0));
  }
  return 0;
}

// dX[R, N_in] = (dY[R, N_out] . W[N_out, N_in slice]) (.) (mask > 0) + add      W given as a view (pointer into wbuf, ld = ldw, col offset folded in)
static int dgrad(gw_plan* p, TrainState* T, const float* dY, int ldy, int n_out, int rows, int batch, const float* W_view, int w_rows, int col0,
                 int n_in, const float* mask, int ld_mask, const float* add, int ld_add, float* dX, int ldx) {
  // transposed weight: WT[k, n] for the whole matrix [columns of W, w_rows]; the slice starts at row col0
  const float* WT = wT_of(p, T, W_view) + (size_t)col0 * w_rows;
  GemmOp op;
  op.rows_per_sample = rows, op.batch = batch;
  op.a[0] = src_stream(dY, ldy, n_out, rows);
  op.W = WT, op.K = n_out, op.N = n_in, op.ldw = w_rows;
  if (add) op.add[0] = src_stream(add, ld_add, n_in, rows);
  if (mask) op.mask = src_stream(mask, ld_mask, n_in, rows);
  op.out = dX, op.ldo = ldx;
  return train_op(p, T, op, TAG_TRAIN_DGRAD);
}

// backward of an MLP from the gradient of its output down to the gradient at Linear 0's output (after the ReLU mask): dh0 [R, out_0]
static int mlp_bwd(gw_plan* p, TrainState* T, const Mlp& m, const MlpTape& tape, const float* dOut, int ld_dout, float** dh0_out) {
  const int rows = tape.rows, batch = tape.batch;
  const size_t R = (size_t)rows * batch;
  const float* cur = dOut;
  int ldc = ld_dout;
  if (tape.z) {
    GW_TALLOC(dz, R * m.out[m.L]);
    if (p->train_deterministic) {
      GW_TRY(det_workspace(T, ln_bwd_det_workspace_floats((long long)R, m.out[m.L])));
      GW_OTHER(launch_ln_bwd_det(dOut, ld_dout, tape.z, m.out[m.L], m.out[m.L], m.ln_g, (long long)R, dz, m.out[m.L], grad_of(p, T, m.ln_g),
                                 grad_of(p, T, m.ln_b), T->det_ws.p, T->det_ws.n, T->st));
    } else {
      GW_OTHER(launch_ln_bwd(dOut, ld_dout, tape.z, m.out[m.L], m.out[m.L], m.ln_g, (long long)R, dz, m.out[m.L], grad_of(p, T, m.ln_g),
                             grad_of(p, T, m.ln_b), T->st));
    }
    cur = dz, ldc = m.out[m.L];
  }
  for (int l = m.L; l >= 1; --l) {
    GW_TRY(train_wgrad(p, T, cur, ldc, m.out[l], src_stream(tape.h[l - 1], m.in[l], m.in[l], rows), m.in[l], rows, batch, grad_of(p, T, m.W[l]), m.in[l],
                       grad_of(p, T, m.b[l])));
    GW_TALLOC(dh, R * m.in[l]);
    GW_TRY(dgrad(p, T, cur, ldc, m.out[l], rows, batch, m.W[l], m.out[l], 0, m.in[l], tape.h[l - 1], m.in[l], nullptr, 0, dh, m.in[l]));
    cur = dh, ldc = m.in[l];
  }
  *dh0_out = const_cast<float*>(cur);
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// chunks of the bounded-memory step (training-only plans, gw_plan_create_train)
// ---------------------------------------------------------------------------------------------------------------------------
// Working set one chunk of a grid-sized phase may hold.  A constant: chunk boundaries, and with them the fp32 summation order of
// the gradients, follow from the shapes alone -- never from the free memory of a device that other processes share.
constexpr double TRAIN_CHUNK_BYTES = 4.0 * (1ull << 30);

// points per chunk for a phase with `rows_per_point` edge rows per lat/lon point (encoder 1, decoder ~7): per point and sample,
// about 18 rows of the widest width per edge (the edge MLPs' tape and backward temporaries, the batch-shared ones counted per
// sample) and 12 per point (node MLPs).  GW_B200_TRAIN_CHUNK (read at plan creation) overrides it: many chunks on small grids.
static int chunk_points(const gw_plan* p, int batch, double rows_per_point) {
  if (p->train_chunk_pts > 0) return p->train_chunk_pts;
  const gw_dims& d = p->d;
  const double w = std::max({d.node_dim, d.edge_dim, d.hidden_node, d.hidden_edge, d.hidden_dec, d.in_dim, d.out_dim});
  const double per_point = 4.0 * w * (18.0 * rows_per_point + 12.0);
  return (int)std::max(1.0, std::min(2.0e9, std::floor(TRAIN_CHUNK_BYTES / (batch * per_point))));
}

// Encoder chunks: whole mesh slots in enc_perm order (a slot's sum is never split; a slot larger than the budget is a chunk of its
// own).  Decoder chunks: runs of consecutive points, whose edges are consecutive too, each with the source-sorted CSR of its edges.
// The decoder tables are built per batch size and graph generation (gw_plan::graph_gen): RegionalForecaster.forward_regions uploads
// a new decoder graph on every call, and source-sorted edges of an earlier graph would send each gradient to the wrong cell.  The
// encoder tables are built per batch size and encoder graph (gw_plan::enc_graph_gen): the assimilator's observation graph changes on
// every call, and chunks of an earlier graph would cover the wrong points.  Building them copies enc_ptr to the host, so a step whose encoder graph changed synchronises its stream once (every
// bounded step of the assimilator and of a standalone AssimilatorEncoder; the taped step builds no chunk tables).  Only the tables
// of the stages the plan holds are built: a standalone encoder's plan has no decoder graph, a standalone decoder's no encoder graph.
// Both phases index iota: encoder chunks by mesh slot, decoder chunks by point.
static int build_chunks(gw_plan* p, TrainState* T, int batch) {
  const gw_dims& d = p->d;
  const int H = d.n_mesh, N = p->n_in_cur, No = d.n_out, Ed = d.n_dec_edges;
  const size_t n_iota = std::max(p->have_enc ? H : 0, p->have_dec ? No : 0);
  if (T->iota.n < n_iota) {
    std::vector<int32_t> iota(n_iota);
    for (size_t i = 0; i < iota.size(); ++i) iota[i] = (int32_t)i;
    GW_TRY(T->iota.alloc(iota.size()));
    GW_CUDA(cudaMemcpyAsync(T->iota.p, iota.data(), iota.size() * sizeof(int32_t), cudaMemcpyHostToDevice, T->st));
    GW_CUDA(cudaStreamSynchronize(T->st));  // (the copy reads `iota`, which goes out of scope with this block)
  }
  if (p->have_enc && (T->enc_chunks_batch != batch || T->enc_chunks_gen != p->enc_graph_gen)) {
    std::vector<int32_t> eptr(H + 1), slot(std::max(N, 1));
    GW_CUDA(cudaMemcpyAsync(eptr.data(), p->enc_ptr.p, (H + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, T->st));
    GW_CUDA(cudaStreamSynchronize(T->st));
    for (int s = 0; s < H; ++s)
      for (int j = eptr[s]; j < eptr[s + 1]; ++j) slot[j] = s;
    if (T->enc_slot_sorted.n < slot.size()) GW_TRY(T->enc_slot_sorted.alloc(slot.size()));
    GW_CUDA(cudaMemcpyAsync(T->enc_slot_sorted.p, slot.data(), slot.size() * sizeof(int32_t), cudaMemcpyHostToDevice, T->st));
    GW_CUDA(cudaStreamSynchronize(T->st));  // (the copy reads `slot`, which goes out of scope with this block)
    long long most = 0;  // most rows (samples x rows) of one chunk's row op
    T->enc_chunks.clear();
    const int pe = chunk_points(p, batch, 1.0);
    for (int s0 = 0; s0 < H;) {
      int s1 = s0 + 1;
      // (leading slots without points join the first slot that has some, even one larger than the budget: a chunk of no
      // points would run its row ops on zero rows)
      while (s1 < H && (eptr[s1 + 1] - eptr[s0] <= pe || (T->enc_chunks.empty() && eptr[s1] == eptr[s0]))) ++s1;
      if (eptr[s1] == eptr[s0] && !T->enc_chunks.empty()) {  // trailing slots without points join the previous chunk
        T->enc_chunks.back().s1 = s1;
      } else {
        GridRange r;
        r.whole = false, r.s0 = s0, r.s1 = s1, r.r0 = eptr[s0], r.r1 = eptr[s1];
        T->enc_chunks.push_back(r);
        most = std::max(most, (long long)batch * (r.r1 - r.r0));
      }
      s0 = s1;
    }
    GW_CHECK(most <= INT32_MAX, "training step: one chunk of the grid-sized stages holds more than 2^31 rows (lower the batch)");
    T->enc_chunks_batch = batch, T->enc_chunks_gen = p->enc_graph_gen;
  }
  if (p->have_dec && (T->dec_chunks_batch != batch || T->dec_chunks_gen != p->graph_gen)) {
    std::vector<int32_t> dptr(No + 1);
    GW_CUDA(cudaMemcpyAsync(dptr.data(), p->dec_ptr.p, (No + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, T->st));
    GW_CUDA(cudaStreamSynchronize(T->st));
    long long most = 0;
    T->dec_chunks.clear();
    const int pd = chunk_points(p, batch, (double)Ed / std::max(No, 1));
    for (int n0 = 0; n0 < No; n0 += pd) {
      GridRange r;
      r.whole = false, r.r0 = n0, r.r1 = std::min(No, n0 + pd), r.e0 = dptr[n0], r.e1 = dptr[r.r1], r.c = (int)T->dec_chunks.size();
      T->dec_chunks.push_back(r);
      most = std::max(most, (long long)batch * (r.e1 - r.e0));
    }
    GW_CHECK(most <= INT32_MAX, "training step: one chunk of the grid-sized stages holds more than 2^31 rows (lower the batch)");
    GW_TRY(T->dec_cperm.alloc(std::max(Ed, 1)) | T->dec_cptr.alloc(T->dec_chunks.size() * (size_t)(H + 1)));
    for (const GridRange& r : T->dec_chunks) {
      int32_t* cptr = T->dec_cptr.p + (size_t)r.c * (H + 1);
      if (r.e1 == r.e0)
        GW_CUDA(cudaMemsetAsync(cptr, 0, (H + 1) * sizeof(int32_t), T->st));
      else
        GW_CUDA(launch_sort_csr(p->dec_src.p + r.e0, r.e1 - r.e0, H, T->dec_cperm.p + r.e0, cptr, T->sort_ws.p, T->sort_ws.n, T->st));
    }
    T->dec_chunks_batch = batch, T->dec_chunks_gen = p->graph_gen;
  }
  return 0;
}

// need: the stages the forward runs (check_ready's NEED_ENC / NEED_PROC / NEED_DEC)
static int train_prepare(gw_plan* p, TrainState* T, int batch, int need, cudaStream_t st) {
  const gw_dims& d = p->d;
  GW_CHECK(d.precision == GW_PREC_FP32_SIMT || d.precision == GW_PREC_FP32_TC || d.precision == GW_PREC_BF16_TC, "unknown training precision");
  GW_TRY(check_ready(p, batch, need));
  // the LayerNorm'd widths are node_dim and edge_dim (every other width, feature and hidden, is a plain Linear of any size)
  GW_CHECK(d.node_dim <= LN_BWD_MAX_N && d.edge_dim <= LN_BWD_MAX_N, "training kernels cover node / edge dims <= 1024 (LayerNorm backward)");
  GW_CHECK(!is_tc(p) || (d.node_dim <= 256 && d.edge_dim <= 256 && d.hidden_node <= 256 && d.hidden_edge <= 256),
           "tensor-core training covers node / edge / hidden dims <= 256");
  T->st = st;
  if (T->wT.n != p->wbuf.n) {
    GW_TRY(T->wT.alloc(p->wbuf.n));
    T->wgen = 0;
  }
  if (T->gbuf.n != p->wbuf.n) GW_TRY(T->gbuf.alloc(p->wbuf.n));
  if (T->wgen != p->wgen) {  // per-weight work, once per gw_plan_set_weights: the K forwards of a rollout share it
    p->cur_tag = TAG_TRAIN_WEIGHTS;
    for (const auto& kv : p->params) {  // transposed copies of every matrix
      const int64_t r = kv.second.second.first, c = kv.second.second.second;
      if (c > 1) {
        TimedLaunch tl(p, st);
        GW_CUDA(launch_transpose(kv.second.first, (int)r, (int)c, T->wT.p + (kv.second.first - p->wbuf.p), st));
      }
    }
    if (is_tc(p)) {  // the weight images of these weights are packed on first use (tc_row_op)
      T->images.tag = TAG_TRAIN_WEIGHTS;
      T->images.new_weights(p->wbuf.p);
    }
    T->wgen = p->wgen;
  }
  if (is_tc(p) && T->bslots.n == 0) GW_TRY(T->bslots.alloc(4096));
  if (!T->pool_kept) {  // keep the stream-ordered pool's memory between steps (the default returns it to the driver at every sync)
    cudaMemPool_t pool = nullptr;
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      unsigned long long keep = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    T->pool_kept = true;
  }
  if (T->graphs_gen != p->graph_gen) {  // edges grouped by SOURCE (the x[src] gathers become per-source sums going backward), for
                                        // the graphs the plan holds, rebuilt whenever an upload replaced them
    const int El = d.n_lat_edges, Ed = d.n_dec_edges, H = d.n_mesh;
    const size_t ws = std::max(sort_csr_workspace_bytes(El), sort_csr_workspace_bytes(Ed));
    if (T->sort_ws.n < ws) GW_TRY(T->sort_ws.alloc(ws));
    if (p->have_lat) {
      GW_TRY(T->lat_perm_src.alloc(El) | T->lat_ptr_src.alloc(H + 1));
      GW_CUDA(launch_sort_csr(p->lat_src.p, El, H, T->lat_perm_src.p, T->lat_ptr_src.p, T->sort_ws.p, T->sort_ws.n, st));
    }
    if (p->have_dec) {
      GW_TRY(T->dec_perm_src.alloc(Ed) | T->dec_ptr_src.alloc(H + 1));
      GW_CUDA(launch_sort_csr(p->dec_src.p, Ed, H, T->dec_perm_src.p, T->dec_ptr_src.p, T->sort_ws.p, T->sort_ws.n, st));
    }
    T->graphs_gen = p->graph_gen;
  }
  if (p->train_only) GW_TRY(build_chunks(p, T, batch));
  return 0;
}

static int reset_bounds(TrainState* T) {
  T->bslot_used = 0;
  if (T->bslots.n) GW_CUDA(cudaMemsetAsync(T->bslots.p, 0, T->bslots.bytes(), T->st));  // (absmax accumulates with atomicMax)
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// grid-sized phases, on the rows of one GridRange (the taped step: one whole range whose tape is kept from the forward; the
// chunked step: chunk after chunk, each recomputed by the same forward ops ahead of its backward)
// ---------------------------------------------------------------------------------------------------------------------------
static int enc_rows(const gw_plan* p, const GridRange& r) { return r.whole ? p->n_in_cur : r.r1 - r.r0; }
static int dec_rows(const gw_plan* p, const GridRange& r) { return r.whole ? p->d.n_out : r.r1 - r.r0; }
static int dec_edges(const gw_plan* p, const GridRange& r) { return r.whole ? p->d.n_dec_edges : r.e1 - r.e0; }

// encoder, lat/lon rows: xg = node_encoder(features), e_enc = edge_encoder(attr), the encoder block's edge MLP
// e' = LN(MLP(h1)) + e_enc with h1 = relu(xg W1s^T + Pm[mesh] + e_enc W1e^T + b1); agg_m (not null): the per-slot sums of e'
static int enc_fwd(gw_plan* p, TrainState* T, const GridRange& r, const float* Pm, float* agg_m, EncTape* tp) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, N = p->n_in_cur, H = d.n_mesh, B = T->tp->batch, n = enc_rows(p, r),
            ad = d.enc_edge_attr_dim;
  RowSrc none;
  if (r.whole) {
    tp->feat = T->tp->features, tp->attr = p->enc_attr.p, tp->mesh = p->enc_mesh.p;
  } else {  // the chunk's points in enc_perm order
    GW_TALLOC(fc, (size_t)B * n * d.in_dim);
    GW_OTHER(launch_permute_rows(T->tp->features, d.in_dim, p->enc_perm.p + r.r0, n, N, d.in_dim, B, fc, d.in_dim, false, T->st));
    GW_TALLOC(ac, (size_t)n * ad);
    GW_OTHER(launch_permute_rows(p->enc_attr.p, ad, p->enc_perm.p + r.r0, n, N, ad, 1, ac, ad, false, T->st));
    tp->feat = fc, tp->attr = ac, tp->mesh = T->enc_slot_sorted.p + r.r0;
  }
  const Mlp& mne = p->enc_node;
  GW_TALLOC(xg, (size_t)B * n * Dn);
  GW_TRY(mlp_fwd(p, T, mne, first_op(n, B, src_stream(tp->feat, d.in_dim, d.in_dim, n), none, mne.W[0], mne.in[0], mne.in[0], mne.b[0]), none, xg, Dn,
                 &tp->node_g, true));
  const Mlp& mee = p->enc_edge_enc;
  GW_TALLOC(e_enc, (size_t)n * De);
  GW_TRY(mlp_fwd(p, T, mee, first_op(n, 1, src_stream(tp->attr, ad, ad, n), none, mee.W[0], mee.in[0], mee.in[0], mee.b[0]), none, e_enc, De,
                 &tp->edge_enc));
  const Mlp& meb = p->enc_blk_edge;
  GW_TALLOC(Pe, (size_t)n * He);
  {
    GemmOp c;
    c.rows_per_sample = n, c.batch = 1, c.a[0] = src_stream(e_enc, De, De, n), c.W = meb.W[0] + 2 * Dn, c.K = De, c.ldw = meb.in[0], c.N = He, c.out = Pe, c.ldo = He;
    GW_TRY(train_op(p, T, c, TAG_TRAIN_FWD));
  }
  GW_TALLOC(ep_enc, (size_t)B * n * De);
  {
    GemmOp fo = first_op(n, B, src_stream(xg, Dn, Dn, n), none, meb.W[0], Dn, meb.in[0], meb.b[0]);
    fo.add[0] = src_bgather(Pm, He, He, tp->mesh);
    fo.add[1] = src_bcast(Pe, He, He);
    GW_TRY(mlp_fwd(p, T, meb, fo, src_bcast(e_enc, De, De), ep_enc, De, &tp->edge));
  }
  tp->xg = xg, tp->e_enc = e_enc;
  if (!agg_m) return 0;
  if (r.whole) {
    GW_OTHER(launch_segsum(ep_enc, De, De, p->enc_ptr.p, p->enc_perm.p, N, H, B, agg_m, De, T->st));
  } else {  // whole slots: every slot's sum adds the rows of the unchunked sum, in its order
    const int ns = r.s1 - r.s0;
    GW_TALLOC(ag, (size_t)B * ns * De);
    GW_OTHER(launch_segsum(ep_enc, De, De, p->enc_ptr.p + r.s0, nullptr, n, ns, B, ag, De, T->st, r.r0));
    GW_OTHER(launch_permute_rows(ag, De, T->iota.p + r.s0, ns, H, De, B, agg_m, De, true, T->st));
  }
  return 0;
}

// backward of enc_fwd's block edge MLP and edge encoder: weight gradients, this range's rows of dPm [H, He] (the gradient of Pm,
// summed over the batch), and d_xg (the gradient of xg, left for enc_node_bwd)
static int enc_bwd(gw_plan* p, TrainState* T, const GridRange& r, const EncTape& tp, const float* d_agg_m, float* dPm, float** d_xg_out) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, N = p->n_in_cur, H = d.n_mesh, B = T->tp->batch, n = enc_rows(p, r),
            ad = d.enc_edge_attr_dim;
  const Mlp& meb = p->enc_blk_edge;
  GW_TALLOC(d_epe, (size_t)B * n * De);
  GW_OTHER(launch_gather_rows(d_agg_m, De, H, tp.mesh, n, De, B, d_epe, De, false, T->st));
  GW_TALLOC(d_e_enc, (size_t)n * De);
  GW_OTHER(launch_batch_reduce(d_epe, De, n, De, B, d_e_enc, De, false, T->st));
  float* dh = nullptr;
  GW_TRY(mlp_bwd(p, T, meb, tp.edge, d_epe, De, &dh));
  GW_TRY(train_wgrad(p, T, dh, He, He, src_stream(tp.xg, Dn, Dn, n), Dn, n, B, grad_of(p, T, meb.W[0]), meb.in[0], grad_of(p, T, meb.b[0])));
  GW_TALLOC(d_xg, (size_t)B * n * Dn);
  GW_TRY(dgrad(p, T, dh, He, He, n, B, meb.W[0], meb.out[0], 0, Dn, nullptr, 0, nullptr, 0, d_xg, Dn));
  if (r.whole) {
    GW_TALLOC(dPm_b, (size_t)B * H * He);
    GW_OTHER(launch_segsum(dh, He, He, p->enc_ptr.p, p->enc_perm.p, N, H, B, dPm_b, He, T->st));
    GW_OTHER(launch_batch_reduce(dPm_b, He, H, He, B, dPm, He, false, T->st));
  } else {  // the range owns its slots' rows of dPm
    const int ns = r.s1 - r.s0;
    GW_TALLOC(dPm_b, (size_t)B * ns * He);
    GW_OTHER(launch_segsum(dh, He, He, p->enc_ptr.p + r.s0, nullptr, n, ns, B, dPm_b, He, T->st, r.r0));
    GW_OTHER(launch_batch_reduce(dPm_b, He, ns, He, B, dPm + (size_t)r.s0 * He, He, false, T->st));
  }
  GW_TALLOC(dPe, (size_t)n * He);
  GW_OTHER(launch_batch_reduce(dh, He, n, He, B, dPe, He, false, T->st));
  GW_TRY(train_wgrad(p, T, dPe, He, He, src_stream(tp.e_enc, De, De, n), De, n, 1, grad_of(p, T, meb.W[0]) + 2 * Dn, meb.in[0], nullptr));
  GW_TRY(dgrad(p, T, dPe, He, He, n, 1, meb.W[0], meb.out[0], 2 * Dn, De, nullptr, 0, d_e_enc, De, d_e_enc, De));
  const Mlp& mee = p->enc_edge_enc;
  float* g0 = nullptr;
  GW_TRY(mlp_bwd(p, T, mee, tp.edge_enc, d_e_enc, De, &g0));
  GW_TRY(train_wgrad(p, T, g0, mee.out[0], mee.out[0], src_stream(tp.attr, ad, ad, n), ad, n, 1, grad_of(p, T, mee.W[0]), mee.in[0],
                     grad_of(p, T, mee.b[0])));
  *d_xg_out = d_xg;
  return 0;
}

// backward of node_encoder on the lat/lon rows; the feature gradient of each row goes to its point (through enc_perm in a chunk)
static int enc_node_bwd(gw_plan* p, TrainState* T, const GridRange& r, const EncTape& tp, const float* d_xg, float* dFeatures) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, N = p->n_in_cur, B = T->tp->batch, n = enc_rows(p, r);
  const Mlp& mne = p->enc_node;
  float* g0 = nullptr;
  GW_TRY(mlp_bwd(p, T, mne, tp.node_g, d_xg, Dn, &g0));
  GW_TRY(train_wgrad(p, T, g0, mne.out[0], mne.out[0], src_stream(tp.feat, d.in_dim, d.in_dim, n), d.in_dim, n, B, grad_of(p, T, mne.W[0]), mne.in[0],
                     grad_of(p, T, mne.b[0])));
  if (!dFeatures) return 0;
  if (r.whole) {
    GW_TRY(dgrad(p, T, g0, mne.out[0], mne.out[0], N, B, mne.W[0], mne.out[0], 0, d.in_dim, nullptr, 0, nullptr, 0, dFeatures, d.in_dim));
  } else {
    GW_TALLOC(df, (size_t)B * n * d.in_dim);
    GW_TRY(dgrad(p, T, g0, mne.out[0], mne.out[0], n, B, mne.W[0], mne.out[0], 0, d.in_dim, nullptr, 0, nullptr, 0, df, d.in_dim));
    GW_OTHER(launch_permute_rows(df, d.in_dim, p->enc_perm.p + r.r0, n, N, d.in_dim, B, dFeatures, d.in_dim, true, T->st));
  }
  return 0;
}

// decoder, lat/lon side: e_dec = edge_encoder(attr); e' = LN(MLP(h1)) + e_dec with h1 = relu(e_dec W1e^T + b1 + Pd[src]) (the lat/lon
// end of every decoder edge is a zero row: its W1d term vanishes); agg_g = per-point sums of e'; xg2 = LN(MLP(agg_g with W1[:, Dn:]))
// (the x half of the concat is identically zero); out = node_decoder(xg2) (+ features[..., :out_dim]).  out null: not stored.
static int dec_fwd(gw_plan* p, TrainState* T, const GridRange& r, const float* Pd, float* out, DecTape* tp) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = d.n_mesh, No = d.n_out, B = T->tp->batch, n = dec_rows(p, r),
            ne = dec_edges(p, r), r0 = r.whole ? 0 : r.r0, e0 = r.whole ? 0 : r.e0;
  RowSrc none;
  const Mlp& mde = p->dec_edge_enc;
  GW_TALLOC(e_dec, (size_t)ne * De);
  GW_TRY(mlp_fwd(p, T, mde, first_op(ne, 1, src_stream(p->dec_attr.p + (size_t)e0 * 2, 2, 2, ne), none, mde.W[0], mde.in[0], mde.in[0], mde.b[0]),
                 none, e_dec, De, &tp->edge_enc));
  const Mlp& mdb = p->dec_blk_edge;
  GW_TALLOC(ep_dec, (size_t)B * ne * De);
  {
    GemmOp fo = first_op(ne, B, src_bcast(e_dec, De, De), none, mdb.W[0] + 2 * Dn, De, mdb.in[0], mdb.b[0]);
    fo.add[0] = src_gather(Pd, He, He, p->dec_src.p + e0, H, 0);
    GW_TRY(mlp_fwd(p, T, mdb, fo, src_bcast(e_dec, De, De), ep_dec, De, &tp->edge));
  }
  GW_TALLOC(agg_g, (size_t)B * n * De);
  GW_OTHER(launch_segsum(ep_dec, De, De, p->dec_ptr.p + r0, nullptr, ne, n, B, agg_g, De, T->st, e0));
  const Mlp& mdn = p->dec_blk_node;
  GW_TALLOC(xg2, (size_t)B * n * Dn);
  GW_TRY(mlp_fwd(p, T, mdn, first_op(n, B, src_stream(agg_g, De, De, n), none, mdn.W[0] + Dn, De, mdn.in[0], mdn.b[0]), none, xg2, Dn, &tp->node));
  const Mlp& mdo = p->dec_node_dec;
  RowSrc res;
  float* o = out;
  const gw_tape* K = T->tp;
  if (r.whole) {
    if (d.residual_dim > 0) res = src_stream(K->start, K->start_ld, d.out_dim, No);
  } else {
    if (d.residual_dim > 0) {
      GW_TALLOC(fr, (size_t)B * n * d.out_dim);
      GW_OTHER(launch_permute_rows(K->start, K->start_ld, T->iota.p + r0, n, No, d.out_dim, B, fr, d.out_dim, false, T->st));
      res = src_stream(fr, d.out_dim, d.out_dim, n);
    }
    GW_TALLOC(oc, (size_t)B * n * d.out_dim);
    o = oc;
  }
  GW_TRY(mlp_fwd(p, T, mdo, first_op(n, B, src_stream(xg2, Dn, Dn, n), none, mdo.W[0], mdo.in[0], mdo.in[0], mdo.b[0]), res, o, d.out_dim, &tp->out));
  if (!r.whole && out) GW_OTHER(launch_permute_rows(o, d.out_dim, T->iota.p + r0, n, No, d.out_dim, B, out, d.out_dim, true, T->st));
  tp->e_dec = e_dec, tp->agg_g = agg_g, tp->xg2 = xg2;
  return 0;
}

// backward of dec_fwd: weight gradients, and the per-source sums of the edge MLP's dh1 added into dPd [B, H, He] (the first
// decoder chunk writes them, later ones add theirs in chunk order)
static int dec_bwd(gw_plan* p, TrainState* T, const GridRange& r, const DecTape& tp, const float* dOut, float* dPd) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = d.n_mesh, No = d.n_out, Ed = d.n_dec_edges, B = T->tp->batch, n = dec_rows(p, r),
            ne = dec_edges(p, r), r0 = r.whole ? 0 : r.r0, e0 = r.whole ? 0 : r.e0;
  const float* dO = dOut;
  if (!r.whole) {
    GW_TALLOC(dc, (size_t)B * n * d.out_dim);
    GW_OTHER(launch_permute_rows(dOut, d.out_dim, T->iota.p + r0, n, No, d.out_dim, B, dc, d.out_dim, false, T->st));
    dO = dc;
  }
  float* dh = nullptr;
  // node_decoder (the residual's share of d features is added at the end of the step)
  const Mlp& mdo = p->dec_node_dec;
  GW_TRY(mlp_bwd(p, T, mdo, tp.out, dO, d.out_dim, &dh));
  GW_TRY(train_wgrad(p, T, dh, mdo.out[0], mdo.out[0], src_stream(tp.xg2, Dn, Dn, n), Dn, n, B, grad_of(p, T, mdo.W[0]), mdo.in[0], grad_of(p, T, mdo.b[0])));
  GW_TALLOC(d_xg2, (size_t)B * n * Dn);
  GW_TRY(dgrad(p, T, dh, mdo.out[0], mdo.out[0], n, B, mdo.W[0], mdo.out[0], 0, Dn, nullptr, 0, nullptr, 0, d_xg2, Dn));
  // decoder node MLP
  const Mlp& mdn = p->dec_blk_node;
  GW_TRY(mlp_bwd(p, T, mdn, tp.node, d_xg2, Dn, &dh));
  GW_TRY(train_wgrad(p, T, dh, mdn.out[0], mdn.out[0], src_stream(tp.agg_g, De, De, n), De, n, B, grad_of(p, T, mdn.W[0]) + Dn, mdn.in[0],
                     grad_of(p, T, mdn.b[0])));
  GW_TALLOC(d_agg_g, (size_t)B * n * De);
  GW_TRY(dgrad(p, T, dh, mdn.out[0], mdn.out[0], n, B, mdn.W[0], mdn.out[0], Dn, De, nullptr, 0, nullptr, 0, d_agg_g, De));
  // decoder edge MLP: every edge receives its point's aggregate gradient
  const Mlp& mdb = p->dec_blk_edge;
  GW_TALLOC(d_ep, (size_t)B * ne * De);
  GW_OTHER(launch_gather_rows(d_agg_g, De, n, p->dec_dst.p + e0, ne, De, B, d_ep, De, false, T->st, r0));
  GW_TALLOC(d_e_dec, (size_t)ne * De);
  GW_OTHER(launch_batch_reduce(d_ep, De, ne, De, B, d_e_dec, De, false, T->st));  // residual: e_dec is shared by the batch
  GW_TRY(mlp_bwd(p, T, mdb, tp.edge, d_ep, De, &dh));                             // dh = dh1 [B*ne, He]
  // layer 0: e_dec is shared by the batch, so its terms use the batch-reduced gradient
  GW_TALLOC(dPe, (size_t)ne * He);
  GW_OTHER(launch_batch_reduce(dh, He, ne, He, B, dPe, He, false, T->st));
  GW_TRY(train_wgrad(p, T, dPe, He, He, src_stream(tp.e_dec, De, De, ne), De, ne, 1, grad_of(p, T, mdb.W[0]) + 2 * Dn, mdb.in[0], grad_of(p, T, mdb.b[0])));
  GW_TRY(dgrad(p, T, dPe, He, He, ne, 1, mdb.W[0], mdb.out[0], 2 * Dn, De, nullptr, 0, d_e_dec, De, d_e_dec, De));
  if (r.whole)
    GW_OTHER(launch_segsum(dh, He, He, T->dec_ptr_src.p, T->dec_perm_src.p, Ed, H, B, dPd, He, T->st));
  else
    GW_OTHER(launch_segsum(dh, He, He, T->dec_cptr.p + (size_t)r.c * (H + 1), T->dec_cperm.p + e0, ne, H, B, dPd, He, T->st, 0, r.c > 0));
  // decoder.edge_encoder
  const Mlp& mde = p->dec_edge_enc;
  float* g0 = nullptr;
  GW_TRY(mlp_bwd(p, T, mde, tp.edge_enc, d_e_dec, De, &g0));
  GW_TRY(train_wgrad(p, T, g0, mde.out[0], mde.out[0], src_stream(p->dec_attr.p + (size_t)e0 * 2, 2, 2, ne), 2, ne, 1, grad_of(p, T, mde.W[0]), mde.in[0],
                     grad_of(p, T, mde.b[0])));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// one processor block (the taped forward, the segmented forward and the segments' recompute in the backward all run these)
// ---------------------------------------------------------------------------------------------------------------------------
// the block's edge input e[k]: in block 0 of the whole network, e_lat broadcast over the batch
static RowSrc block_edge_src(TrainState* T, int k, const float* ek, int De, int El) {
  return (k == 0 && T->tp->g.e0_bcast) ? src_bcast(ek, De, De) : src_stream(ek, De, De, El);
}

// block k from x[k] (xk) and e[k] (ek), on the running tape's graph: P [B, H, 2 He] is the caller's scratch for the factored layer
// 1's node terms.  Allocates e[k+1], agg[k] and x[k+1], in that order, on the running tape; tpe / tpn receive the edge and node MLP
// tapes.  Block 0 of a standalone processor reads the caller's rows, and bounds them (train_op's reads_input).
static int block_fwd(gw_plan* p, TrainState* T, int k, const float* xk, const float* ek, float* P, float** en_out, float** ag_out, float** xn_out,
                     MlpTape* tpe, MlpTape* tpn) {
  const gw_dims& d = p->d;
  const LatGraph& g = T->tp->g;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = g.H, El = g.El, B = T->tp->batch;
  const bool in = k == 0 && T->tp->caller_input;
  RowSrc none;
  const Mlp& me = p->proc_edge[k];
  const Mlp& mn = p->proc_node[k];
  for (int h = 0; h < 2; ++h) {
    GemmOp t;
    t.rows_per_sample = H, t.batch = B, t.a[0] = src_stream(xk, Dn, Dn, H), t.W = me.W[0] + h * Dn, t.K = Dn, t.ldw = me.in[0], t.N = He;
    t.out = P + h * He, t.ldo = 2 * He;
    GW_TRY(train_op(p, T, t, TAG_TRAIN_FWD, in));
  }
  const RowSrc e_src = block_edge_src(T, k, ek, De, El);
  GW_TALLOC(en, (size_t)B * El * De);
  {
    GemmOp fo = first_op(El, B, e_src, none, me.W[0] + 2 * Dn, De, me.in[0], me.b[0]);
    fo.add[0] = src_gather(P, 2 * He, He, g.src, H, 0);
    fo.add[1] = src_gather(P, 2 * He, He, g.dst, H, He);
    GW_TRY(mlp_fwd(p, T, me, fo, e_src, en, De, tpe, in));
  }
  GW_TALLOC(ag, (size_t)B * H * De);
  GW_OTHER(launch_segsum(en, De, De, g.ptr, nullptr, El, H, B, ag, De, T->st));
  GW_TALLOC(xn, (size_t)B * H * Dn);
  GW_TRY(mlp_fwd(p, T, mn, first_op(H, B, src_stream(xk, Dn, Dn, H), src_stream(ag, De, De, H), mn.W[0], mn.in[0], mn.in[0], mn.b[0]),
                 src_stream(xk, Dn, Dn, H), xn, Dn, tpn, in));
  *en_out = en, *ag_out = ag, *xn_out = xn;
  return 0;
}

// backward of block k: dx / de are the gradients of x[k+1] / e[k+1] (de null: none flows into the last block's e'); xk, ek, agg,
// tpe, tpn what block_fwd read and kept.  Returns the gradients of x[k] and e[k] (allocated on the running tape).
static int block_bwd(gw_plan* p, TrainState* T, int k, const float* xk, const float* ek, const float* agg, const MlpTape& tpe, const MlpTape& tpn,
                     const float* dx, const float* de, float** dx_out, float** de_out) {
  const gw_dims& d = p->d;
  const LatGraph& g = T->tp->g;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = g.H, El = g.El, B = T->tp->batch;
  const cudaStream_t st = T->st;
  const Mlp& me = p->proc_edge[k];
  const Mlp& mn = p->proc_node[k];
  float* dh = nullptr;
  // node MLP: x[k+1] = LN(MLP([x[k] ; agg[k]])) + x[k]
  GW_TRY(mlp_bwd(p, T, mn, tpn, dx, Dn, &dh));
  GW_TRY(train_wgrad(p, T, dh, mn.out[0], mn.out[0], src_stream(xk, Dn, Dn, H), Dn, H, B, grad_of(p, T, mn.W[0]), mn.in[0], grad_of(p, T, mn.b[0])));
  GW_TRY(train_wgrad(p, T, dh, mn.out[0], mn.out[0], src_stream(agg, De, De, H), De, H, B, grad_of(p, T, mn.W[0]) + Dn, mn.in[0], nullptr));
  GW_TALLOC(dxk, (size_t)B * H * Dn);
  GW_TRY(dgrad(p, T, dh, mn.out[0], mn.out[0], H, B, mn.W[0], mn.out[0], 0, Dn, nullptr, 0, dx, Dn, dxk, Dn));  // + residual path
  GW_TALLOC(d_agg, (size_t)B * H * De);
  GW_TRY(dgrad(p, T, dh, mn.out[0], mn.out[0], H, B, mn.W[0], mn.out[0], Dn, De, nullptr, 0, nullptr, 0, d_agg, De));
  // e[k+1] receives its target's aggregate gradient (+ what the next block sent back)
  GW_TALLOC(d_en, (size_t)B * El * De);
  if (de) {
    GW_CUDA(cudaMemcpyAsync(d_en, de, (size_t)B * El * De * sizeof(float), cudaMemcpyDeviceToDevice, st));
    GW_OTHER(launch_gather_rows(d_agg, De, H, g.dst, El, De, B, d_en, De, true, st));
  } else {
    GW_OTHER(launch_gather_rows(d_agg, De, H, g.dst, El, De, B, d_en, De, false, st));
  }
  // edge MLP: e[k+1] = LN(...) + e[k];  h1 = relu(e[k] W1e^T + P_s[src] + P_d[dst] + b1)
  GW_TRY(mlp_bwd(p, T, me, tpe, d_en, De, &dh));
  const RowSrc e_src = block_edge_src(T, k, ek, De, El);
  GW_TRY(train_wgrad(p, T, dh, He, He, e_src, De, El, B, grad_of(p, T, me.W[0]) + 2 * Dn, me.in[0], grad_of(p, T, me.b[0])));
  GW_TALLOC(d_ek, (size_t)B * El * De);
  GW_TRY(dgrad(p, T, dh, He, He, El, B, me.W[0], me.out[0], 2 * Dn, De, nullptr, 0, d_en, De, d_ek, De));  // + residual path
  GW_TALLOC(dPs, (size_t)B * H * He);
  GW_TALLOC(dPt, (size_t)B * H * He);
  GW_OTHER(launch_segsum(dh, He, He, g.ptr_src, g.perm_src, El, H, B, dPs, He, st));
  GW_OTHER(launch_segsum(dh, He, He, g.ptr, nullptr, El, H, B, dPt, He, st));
  GW_TRY(train_wgrad(p, T, dPs, He, He, src_stream(xk, Dn, Dn, H), Dn, H, B, grad_of(p, T, me.W[0]), me.in[0], nullptr));
  GW_TRY(train_wgrad(p, T, dPt, He, He, src_stream(xk, Dn, Dn, H), Dn, H, B, grad_of(p, T, me.W[0]) + Dn, me.in[0], nullptr));
  GW_TALLOC(dx1, (size_t)B * H * Dn);
  GW_TRY(dgrad(p, T, dPs, He, He, H, B, me.W[0], me.out[0], 0, Dn, nullptr, 0, dxk, Dn, dx1, Dn));
  GW_TALLOC(dx2, (size_t)B * H * Dn);
  GW_TRY(dgrad(p, T, dPt, He, He, H, B, me.W[0], me.out[0], Dn, Dn, nullptr, 0, dx1, Dn, dx2, Dn));
  *dx_out = dx2, *de_out = d_ek;
  return 0;
}

// blocks per processor segment of a tape recorded with `segments` (0: no segments; -1 or >= num_blocks: one segment)
static int segment_blocks(int segments, int nb) { return (segments < 0 || segments >= nb) ? nb : segments; }

// the processor of a forward with segments: every block runs as in the taped step, but the tape keeps only x[k0], e[k0] at the
// start of each segment and the output x[nb]; a block's tapes and sums, and its inputs unless they start a segment, are released
// as soon as the block has run
static int proc_fwd_segmented(gw_plan* p, TrainState* T, gw_tape* K) {
  const gw_dims& d = p->d;
  const int He = d.hidden_edge, H = K->g.H, nb = d.num_blocks, B = K->batch, S = segment_blocks(K->segments, nb);
  GW_TALLOC(P, (size_t)B * H * 2 * He);
  float *x = K->x[0], *e = K->e[0];
  for (int k = 0; k < nb; ++k) {
    const size_t mark = K->allocs.size();
    float *en = nullptr, *ag = nullptr, *xn = nullptr;
    MlpTape tpe, tpn;
    GW_TRY(block_fwd(p, T, k, x, e, P, &en, &ag, &xn, &tpe, &tpn));
    tfree_except(T, mark, {en, xn});
    if (k % S != 0) tfree_one(T, x), tfree_one(T, e);
    x = xn, e = en;
    if ((k + 1) % S == 0 && k + 1 < nb) K->x[k + 1] = xn, K->e[k + 1] = en;
  }
  K->x[nb] = x;
  tfree_one(T, e);  // (no block reads e[nb])
  tfree_one(T, P);
  return 0;
}

// the processor's backward on a tape with segments, last segment first: each segment's blocks are recomputed from its kept x[k0],
// e[k0] with block_fwd, then differentiated last block first; a block's recomputed tape and backward temporaries are released once
// its backward has run.  Every recomputed row op measures its operand bound as the forward did (fp32), from fresh bound slots per
// block, so the recompute reproduces the forward's values and any segment length fits the slots.  dx: gradient of x[nb] in,
// x[0] out; de: gradient of e[0] out.
static int proc_bwd_segmented(gw_plan* p, TrainState* T, gw_tape* K, float** dx, float** de) {
  const gw_dims& d = p->d;
  const int He = d.hidden_edge, H = K->g.H, nb = d.num_blocks, B = K->batch, S = segment_blocks(K->segments, nb);
  float *gx = *dx, *ge = nullptr;
  for (int k1 = nb; k1 > 0;) {
    const int k0 = (k1 - 1) / S * S, n = k1 - k0;
    const float* gx_in = gx;
    const float* ge_in = ge;
    const size_t mark = K->allocs.size();
    std::vector<float*> xs(n + 1), es(n + 1), ags(n);
    std::vector<MlpTape> tpe(n), tpn(n);
    std::vector<size_t> bmark(n);
    GW_TALLOC(P, (size_t)B * H * 2 * He);
    xs[0] = K->x[k0], es[0] = K->e[k0];
    for (int j = 0; j < n; ++j) {
      bmark[j] = K->allocs.size();
      GW_TRY(reset_bounds(T));
      GW_TRY(block_fwd(p, T, k0 + j, xs[j], es[j], P, &es[j + 1], &ags[j], &xs[j + 1], &tpe[j], &tpn[j]));
    }
    for (int j = n - 1; j >= 0; --j) {
      GW_TRY(reset_bounds(T));
      float *gxn = nullptr, *gen = nullptr;
      GW_TRY(block_bwd(p, T, k0 + j, xs[j], es[j], ags[j], tpe[j], tpn[j], gx, ge, &gxn, &gen));
      tfree_except(T, bmark[j], {gxn, gen});  // block j's recompute, its temporaries, and the gradients block j + 1 sent it
      gx = gxn, ge = gen;
    }
    tfree_except(T, mark, {gx, ge});  // (P)
    tfree_one(T, gx_in), tfree_one(T, ge_in);
    k1 = k0;
  }
  *dx = gx, *de = ge;
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// the three stages of the step.  The whole network's forward and backward are their composition; each stage also runs alone, on a
// tape of its own, for the reference's standalone Encoder / Processor / Decoder (gw_train_{encoder,processor,decoder}_*_tape).
// A stage's forward keeps its activations on the running tape; the chunked step (training-only plans) keeps only the mesh-sized
// ones, the agg_m rows and the output.
// ---------------------------------------------------------------------------------------------------------------------------
// the start of a forward on tape K: its previous activations released (a second forward on a tape replaces the first's), the
// training state ready for the stages in `need`, the tape's processor on the plan's latent graph
static int forward_begin(gw_plan* p, TrainState* T, gw_tape* K, int stage, int need, int B, cudaStream_t st) {
  tape_release(T, K, st);
  if (T->cur_bytes == 0) T->peak_bytes = 0;  // no other tape holds memory: the high-water mark starts over
  T->tp = K;
  GW_TRY(train_prepare(p, T, B, need, st));
  GW_TRY(reset_bounds(T));
  K->batch = B, K->wgen = p->wgen, K->segments = p->train_segments, K->stage = stage, K->enc_gen = p->enc_graph_gen;
  K->graph_gen = p->graph_gen;
  K->features = nullptr, K->start = nullptr, K->start_ld = 0, K->xd = nullptr, K->caller_input = false;
  K->g = LatGraph();
  if (p->have_lat) {
    K->g.H = p->d.n_mesh, K->g.El = p->d.n_lat_edges;
    K->g.src = p->lat_src.p, K->g.dst = p->lat_dst.p, K->g.ptr = p->lat_ptr.p, K->g.perm_src = T->lat_perm_src.p, K->g.ptr_src = T->lat_ptr_src.p;
  }
  return 0;
}

// encoder: the features (K->features) -> x[0] [B, H, Dn] (*x0_out, on the tape) and e_lat [El, De] (K->e_lat: one sample's latent
// edge features, shared by the batch)
static int enc_stage_fwd(gw_plan* p, TrainState* T, gw_tape* K, float** x0_out) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = d.n_mesh, El = d.n_lat_edges, B = K->batch;
  RowSrc none;
  const bool chunked = p->train_only;
  // mesh rows: xm0 = node_encoder(h3_nodes), Pm = xm0 W1d^T (the mesh end of every encoder edge)
  const Mlp& mne = p->enc_node;
  GW_TALLOC(xm0, (size_t)H * Dn);
  GW_TRY(mlp_fwd(p, T, mne, first_op(H, 1, src_stream(p->h3_nodes, d.in_dim, d.in_dim, H), none, mne.W[0], mne.in[0], mne.in[0], mne.b[0]), none, xm0, Dn,
                 &K->t_enc_node_h));
  const Mlp& meb = p->enc_blk_edge;
  GW_TALLOC(Pm, (size_t)H * He);
  {
    GemmOp t;
    t.rows_per_sample = H, t.batch = 1, t.a[0] = src_stream(xm0, Dn, Dn, H), t.W = meb.W[0] + Dn, t.K = Dn, t.ldw = meb.in[0], t.N = He, t.out = Pm, t.ldo = He;
    GW_TRY(train_op(p, T, t, TAG_TRAIN_FWD));
  }
  GW_TALLOC(agg_m, (size_t)B * H * De);
  if (!chunked) {
    GW_TRY(enc_fwd(p, T, GridRange(), Pm, agg_m, &K->enc));
  } else {
    for (const GridRange& r : T->enc_chunks) {
      const size_t mark = K->allocs.size();
      GW_TRY(reset_bounds(T));
      EncTape tp;
      GW_TRY(enc_fwd(p, T, r, Pm, agg_m, &tp));
      tfree_to(T, mark);
    }
  }
  const Mlp& mnb = p->enc_blk_node;
  GW_TALLOC(x0, (size_t)B * H * Dn);
  GW_TRY(mlp_fwd(p, T, mnb, first_op(H, B, src_bcast(xm0, Dn, Dn), src_stream(agg_m, De, De, H), mnb.W[0], mnb.in[0], mnb.in[0], mnb.b[0]),
                 src_bcast(xm0, Dn, Dn), x0, Dn, &K->t_enc_mnode));
  const Mlp& mle = p->enc_lat_edge_enc;
  GW_TALLOC(e_lat, (size_t)El * De);
  GW_TRY(mlp_fwd(p, T, mle, first_op(El, 1, src_stream(p->lat_attr.p, 2, 2, El), none, mle.W[0], mle.in[0], mle.in[0], mle.b[0]), none, e_lat, De,
                 &K->t_lat_enc));
  K->xm0 = xm0, K->agg_m = agg_m, K->e_lat = e_lat, K->Pm = Pm;
  *x0_out = x0;
  return 0;
}

// processor: x[0] [B, H, Dn] and e[0] (e_lat broadcast over the batch, or [B, El, De] per edge: K->g.e0_bcast) -> x[nb] (K->x[nb],
// on the tape), on the tape's graph K->g.  x0 and e0 stay the caller's: the backward reads them again.
static int proc_stage_fwd(gw_plan* p, TrainState* T, gw_tape* K, const float* x0, const float* e0) {
  const int He = p->d.hidden_edge, H = K->g.H, nb = p->d.num_blocks, B = K->batch;
  K->x.assign(nb + 1, nullptr), K->e.assign(nb + 1, nullptr), K->agg.assign(nb, nullptr);
  K->t_pe.assign(nb, MlpTape()), K->t_pn.assign(nb, MlpTape());
  K->x[0] = const_cast<float*>(x0), K->e[0] = const_cast<float*>(e0);
  if (K->segments == 0) {
    GW_TALLOC(P, (size_t)B * H * 2 * He);
    for (int k = 0; k < nb; ++k)
      GW_TRY(block_fwd(p, T, k, K->x[k], K->e[k], P, &K->e[k + 1], &K->agg[k], &K->x[k + 1], &K->t_pe[k], &K->t_pn[k]));
  } else {
    K->agg.clear(), K->t_pe.clear(), K->t_pn.clear();
    GW_TRY(proc_fwd_segmented(p, T, K));
  }
  return 0;
}

// decoder: x [B, H, Dn] (K->xd, read again by the backward) -> out [B, n_out, out_dim] (+ the first out_dim columns of K->start
// when the plan has a residual)
static int dec_stage_fwd(gw_plan* p, TrainState* T, gw_tape* K, float* out) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, He = d.hidden_edge, H = d.n_mesh, B = K->batch;
  const Mlp& mdb = p->dec_blk_edge;
  GW_TALLOC(Pd, (size_t)B * H * He);
  {
    GemmOp t;
    t.rows_per_sample = H, t.batch = B, t.a[0] = src_stream(K->xd, Dn, Dn, H), t.W = mdb.W[0], t.K = Dn, t.ldw = mdb.in[0], t.N = He, t.out = Pd, t.ldo = He;
    GW_TRY(train_op(p, T, t, TAG_TRAIN_FWD, K->caller_input));
  }
  K->Pd = Pd;
  if (!p->train_only) {
    GW_TRY(dec_fwd(p, T, GridRange(), Pd, out, &K->dec));
  } else {
    for (const GridRange& r : T->dec_chunks) {
      const size_t mark = K->allocs.size();
      GW_TRY(reset_bounds(T));
      DecTape tp;
      GW_TRY(dec_fwd(p, T, r, Pd, out, &tp));
      tfree_to(T, mark);
    }
  }
  return 0;
}

// the whole network: encoder -> processor (block 0 reads e_lat broadcast) -> decoder with the features as the residual
static int train_forward(gw_plan* p, TrainState* T, gw_tape* K, const float* features, float* out, int B, cudaStream_t st) {
  GW_TRY(forward_begin(p, T, K, TAPE_NET, NEED_ENC | NEED_PROC | NEED_DEC, B, st));
  K->features = features, K->start = features, K->start_ld = p->d.in_dim;
  float* x0 = nullptr;
  GW_TRY(enc_stage_fwd(p, T, K, &x0));
  GW_TRY(proc_stage_fwd(p, T, K, x0, K->e_lat));
  K->xd = K->x[p->d.num_blocks];
  GW_TRY(dec_stage_fwd(p, T, K, out));
  K->have_tape = true;
  return 0;
}

// the start of a backward on tape K: it holds the activations of a forward of `stage`, taken at the plan's current weights (and,
// for a standalone encoder, on its current encoder graph); the gradient buffer is cleared
static int backward_begin(gw_plan* p, TrainState* T, gw_tape* K, int stage, cudaStream_t st) {
  GW_CHECK(K->have_tape, "a training backward needs the activations of a preceding training forward on its tape (one backward per forward)");
  GW_CHECK(K->stage == stage, "this tape holds the activations of another kind of training forward (the whole network or another stage)");
  GW_CHECK(K->wgen == p->wgen, "training backward: the plan's weights were replaced (gw_plan_set_weights) after this tape's forward; "
                               "its gradient would be taken at other weights");
  GW_CHECK(stage != TAPE_ENC || K->enc_gen == p->enc_graph_gen,
           "encoder backward: the plan's encoder graph was replaced after this tape's forward; its gradient would be taken on another graph");
  GW_CHECK(stage == TAPE_PROC || (K->enc_gen == p->enc_graph_gen && K->graph_gen == p->graph_gen),
           "training backward: the plan's graphs or h3_nodes rows were replaced after this tape's forward (a later call on other regions); "
           "its gradient would be taken on other graphs");
  T->st = st;
  T->tp = K;
  if (p->train_only) GW_TRY(build_chunks(p, T, K->batch));  // (a tape of another batch size may have run since this one's forward)
  GW_TRY(reset_bounds(T));
  GW_CUDA(cudaMemsetAsync(T->gbuf.p, 0, T->gbuf.bytes(), st));
  return 0;
}

// decoder backward: dOut [B, n_out, out_dim] -> its weight gradients and the gradient of its input x (*dx_out [B, H, Dn], on the
// tape).  The residual's share of the start features' gradient is dOut itself, added by the caller.
static int dec_stage_bwd(gw_plan* p, TrainState* T, gw_tape* K, const float* dOut, float** dx_out) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, He = d.hidden_edge, H = d.n_mesh, B = K->batch;
  // lat/lon side, then the mesh end of its edges (dPd: gradient of Pd = x W1s^T)
  GW_TALLOC(dPd, (size_t)B * H * He);
  if (!p->train_only) {
    GW_TRY(dec_bwd(p, T, GridRange(), K->dec, dOut, dPd));
  } else {
    for (const GridRange& r : T->dec_chunks) {
      const size_t mark = K->allocs.size();
      GW_TRY(reset_bounds(T));
      DecTape tp;
      GW_TRY(dec_fwd(p, T, r, K->Pd, nullptr, &tp));
      GW_TRY(dec_bwd(p, T, r, tp, dOut, dPd));
      tfree_to(T, mark);
    }
  }
  const Mlp& mdb = p->dec_blk_edge;
  GW_TRY(train_wgrad(p, T, dPd, He, He, src_stream(K->xd, Dn, Dn, H), Dn, H, B, grad_of(p, T, mdb.W[0]), mdb.in[0], nullptr));
  GW_TALLOC(dx, (size_t)B * H * Dn);
  GW_TRY(dgrad(p, T, dPd, He, He, H, B, mdb.W[0], mdb.out[0], 0, Dn, nullptr, 0, nullptr, 0, dx, Dn));
  *dx_out = dx;
  return 0;
}

// processor backward, blocks last to first: dx (the gradient of x[nb]) -> its weight gradients and the gradients of x[0] (*dx0)
// and of e[0] (*de0, per sample and edge [B, El, De]), on the tape
static int proc_stage_bwd(gw_plan* p, TrainState* T, gw_tape* K, const float* dx_in, float** dx0, float** de0) {
  float* dx = const_cast<float*>(dx_in);  // (read only; the segmented backward releases it when it is the tape's)
  float* de = nullptr;                    // gradient of e[k+1] (none flows into the last block's e')
  if (K->segments == 0) {
    for (int k = p->d.num_blocks - 1; k >= 0; --k)
      GW_TRY(block_bwd(p, T, k, K->x[k], K->e[k], K->agg[k], K->t_pe[k], K->t_pn[k], dx, de, &dx, &de));
  } else {
    GW_TRY(proc_bwd_segmented(p, T, K, &dx, &de));
  }
  *dx0 = dx, *de0 = de;
  return 0;
}

// encoder backward: the gradients of x[0] (dx0 [B, H, Dn]) and of e_lat (d_elat [El, De], summed over the batch; null: none) ->
// its weight gradients and, if dFeatures is not null, the gradient of the features [B, n_in, in_dim]
static int enc_stage_bwd(gw_plan* p, TrainState* T, gw_tape* K, const float* dx0, const float* d_elat, float* dFeatures) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, N = p->n_in_cur, H = d.n_mesh, El = d.n_lat_edges, B = K->batch;
  const cudaStream_t st = T->st;
  const bool chunked = p->train_only;
  if (dFeatures) GW_CUDA(cudaMemsetAsync(dFeatures, 0, (size_t)B * N * d.in_dim * sizeof(float), st));
  float* dh = nullptr;
  if (d_elat) {  // back through latent_edge_encoder
    const Mlp& mle = p->enc_lat_edge_enc;
    float* g0 = nullptr;
    GW_TRY(mlp_bwd(p, T, mle, K->t_lat_enc, d_elat, De, &g0));
    GW_TRY(train_wgrad(p, T, g0, mle.out[0], mle.out[0], src_stream(p->lat_attr.p, 2, 2, El), 2, El, 1, grad_of(p, T, mle.W[0]), mle.in[0], grad_of(p, T, mle.b[0])));
  }
  // ---- encoder block, node MLP (mesh rows): x[0] = LN(MLP([xm0 ; agg_m])) + xm0 ------------------------------------------------
  const Mlp& mnb = p->enc_blk_node;
  GW_TALLOC(d_xm0, (size_t)H * Dn);
  GW_OTHER(launch_batch_reduce(dx0, Dn, H, Dn, B, d_xm0, Dn, false, st));  // residual: xm0 is shared by the batch
  GW_TRY(mlp_bwd(p, T, mnb, K->t_enc_mnode, dx0, Dn, &dh));
  GW_TRY(train_wgrad(p, T, dh, mnb.out[0], mnb.out[0], src_bcast(K->xm0, Dn, Dn), Dn, H, B, grad_of(p, T, mnb.W[0]), mnb.in[0], grad_of(p, T, mnb.b[0])));
  GW_TRY(train_wgrad(p, T, dh, mnb.out[0], mnb.out[0], src_stream(K->agg_m, De, De, H), De, H, B, grad_of(p, T, mnb.W[0]) + Dn, mnb.in[0], nullptr));
  {
    GW_TALLOC(t1, (size_t)B * H * Dn);
    GW_TRY(dgrad(p, T, dh, mnb.out[0], mnb.out[0], H, B, mnb.W[0], mnb.out[0], 0, Dn, nullptr, 0, nullptr, 0, t1, Dn));
    GW_OTHER(launch_batch_reduce(t1, Dn, H, Dn, B, d_xm0, Dn, true, st));
  }
  GW_TALLOC(d_agg_m, (size_t)B * H * De);
  GW_TRY(dgrad(p, T, dh, mnb.out[0], mnb.out[0], H, B, mnb.W[0], mnb.out[0], Dn, De, nullptr, 0, nullptr, 0, d_agg_m, De));
  // ---- encoder block, edge MLP and edge encoder (lat/lon rows); then the mesh end of its edges (dPm) ---------------------------------
  const Mlp& meb = p->enc_blk_edge;
  GW_TALLOC(dPm, (size_t)H * He);
  float* d_xg = nullptr;
  if (!chunked) {
    GW_TRY(enc_bwd(p, T, GridRange(), K->enc, d_agg_m, dPm, &d_xg));
  } else {  // (node_encoder's lat/lon rows go with their chunk's tape)
    for (const GridRange& r : T->enc_chunks) {
      const size_t mark = K->allocs.size();
      GW_TRY(reset_bounds(T));
      EncTape tp;
      GW_TRY(enc_fwd(p, T, r, K->Pm, nullptr, &tp));
      GW_TRY(enc_bwd(p, T, r, tp, d_agg_m, dPm, &d_xg));
      GW_TRY(enc_node_bwd(p, T, r, tp, d_xg, dFeatures));
      tfree_to(T, mark);
    }
  }
  GW_TRY(train_wgrad(p, T, dPm, He, He, src_stream(K->xm0, Dn, Dn, H), Dn, H, 1, grad_of(p, T, meb.W[0]) + Dn, meb.in[0], nullptr));
  GW_TRY(dgrad(p, T, dPm, He, He, H, 1, meb.W[0], meb.out[0], Dn, Dn, nullptr, 0, d_xm0, Dn, d_xm0, Dn));
  // node_encoder on the h3 rows, then (taped step) on the lat/lon rows
  {
    const Mlp& mne = p->enc_node;
    float* g0 = nullptr;
    GW_TRY(mlp_bwd(p, T, mne, K->t_enc_node_h, d_xm0, Dn, &g0));
    GW_TRY(train_wgrad(p, T, g0, mne.out[0], mne.out[0], src_stream(p->h3_nodes, d.in_dim, d.in_dim, H), d.in_dim, H, 1, grad_of(p, T, mne.W[0]), mne.in[0],
                       grad_of(p, T, mne.b[0])));
    if (p->params.count("encoder.h3_nodes"))  // h3_nodes is a learned parameter of the forecaster (encoder.py:113)
      GW_TRY(dgrad(p, T, g0, mne.out[0], mne.out[0], H, 1, mne.W[0], mne.out[0], 0, d.in_dim, nullptr, 0, nullptr, 0,
                   grad_of(p, T, p->h3_nodes), d.in_dim));
  }
  if (!chunked) GW_TRY(enc_node_bwd(p, T, GridRange(), K->enc, d_xg, dFeatures));
  return 0;
}

// the whole network's backward: decoder, processor, then the encoder with e[0]'s gradient summed over the batch (e_lat is
// broadcast), and the residual's share of the features' gradient
static int train_backward(gw_plan* p, TrainState* T, gw_tape* K, const float* dOut, float* dFeatures, cudaStream_t st) {
  const gw_dims& d = p->d;
  const int De = d.edge_dim, N = p->n_in_cur, El = d.n_lat_edges, B = K->batch;
  GW_TRY(backward_begin(p, T, K, TAPE_NET, st));
  float *dx = nullptr, *dx0 = nullptr, *de0 = nullptr;
  GW_TRY(dec_stage_bwd(p, T, K, dOut, &dx));
  GW_TRY(proc_stage_bwd(p, T, K, dx, &dx0, &de0));
  GW_TALLOC(d_elat, (size_t)El * De);
  GW_OTHER(launch_batch_reduce(de0, De, El, De, B, d_elat, De, false, st));
  GW_TRY(enc_stage_bwd(p, T, K, dx0, d_elat, dFeatures));
  if (dFeatures && d.residual_dim > 0)  // out = node_decoder(...) + features[..., :out]: the residual passes dOut straight through
    GW_OTHER(launch_strided_add(dOut, d.out_dim, dFeatures, d.in_dim, (long long)B * N, d.out_dim, st));
  tape_release(T, K, st);  // the backward consumes its tape
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// one stage alone (the reference's sub-modules, each trained on its own tape)
// ---------------------------------------------------------------------------------------------------------------------------
static int copy_rows(float* dst, const float* src, size_t floats, cudaStream_t st) {
  GW_CUDA(cudaMemcpyAsync(dst, src, floats * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

static int encoder_forward(gw_plan* p, TrainState* T, gw_tape* K, const float* features, float* x_out, float* e_lat_out, int B, cudaStream_t st) {
  const gw_dims& d = p->d;
  GW_TRY(forward_begin(p, T, K, TAPE_ENC, NEED_ENC, B, st));
  K->features = features;
  float* x0 = nullptr;
  GW_TRY(enc_stage_fwd(p, T, K, &x0));
  GW_TRY(copy_rows(x_out, x0, (size_t)B * d.n_mesh * d.node_dim, st));
  GW_TRY(copy_rows(e_lat_out, K->e_lat, (size_t)d.n_lat_edges * d.edge_dim, st));
  tfree_one(T, x0), tfree_one(T, K->e_lat);  // (the encoder's backward reads neither)
  K->e_lat = nullptr;
  K->have_tape = true;
  return 0;
}

static int encoder_backward(gw_plan* p, TrainState* T, gw_tape* K, const float* dx, const float* d_elat, float* dFeatures, cudaStream_t st) {
  GW_TRY(backward_begin(p, T, K, TAPE_ENC, st));
  GW_TRY(enc_stage_bwd(p, T, K, dx, d_elat, dFeatures));
  tape_release(T, K, st);
  return 0;
}

// the caller's graph is copied onto the tape, with its edges grouped by source: it may change from call to call, and several
// tapes may hold forwards on different graphs
static int processor_forward(gw_plan* p, TrainState* T, gw_tape* K, const float* x_in, float* x_out, const float* edge_attr, int n_nodes, int n_edges,
                             const int32_t* src, const int32_t* dst, const int32_t* ptr, cudaStream_t st) {
  const gw_dims& d = p->d;
  GW_TRY(forward_begin(p, T, K, TAPE_PROC, NEED_PROC, 1, st));
  const size_t E = n_edges, V = (size_t)n_nodes + 1;
  float* gbuf = talloc(T, 3 * E + 2 * V);
  GW_CHECK(gbuf != nullptr, "training step: out of device memory");
  int32_t* s = reinterpret_cast<int32_t*>(gbuf);
  int32_t *t = s + E, *pt = t + E, *perm = pt + V, *ps = perm + E;
  GW_CUDA(cudaMemcpyAsync(s, src, E * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(t, dst, E * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(pt, ptr, V * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  const size_t ws = sort_csr_workspace_bytes(n_edges);
  if (T->sort_ws.n < ws) GW_TRY(T->sort_ws.alloc(ws));
  GW_CUDA(launch_sort_csr(s, n_edges, n_nodes, perm, ps, T->sort_ws.p, T->sort_ws.n, st));
  K->g.H = n_nodes, K->g.El = n_edges, K->g.src = s, K->g.dst = t, K->g.ptr = pt, K->g.perm_src = perm, K->g.ptr_src = ps, K->g.e0_bcast = false;
  K->caller_input = true;
  GW_TRY(proc_stage_fwd(p, T, K, x_in, edge_attr));
  float* xo = K->x[d.num_blocks];
  GW_TRY(copy_rows(x_out, xo, (size_t)n_nodes * d.node_dim, st));
  tfree_one(T, xo);  // (no block's backward reads the output)
  K->x[d.num_blocks] = nullptr;
  K->have_tape = true;
  return 0;
}

static int processor_backward(gw_plan* p, TrainState* T, gw_tape* K, const float* grad_x_out, float* grad_x_in, float* grad_edge_attr, cudaStream_t st) {
  const gw_dims& d = p->d;
  GW_TRY(backward_begin(p, T, K, TAPE_PROC, st));
  float *dx0 = nullptr, *de0 = nullptr;
  GW_TRY(proc_stage_bwd(p, T, K, grad_x_out, &dx0, &de0));
  if (grad_x_in) GW_TRY(copy_rows(grad_x_in, dx0, (size_t)K->g.H * d.node_dim, st));
  if (grad_edge_attr) GW_TRY(copy_rows(grad_edge_attr, de0, (size_t)K->g.El * d.edge_dim, st));
  tape_release(T, K, st);
  return 0;
}

static int decoder_forward(gw_plan* p, TrainState* T, gw_tape* K, const float* x_in, const float* start, int start_ld, float* out, int B, cudaStream_t st) {
  GW_TRY(forward_begin(p, T, K, TAPE_DEC, NEED_DEC, B, st));
  K->xd = x_in, K->start = start, K->start_ld = start_ld, K->caller_input = true;
  GW_TRY(dec_stage_fwd(p, T, K, out));
  K->have_tape = true;
  return 0;
}

static int decoder_backward(gw_plan* p, TrainState* T, gw_tape* K, const float* grad_out, float* grad_x_in, cudaStream_t st) {
  const gw_dims& d = p->d;
  GW_TRY(backward_begin(p, T, K, TAPE_DEC, st));
  float* dx = nullptr;
  GW_TRY(dec_stage_bwd(p, T, K, grad_out, &dx));
  if (grad_x_in) GW_TRY(copy_rows(grad_x_in, dx, (size_t)K->batch * d.n_mesh * d.node_dim, st));
  tape_release(T, K, st);
  return 0;
}

}  // namespace gw

void gw::train_destroy(gw_plan* p) {
  gw::TrainState* T = p->train;
  if (!T) return;
  for (gw_tape* k : T->tapes) {  // every live tape's memory goes with the plan; the tapes stay as dead handles
    gw::tape_release(T, k, T->st);
    k->plan = nullptr;
  }
  delete T;
  p->train = nullptr;
}

extern "C" {

int gw_tape_create(gw_plan* p, gw_tape** out) {
  GW_CHECK(p && out, "null argument");
  if (!p->train) p->train = new gw::TrainState();  // the plan's training state, made on first use
  gw_tape* k = new gw_tape();
  k->plan = p;
  p->train->tapes.insert(k);
  *out = k;
  return 0;
}

int gw_tape_destroy(gw_tape* k, void* stream) {
  if (!k) return 0;
  if (gw_plan* p = k->plan) {
    GW_CUDA(cudaSetDevice(p->device));
    gw::tape_release(p->train, k, (cudaStream_t)stream);
    p->train->tapes.erase(k);
  }
  delete k;
  return 0;
}

int64_t gw_tape_bytes(const gw_tape* k) { return k ? (int64_t)k->bytes : 0; }

// a tape of plan p that is still alive (its plan not destroyed)
static int check_tape(gw_plan* p, gw_tape* k) {
  GW_CHECK(k != nullptr, "null tape");
  GW_CHECK(k->plan != nullptr, "this tape is dead: its plan was destroyed, and its activations with it");
  GW_CHECK(k->plan == p, "this tape belongs to another plan");
  return 0;
}

int gw_train_forward_tape(gw_plan* p, gw_tape* k, const float* features, float* out, int32_t batch, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_TRY(gw::check_ready(p, batch, gw::NEED_ENC | gw::NEED_PROC | gw::NEED_DEC));
  GW_CHECK(features && out, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = gw::train_forward(p, p->train, k, features, out, batch, st);
  if (rc) gw::tape_release(p->train, k, st);  // a refused forward leaves no tape
  return rc;
}

// gradients are handed out under the reference's parameter names, shaped like the parameters
static int hand_out_grads(gw_plan* p, const gw_param* grads, int32_t n, const char* what, cudaStream_t st) {
  for (int i = 0; i < n; ++i) {
    GW_CHECK(grads[i].name && grads[i].data, "malformed gw_param entry");
    auto it = p->params.find(grads[i].name);
    GW_CHECK(it != p->params.end(), std::string(what) + ": unknown parameter '" + grads[i].name + "'");
    const size_t cnt = (size_t)it->second.second.first * it->second.second.second;
    GW_CHECK((size_t)grads[i].rows * grads[i].cols == cnt, std::string(what) + ": shape of '" + grads[i].name + "' differs");
    GW_CUDA(cudaMemcpyAsync(const_cast<float*>(grads[i].data), p->train->gbuf.p + (it->second.first - p->wbuf.p), cnt * sizeof(float),
                            cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

int gw_train_backward_tape(gw_plan* p, gw_tape* k, const float* grad_out, float* grad_features, const gw_param* grads, int32_t n, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_CHECK(grad_out && (n == 0 || grads), "null argument");
  GW_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  GW_TRY(gw::train_backward(p, p->train, k, grad_out, grad_features, st));
  return hand_out_grads(p, grads, n, "gw_train_backward_tape", st);
}

// The stages alone.  The encoder and decoder run the step of their plan: the taped step on a gw_plan_create plan, the bounded one
// on a training-only plan (their grid-sized work chunked as in the whole network).  The processor has no grid-sized work, so its
// bounded step would be its taped one; its memory is bounded by processor segments, and it takes a gw_plan_create plan only.
static const char* const kProcPlan = "the processor's training calls run the taped step: they need a gw_plan_create plan, not a training-only one "
                                     "(bound its memory with gw_train_set_processor_segments)";

int gw_train_encoder_forward_tape(gw_plan* p, gw_tape* k, const float* features, float* x_out, float* e_lat_out, int32_t batch, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_TRY(gw::check_ready(p, batch, gw::NEED_ENC));
  GW_CHECK(features && x_out && e_lat_out, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = gw::encoder_forward(p, p->train, k, features, x_out, e_lat_out, batch, st);
  if (rc) gw::tape_release(p->train, k, st);
  return rc;
}

int gw_train_encoder_backward_tape(gw_plan* p, gw_tape* k, const float* grad_x, const float* grad_e_lat, float* grad_features, const gw_param* grads,
                                   int32_t n, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_CHECK(grad_x && (n == 0 || grads), "null argument");
  GW_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  GW_TRY(gw::encoder_backward(p, p->train, k, grad_x, grad_e_lat, grad_features, st));
  return hand_out_grads(p, grads, n, "gw_train_encoder_backward_tape", st);
}

int gw_train_processor_forward_tape(gw_plan* p, gw_tape* k, const float* x_in, float* x_out, const float* edge_attr, int32_t n_nodes, int32_t n_edges,
                                    const int32_t* src, const int32_t* dst, const int32_t* ptr, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_TRY(gw::check_ready(p, 1, gw::NEED_PROC));
  GW_CHECK(x_in && x_out && edge_attr && src && dst && ptr, "null argument");
  GW_CHECK(x_out != x_in, "the training forward reads x_in again in its backward: x_out must be another buffer");
  GW_CHECK(!p->train_only, kProcPlan);
  GW_CHECK(n_nodes >= 1 && n_edges >= 1, "the graph needs at least one node and one edge");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = gw::processor_forward(p, p->train, k, x_in, x_out, edge_attr, n_nodes, n_edges, src, dst, ptr, st);
  if (rc) gw::tape_release(p->train, k, st);
  return rc;
}

int gw_train_processor_backward_tape(gw_plan* p, gw_tape* k, const float* grad_x_out, float* grad_x_in, float* grad_edge_attr, const gw_param* grads,
                                     int32_t n, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_CHECK(grad_x_out && (n == 0 || grads), "null argument");
  GW_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  GW_TRY(gw::processor_backward(p, p->train, k, grad_x_out, grad_x_in, grad_edge_attr, st));
  return hand_out_grads(p, grads, n, "gw_train_processor_backward_tape", st);
}

int gw_train_decoder_forward_tape(gw_plan* p, gw_tape* k, const float* x_in, const float* start_features, int32_t start_ld, float* out, int32_t batch,
                                  void* stream) {
  GW_TRY(check_tape(p, k));
  GW_TRY(gw::check_ready(p, batch, gw::NEED_DEC));
  GW_CHECK(x_in && out, "null argument");
  GW_CHECK(p->d.residual_dim == 0 || (start_features && start_ld >= p->d.residual_dim), "start features required (decoder.py:93)");
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = gw::decoder_forward(p, p->train, k, x_in, start_features, start_ld, out, batch, st);
  if (rc) gw::tape_release(p->train, k, st);
  return rc;
}

int gw_train_decoder_backward_tape(gw_plan* p, gw_tape* k, const float* grad_out, float* grad_x_in, const gw_param* grads, int32_t n, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_CHECK(grad_out && (n == 0 || grads), "null argument");
  GW_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  GW_TRY(gw::decoder_backward(p, p->train, k, grad_out, grad_x_in, st));
  return hand_out_grads(p, grads, n, "gw_train_decoder_backward_tape", st);
}

int64_t gw_train_peak_bytes(const gw_plan* p) { return (p && p->train) ? (int64_t)p->train->peak_bytes : 0; }

int gw_train_set_processor_segments(gw_plan* p, int32_t segments) {
  GW_CHECK(p != nullptr, "null plan");
  GW_CHECK(segments >= -1, "processor segments must be -1 (the whole processor), 0 (none) or a positive number of blocks");
  p->train_segments = segments;
  return 0;
}

int gw_train_set_deterministic(gw_plan* p, int32_t on) {
  GW_CHECK(p != nullptr, "null plan");
  p->train_deterministic = on != 0;
  return 0;
}

int64_t gw_train_deterministic_bytes(const gw_plan* p) { return (p && p->train) ? (int64_t)p->train->det_ws.bytes() : 0; }

}  // extern "C"
