// gw_api.cu -- the C ABI of libgwb200.so (include/gw_b200.h): plan, graph / weight upload, weight-constant
// precompute, and the encode-process-decode forward expressed as chains of gw::GemmOp row ops.
//
// Algebra used (results equal the reference's up to fp32 summation order; SURVEY.md section 7 "dead work"):
//   * layer 1 of every edge MLP is factored   W1 [x_s ; x_d ; e] = W1s x_s + W1d x_d + W1e e      (graph_net_block.py:131)
//     so the per-edge K=768 contraction becomes two per-NODE products (P = x [W1s;W1d]^T) gathered in the epilogue
//     plus a K=256 per-edge product; in the decoder x_d == 0 (assimilator_decoder.py:84,189-193) and e is constant,
//     so layer 1 there needs no per-edge GEMM at all: relu(P[src] + E1).
//   * batch-invariant tensors are computed once per weight set: edge_encoder(edge_attr) for the three graphs
//     (encoder.py:206, :235-241; assimilator_decoder.py:175), node_encoder(h3_nodes) (encoder.py:199-205),
//     and the constant layer-1 terms C1_enc / E1_dec.
//   * rows whose results the reference discards are not computed: the encoder block's lat/lon node update
//     (encoder.py:221-223), the decoder block's mesh node update and node_decoder on mesh rows
//     (assimilator_decoder.py:195-199).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cmath>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/gw_b200.h"
#include "gw_internal.h"
#include "gw_ops.h"

namespace gw {

static thread_local std::string g_err;
static thread_local long long g_launches = 0;
void set_error(const std::string& msg) { g_err = msg; }
void count_launch(int n) { g_launches += n; }

#define GW_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      gw::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                            \
      return 1;                                                                                    \
    }                                                                                              \
  } while (0)
#define GW_CHECK(cond, msg)       \
  do {                            \
    if (!(cond)) {                \
      gw::set_error(msg);         \
      return 1;                   \
    }                             \
  } while (0)
#define GW_TRY(expr)        \
  do {                      \
    int _r = (expr);        \
    if (_r != 0) return _r; \
  } while (0)

struct Mlp {  // views into the plan-owned weight buffer; Linear l: W[l] [out_l, in_l], b[l] [out_l]
  int L = 0;  // hidden layers; there are L+1 Linear layers
  std::vector<const float*> W, b;
  std::vector<int> in, out;
  const float* ln_g = nullptr;
  const float* ln_b = nullptr;
  // magnitudes (filled by pack_tc_weights; tensor-core chains only): max |b[l]|, and the bound of the LayerNorm'd row
  std::vector<float> bmax;
  float ln_bound = 0.f;  // tc_ln_bound of the LayerNorm
};

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  int alloc(size_t count) {
    release();
    n = count;
    if (count == 0) return 0;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e != cudaSuccess) {
      set_error(std::string("cudaMalloc(") + std::to_string(count * sizeof(T)) + " B): " + cudaGetErrorString(e));
      p = nullptr;
      n = 0;
      return 1;
    }
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  size_t bytes() const { return n * sizeof(T); }
};

}  // namespace gw

using namespace gw;

namespace gw {
struct TrainState;
}

struct gw_plan {
  gw::TrainState* train = nullptr;  // training step state (gw_train.inl), created on first use
  bool train_only = false;          // gw_plan_create_train: graphs, weights and the bounded-memory (chunked) training step only
  int train_chunk_pts = 0;          // GW_B200_TRAIN_CHUNK: points per chunk of that step (0: from the shapes, gw_train.inl)
  gw_dims d;
  int device = 0;
  int n_in_cur = 0;
  unsigned enc_graph_gen = 0;  // bumped whenever the encoder graph is replaced (the training step's chunk tables are built per graph)
  unsigned wgen = 0;           // bumped by every gw_plan_set_weights (the training step's per-weight work and its tapes key on it)
  // graphs
  DevBuf<int32_t> enc_mesh, enc_perm, enc_ptr, lat_src, lat_dst, lat_ptr, dec_src, dec_ptr;
  DevBuf<float> enc_attr, lat_attr, dec_attr;
  bool have_enc = false, have_lat = false, have_dec = false;   // graphs uploaded
  bool w_enc = false, w_proc = false, w_dec = false;            // weight groups bound (standalone sub-modules bind one)
  // weights (plan-owned copy) and views
  DevBuf<float> wbuf;
  std::map<std::string, std::pair<const float*, std::pair<int64_t, int64_t>>> params;
  Mlp enc_node, enc_edge_enc, enc_lat_edge_enc, enc_blk_edge, enc_blk_node;
  Mlp dec_edge_enc, dec_blk_edge, dec_blk_node, dec_node_dec;
  std::vector<Mlp> proc_edge, proc_node;
  const float* h3_nodes = nullptr;  // [n_mesh, in_dim] or null (assimilator: zeros)
  DevBuf<float> zeros_h3;
  // weight constants
  DevBuf<float> e_enc, xm0, C1_enc, e_lat, e_dec, E1_dec, tmpP;
  DevBuf<float> S_dec;  // [n_out, De] tensor-core plans: per lat/lon point, the sum of e_dec over the point's decoder edges (the constant residual of
                        // the decoder's edge MLP, summed once per weight set instead of being read per edge in every forward)
  // scratch
  // scratch.  chunk = samples processed per pass through the encoder / decoder stages.
  int chunk = 1;
  DevBuf<float> bufA, bufB;   // [chunk*max_rows, max_hidden]   hidden-activation ping-pong of run_mlp
  DevBuf<float> rows_n;       // [chunk*max(n_in,n_out), Dn]    node-encoded lat/lon rows (encoder) / updated lat/lon rows (decoder)
  DevBuf<float> rows_e;       // [chunk*max(n_in,n_dec_edges), De]  updated edge features e' of the encoder / decoder block
  DevBuf<float> xbuf0, xbuf1; // [max_batch*n_mesh, Dn]         mesh node state, double buffered (Jacobi update)
  DevBuf<float> ebuf0, ebuf1; // [max_batch*n_lat_edges, De]    latent edge state, double buffered
  DevBuf<float> P;            // [max_batch*n_mesh, 2*He]       per-node layer-1 products [W1s x | W1d x]
  size_t total_bytes = 0;
  // tensor-core path: packed weight images (GMMA operand layout) and their descriptors
  struct TcMlp { TcWeights w0, w0b, w0c, w1, w2; };  // w0*: slices of the first Linear as each chain needs them
  DevBuf<unsigned char> tc_packed;
  DevBuf<float> tc_absmax;
  long long* trace_buf = nullptr;   // debug: device buffer [8][1024][2] handed to the next chain launched under trace_tag
  int trace_tag = -1;
  int32_t* tc_status_host = nullptr;  // 16 words, pinned + mapped: stays readable by the host after a device trap
  int32_t* tc_status_dev = nullptr;
  TcMlp tc_enc_node, tc_enc_edge, tc_enc_mnode, tc_dec_edge, tc_dec_node, tc_dec_out;
  bool tc_dec_out_ok = false;  // node_decoder fits the chain kernel (hidden_dec multiple of 64, 2 hidden layers)
  DevBuf<float> agg_mesh;     // [max_batch*n_mesh, De] per-mesh-node aggregation (segment sums) of the encoder / processor blocks
  DevBuf<float> agg_grid;     // [chunk*n_out, De] per-lat/lon-point aggregation of the decoder block
  std::vector<TcMlp> tc_proc_edge, tc_proc_node;
  // operand range of the tensor-core chains: one device float per tensor = a rigorous bound of its magnitudes (SL_*)
  DevBuf<float> bounds;
  // fused per-target sums (gw_tc3.cu F_SEG): target of every decoder edge, carry rows of segments cut by a tile quadrant
  DevBuf<int32_t> dec_dst;
  DevBuf<float> seg_carry;
  DevBuf<int> deg_stats, enc_deg;  // {longest, shortest} segment: scratch for host reads; the encoder graph's stays on the device
  int lat_maxdeg = 0, lat_mindeg = 0, dec_maxdeg = 0, dec_mindeg = 0;
  // H3 tables for the device-side observation graph (gw_graph.cu): plan-owned copies
  DevBuf<double> h3_frames, h3_lat, h3_lng;
  DevBuf<int32_t> h3_cell_of, h3_slot;
  DevBuf<unsigned char> obs_ws;
  gw::H3Tables h3;
  // chunk table + partial sums of the encoder's two-level segment sum (gw_simt.cu)
  DevBuf<int32_t> enc_chunk_seg, enc_chunk_j0, enc_seg_chunk0;
  DevBuf<float> enc_partial;
  int enc_max_chunks = 0;
  bool fuse_seg = true;
  // loss-boundary gather fused into the forecast chain (gw_plan_set_output_peers): byte offsets from `out` to its aliases
  int out_mode = 0, n_out_peers = 0;
  long long out_delta[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // optional per-launch CUDA-event timing (gw_timing_*): events are recorded on the launching stream
  bool timing = false;
  int cur_tag = 0;
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_used = 0;
  struct Stamp { int tag; cudaEvent_t a, b; };
  std::vector<Stamp> stamps;
};

namespace gw {

static RowSrc src_stream(const float* base, int ld, int width, int rows_per_sample, int col0 = 0) {
  RowSrc s;
  s.kind = SRC_STREAM, s.base = base, s.ld = ld, s.width = width, s.src_rows = rows_per_sample, s.col0 = col0;
  return s;
}
static RowSrc src_bcast(const float* base, int ld, int width, int col0 = 0) {
  RowSrc s;
  s.kind = SRC_BCAST, s.base = base, s.ld = ld, s.width = width, s.col0 = col0;
  return s;
}
static RowSrc src_gather(const float* base, int ld, int width, const int32_t* idx, int src_rows, int col0 = 0) {
  RowSrc s;
  s.kind = SRC_GATHER, s.base = base, s.ld = ld, s.width = width, s.idx = idx, s.src_rows = src_rows, s.col0 = col0;
  return s;
}
static RowSrc src_bgather(const float* base, int ld, int width, const int32_t* idx) {
  RowSrc s;
  s.kind = SRC_BGATHER, s.base = base, s.ld = ld, s.width = width, s.idx = idx;
  return s;
}
static RowSrc src_segsum(const float* base, int ld, int width, const int32_t* ptr, const int32_t* perm, int src_rows) {
  RowSrc s;
  s.kind = SRC_SEGSUM, s.base = base, s.ld = ld, s.width = width, s.ptr = ptr, s.perm = perm, s.src_rows = src_rows;
  return s;
}
static RowSrc src_gather_bcast_relu(const float* base, int ld, int width, const int32_t* idx, int src_rows,
                                    const float* base2, int ld2) {
  RowSrc s;
  s.kind = SRC_GATHER_BCAST_RELU, s.base = base, s.ld = ld, s.width = width, s.idx = idx, s.src_rows = src_rows;
  s.base2 = base2, s.ld2 = ld2;
  return s;
}

// magnitude-bound slots (gw_plan::bounds)
enum BoundSlot { SL_FEAT = 0, SL_XIN, SL_XOUT, SL_X0, SL_X1, SL_E0, SL_E1, SL_EIN, SL_P, SL_AGG_MESH, SL_AGG_GRID, SL_ROWS_N, SL_ROWS_E,
                 SL_EENC, SL_C1ENC, SL_XM0, SL_ELAT, SL_EDEC, SL_E1DEC, SL_SDEC, SL_COUNT };
static float* sl(gw_plan* p, int i) { return p->bounds.p + i; }
static RowSrc bounded(RowSrc s, const float* b, float mul = 1.f) {
  s.bound = b, s.bound_mul = mul;
  return s;
}
// |x| of a raw caller tensor -> slot (the slot is reset first: absmax accumulates with atomicMax)
static int raw_bound(gw_plan* p, int slot, const float* x, long long n, cudaStream_t st) {
  GW_CUDA(cudaMemsetAsync(sl(p, slot), 0, sizeof(float), st));
  GW_CUDA(launch_absmax_flat(x, n, sl(p, slot), st));
  return 0;
}

// (the training step's phases, gw_train.inl: taped forward products, data gradients, weight gradients, operand bounds, the
// memory-bound rest -- LayerNorm backward, segment sums, gathers, batch reductions -- and the per-weight work done once per weight
// upload: transposes and weight images)
enum KernelTag { TAG_CONST = 0, TAG_ENC_GRID, TAG_ENC_MESH, TAG_PROC_P, TAG_PROC_EDGE, TAG_PROC_NODE, TAG_DEC_P, TAG_DEC_EDGE,
                 TAG_DEC_NODE, TAG_TRAIN_FWD, TAG_TRAIN_DGRAD, TAG_TRAIN_WGRAD, TAG_TRAIN_PACK, TAG_TRAIN_OTHER, TAG_TRAIN_WEIGHTS,
                 TAG_COUNT };
static const char* kTagNames[TAG_COUNT] = {"const", "enc_grid", "enc_mesh", "proc_p", "proc_edge", "proc_node", "dec_p",
                                           "dec_edge", "dec_node", "train_fwd", "train_dgrad", "train_wgrad", "train_pack",
                                           "train_other", "train_weights"};

static cudaEvent_t take_event(gw_plan* p) {
  if (p->ev_used == p->ev_pool.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    p->ev_pool.push_back(e);
  }
  return p->ev_pool[p->ev_used++];
}
struct TimedLaunch {  // RAII bracket: records an event pair on `st` around one kernel launch when timing is on
  gw_plan* p;
  cudaStream_t st;
  cudaEvent_t a = nullptr, b = nullptr;
  TimedLaunch(gw_plan* p_, cudaStream_t st_) : p(p_), st(st_) {
    if (p->timing) {
      a = take_event(p), b = take_event(p);
      cudaEventRecord(a, st);
    }
  }
  ~TimedLaunch() {
    if (p->timing) {
      cudaEventRecord(b, st);
      p->stamps.push_back({p->cur_tag, a, b});
    }
  }
};

static int run_op(gw_plan* p, const GemmOp& op, cudaStream_t st) {
  cudaError_t e;
  {
    TimedLaunch t(p, st);
    e = launch_rowop_simt(op, st);
  }
  if (e != cudaSuccess) {
    set_error(std::string("row-op launch failed: ") + cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

static int run_chain(gw_plan* p, TcChain& ch, cudaStream_t st) {
  ch.split = (p->d.precision == GW_PREC_FP32_TC) ? 1 : 0;
  ch.status = p->tc_status_dev;
#ifdef GW_ABLATE
  {
    const char* abl = getenv("GW_ABLATE");  // re-read per launch: tools/ablate.py sweeps masks in one process
    ch.ablate = abl ? atoi(abl) : 0;
  }
#endif
  if (p->trace_buf && p->cur_tag == p->trace_tag) {
    ch.trace = p->trace_buf;
    p->trace_buf = nullptr;  // one launch only
  }
  cudaError_t e;
  {
    TimedLaunch t(p, st);
    e = launch_chain_tc3(ch, st);
  }
  if (e != cudaSuccess) {
    set_error(std::string("tensor-core chain launch failed: ") + cudaGetErrorString(e));
    return 1;
  }
  return 0;
}
static bool is_tc(const gw_plan* p) { return p->d.precision != GW_PREC_FP32_SIMT; }

// layer = Linear `w` (+ bias b[l] of MLP m when l >= 0) (+ ReLU); magnitudes for the operand-range ladder travel along
static TcLayer tc_layer(const TcWeights& w, const Mlp* m, int l, bool relu, bool feeds) {
  TcLayer L;
  L.Wp = w.p, L.K = w.K, L.N = w.N, L.N32 = w.N32, L.n_valid = w.n_valid, L.wscale_inv = w.winv;
  L.bias = (m && l >= 0) ? m->b[l] : nullptr, L.relu = relu ? 1 : 0, L.feeds_next = feeds ? 1 : 0;
  L.gain = w.gain, L.off = (m && l >= 0 && (size_t)l < m->bmax.size()) ? m->bmax[l] : 0.f;
  return L;
}
static void tc_ln(TcLayer& L, const Mlp& m, const RowSrc& residual) {
  L.ln_g = m.ln_g, L.ln_b = m.ln_b, L.residual = residual, L.ln_bound = m.ln_bound;
}
static void tc_out(TcLayer& L, float* out, int ldo, int cols, float* bound = nullptr) { L.out = out, L.ldo = ldo, L.out_cols = cols, L.out_bound = bound; }

// Runs an MLP whose first Linear is described by `first` (A sources / addends / weight slice already set; its
// W/K/ldw/bias may have been overridden by the caller for factored layer 1) and whose remaining layers stream
// through the ping-pong scratch.  If `first_is_virtual`, layer 0 has already been applied by the A-assembly of
// `first` (decoder edge MLP: relu(P[src]+E1)) and `first` describes Linear 1.
static int run_mlp(gw_plan* p, const Mlp& m, GemmOp first, bool first_is_virtual, bool use_ln, const RowSrc& residual,
                   float* out, int ldo, cudaStream_t st) {
  const int rows = first.rows_per_sample, batch = first.batch;
  float* ping = p->bufA.p;
  float* pong = p->bufB.p;
  const int l0 = first_is_virtual ? 1 : 0;
  for (int l = l0; l <= m.L; ++l) {
    GemmOp op;
    if (l == l0) {
      op = first;
    } else {
      op.rows_per_sample = rows, op.batch = batch;
      op.a[0] = src_stream(ping, m.in[l], m.in[l], rows);
      op.W = m.W[l], op.K = m.in[l], op.ldw = m.in[l], op.bias = m.b[l];
    }
    op.N = m.out[l];
    if (l < m.L) {
      op.relu = 1;
      op.out = pong, op.ldo = m.out[l];
    } else {
      op.relu = 0;
      if (use_ln) op.ln_gamma = m.ln_g, op.ln_beta = m.ln_b;
      op.residual = residual;
      op.out = out, op.ldo = ldo;
    }
    GW_TRY(run_op(p, op, st));
    std::swap(ping, pong);
  }
  return 0;
}

static GemmOp first_op(int rows, int batch, const RowSrc& a0, const RowSrc& a1, const float* W, int K, int ldw,
                       const float* bias) {
  GemmOp op;
  op.rows_per_sample = rows, op.batch = batch;
  op.a[0] = a0, op.a[1] = a1;
  op.W = W, op.K = K, op.ldw = ldw, op.bias = bias;
  return op;
}

// ---------------------------------------------------------------------------------------------------------------
// weight lookup
// ---------------------------------------------------------------------------------------------------------------
static int find_param(gw_plan* p, const std::string& name, int64_t rows, int64_t cols, const float** out) {
  auto it = p->params.find(name);
  if (it == p->params.end()) {
    set_error("missing parameter '" + name + "'");
    return 1;
  }
  if (it->second.second.first != rows || it->second.second.second != cols) {
    set_error("parameter '" + name + "' has shape [" + std::to_string(it->second.second.first) + "," +
              std::to_string(it->second.second.second) + "], expected [" + std::to_string(rows) + "," +
              std::to_string(cols) + "]");
    return 1;
  }
  *out = it->second.first;
  return 0;
}

static int bind_mlp(gw_plan* p, const std::string& prefix, int in_dim, int hidden, int out_dim, int L, bool norm, Mlp* m) {
  m->L = L;
  m->W.assign(L + 1, nullptr), m->b.assign(L + 1, nullptr), m->in.assign(L + 1, 0), m->out.assign(L + 1, 0);
  int d = in_dim;
  for (int l = 0; l <= L; ++l) {
    int o = (l < L) ? hidden : out_dim;
    std::string k = prefix + ".model." + std::to_string(2 * l);
    GW_TRY(find_param(p, k + ".weight", o, d, &m->W[l]));
    GW_TRY(find_param(p, k + ".bias", o, 1, &m->b[l]));
    m->in[l] = d, m->out[l] = o;
    d = o;
  }
  if (norm) {
    std::string k = prefix + ".model." + std::to_string(2 * L + 1);
    GW_TRY(find_param(p, k + ".weight", out_dim, 1, &m->ln_g));
    GW_TRY(find_param(p, k + ".bias", out_dim, 1, &m->ln_b));
  }
  return 0;
}

static int bind_all(gw_plan* p) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, Hn = d.hidden_node, He = d.hidden_edge;
  const int Ln = d.hidden_layers_node, Le = d.hidden_layers_edge;
  auto has = [&](const char* k) { return p->params.count(k) != 0; };
  p->w_enc = p->w_proc = p->w_dec = false;
  if (has("encoder.node_encoder.model.0.weight")) {
    GW_TRY(bind_mlp(p, "encoder.node_encoder", d.in_dim, Hn, Dn, Ln, true, &p->enc_node));
    GW_TRY(bind_mlp(p, "encoder.edge_encoder", d.enc_edge_attr_dim, He, De, Le, true, &p->enc_edge_enc));
    GW_TRY(bind_mlp(p, "encoder.latent_edge_encoder", 2, He, De, Le, true, &p->enc_lat_edge_enc));
    GW_TRY(bind_mlp(p, "encoder.graph_processor.blocks.0.edge_model.edge_mlp", 2 * Dn + De, He, De, Le, true, &p->enc_blk_edge));
    GW_TRY(bind_mlp(p, "encoder.graph_processor.blocks.0.node_model.node_mlp", Dn + De, Hn, Dn, Ln, true, &p->enc_blk_node));
    if (has("encoder.h3_nodes")) {
      GW_TRY(find_param(p, "encoder.h3_nodes", d.n_mesh, d.in_dim, &p->h3_nodes));
    } else {  // AssimilatorEncoder keeps h3_nodes as a plain zero tensor (assimilator_encoder.py:80)
      p->h3_nodes = p->zeros_h3.p;
    }
    p->w_enc = true;
  }
  if (has("processor.graph_processor.blocks.0.edge_model.edge_mlp.model.0.weight")) {
    p->proc_edge.assign(d.num_blocks, Mlp()), p->proc_node.assign(d.num_blocks, Mlp());
    for (int b = 0; b < d.num_blocks; ++b) {
      std::string pre = "processor.graph_processor.blocks." + std::to_string(b);
      GW_TRY(bind_mlp(p, pre + ".edge_model.edge_mlp", 2 * Dn + De, He, De, Le, true, &p->proc_edge[b]));
      GW_TRY(bind_mlp(p, pre + ".node_model.node_mlp", Dn + De, Hn, Dn, Ln, true, &p->proc_node[b]));
    }
    p->w_proc = true;
  }
  if (has("decoder.edge_encoder.model.0.weight")) {
    GW_TRY(bind_mlp(p, "decoder.edge_encoder", 2, He, De, 2, true, &p->dec_edge_enc));  // 2 hidden layers hard-coded: assimilator_decoder.py:109
    GW_TRY(bind_mlp(p, "decoder.graph_processor.blocks.0.edge_model.edge_mlp", 2 * Dn + De, He, De, Le, true, &p->dec_blk_edge));
    GW_TRY(bind_mlp(p, "decoder.graph_processor.blocks.0.node_model.node_mlp", Dn + De, Hn, Dn, Ln, true, &p->dec_blk_node));
    // (no norm in the forecaster / assimilator decoders, decoder.py / assimilator_decoder.py; the regional forecaster builds its
    // node decoder WITH the configured norm, regional_forecast.py:224-231: bound when its parameters are present)
    const bool nd_norm = has(("decoder.node_decoder.model." + std::to_string(2 * d.hidden_layers_dec + 1) + ".weight").c_str());
    GW_TRY(bind_mlp(p, "decoder.node_decoder", Dn, d.hidden_dec, d.out_dim, d.hidden_layers_dec, nd_norm, &p->dec_node_dec));
    p->w_dec = true;
  }
  GW_CHECK(p->w_enc || p->w_proc || p->w_dec, "no encoder./processor./decoder. parameter group found in the table");
  return 0;
}

// Packs every weight panel the tensor-core chains stream.  Each panel is scaled by a power of two chosen from its
// largest magnitude so that the fp16 lo parts of the split stay normal; the inverse scale is applied in the epilogue.
static int pack_tc_weights(gw_plan* p, cudaStream_t st) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim;
  const int parts = (d.precision == GW_PREC_FP32_TC) ? 2 : 1;
  struct Req { const float* W; int ldw, K, N; TcWeights* out; };
  std::vector<Req> reqs;
  auto want = [&](const float* W, int ldw, int K, int N, TcWeights* out) { reqs.push_back({W, ldw, K, N, out}); };
  auto tail = [&](const Mlp& m, gw_plan::TcMlp& t) {
    want(m.W[1], m.in[1], m.in[1], m.out[1], &t.w1);
    want(m.W[2], m.in[2], m.in[2], m.out[2], &t.w2);
  };
  if (p->w_enc) {
    want(p->enc_node.W[0], d.in_dim, d.in_dim, p->enc_node.out[0], &p->tc_enc_node.w0);
    tail(p->enc_node, p->tc_enc_node);
    want(p->enc_blk_edge.W[0], p->enc_blk_edge.in[0], Dn, p->enc_blk_edge.out[0], &p->tc_enc_edge.w0);  // src slice
    tail(p->enc_blk_edge, p->tc_enc_edge);
    want(p->enc_blk_node.W[0], p->enc_blk_node.in[0], Dn + De, p->enc_blk_node.out[0], &p->tc_enc_mnode.w0);
    tail(p->enc_blk_node, p->tc_enc_mnode);
  }
  if (p->w_proc) {
    p->tc_proc_edge.assign(d.num_blocks, gw_plan::TcMlp()), p->tc_proc_node.assign(d.num_blocks, gw_plan::TcMlp());
    for (int k = 0; k < d.num_blocks; ++k) {
      const Mlp& me = p->proc_edge[k];
      want(me.W[0], me.in[0], Dn, me.out[0], &p->tc_proc_edge[k].w0);            // W1s
      want(me.W[0] + Dn, me.in[0], Dn, me.out[0], &p->tc_proc_edge[k].w0b);      // W1d
      want(me.W[0] + 2 * Dn, me.in[0], De, me.out[0], &p->tc_proc_edge[k].w0c);  // W1e
      tail(me, p->tc_proc_edge[k]);
      const Mlp& mn = p->proc_node[k];
      want(mn.W[0], mn.in[0], Dn + De, mn.out[0], &p->tc_proc_node[k].w0);
      tail(mn, p->tc_proc_node[k]);
    }
  }
  if (p->w_dec) {
    want(p->dec_blk_edge.W[0], p->dec_blk_edge.in[0], Dn, p->dec_blk_edge.out[0], &p->tc_dec_edge.w0);  // W1s
    tail(p->dec_blk_edge, p->tc_dec_edge);
    want(p->dec_blk_node.W[0] + Dn, p->dec_blk_node.in[0], De, p->dec_blk_node.out[0], &p->tc_dec_node.w0);  // agg half
    tail(p->dec_blk_node, p->tc_dec_node);
    const Mlp& md = p->dec_node_dec;
    p->tc_dec_out_ok = md.L == 2 && (d.hidden_dec % 64 == 0) && d.hidden_dec <= 256 && d.out_dim <= 256 && !md.ln_g;  // (a LayerNorm over out_dim columns: CUDA cores)
    if (p->tc_dec_out_ok) {
      want(md.W[0], md.in[0], md.in[0], md.out[0], &p->tc_dec_out.w0);
      tail(md, p->tc_dec_out);
    }
  }
  // bias / LayerNorm parameter magnitudes of every MLP a chain runs (operand-range ladder, gw_tc3.cu)
  struct VReq { const float* v; int n; Mlp* m; int what, l; };  // what: 0 = bias l, 1 = gamma, 2 = beta
  std::vector<VReq> vreqs;
  auto want_mlp = [&](Mlp& m) {
    m.bmax.assign(m.L + 1, 0.f);
    m.ln_bound = 0.f;
    for (int l = 0; l <= m.L; ++l) vreqs.push_back({m.b[l], m.out[l], &m, 0, l});
    if (m.ln_g) vreqs.push_back({m.ln_g, m.out[m.L], &m, 1, 0}), vreqs.push_back({m.ln_b, m.out[m.L], &m, 2, 0});
  };
  if (p->w_enc) want_mlp(p->enc_node), want_mlp(p->enc_blk_edge), want_mlp(p->enc_blk_node);
  if (p->w_proc)
    for (int k = 0; k < d.num_blocks; ++k) want_mlp(p->proc_edge[k]), want_mlp(p->proc_node[k]);
  if (p->w_dec) want_mlp(p->dec_blk_edge), want_mlp(p->dec_blk_node), want_mlp(p->dec_node_dec);
  const size_t n = reqs.size(), nv = vreqs.size();
  GW_TRY(p->tc_absmax.alloc(n + nv));
  GW_CUDA(cudaMemsetAsync(p->tc_absmax.p, 0, (n + nv) * sizeof(float), st));
  size_t total = 0;
  for (size_t i = 0; i < n; ++i) {
    GW_CUDA(launch_absmax(reqs[i].W, reqs[i].ldw, reqs[i].K, reqs[i].N, p->tc_absmax.p + i, st));
    total += (tc_packed_bytes(reqs[i].K, reqs[i].N, parts) + 1023) / 1024 * 1024;
  }
  for (size_t i = 0; i < nv; ++i) GW_CUDA(launch_absmax(vreqs[i].v, vreqs[i].n, vreqs[i].n, 1, p->tc_absmax.p + n + i, st));
  std::vector<float> amax(n + nv);
  GW_CUDA(cudaMemcpyAsync(amax.data(), p->tc_absmax.p, (n + nv) * sizeof(float), cudaMemcpyDeviceToHost, st));
  GW_CUDA(cudaStreamSynchronize(st));
  for (size_t i = 0; i < nv; ++i) {
    const VReq& r = vreqs[i];
    if (r.what == 0) r.m->bmax[r.l] = amax[n + i];
    else if (r.what == 1) r.m->ln_bound = tc_ln_bound(r.n, amax[n + i], amax[n + i + 1]);  // (beta's entry follows gamma's)
  }
  if (p->tc_packed.n != total) GW_TRY(p->tc_packed.alloc(total));
  size_t off = 0;
  for (size_t i = 0; i < n; ++i) {
    const Req& r = reqs[i];
    *r.out = tc_weights(p->tc_packed.p + off, r.K, r.N, amax[i], parts);
    GW_CUDA(launch_pack_weights(r.W, r.ldw, r.K, r.N, 1.f / r.out->winv, parts, p->tc_packed.p + off, st));
    off += (tc_packed_bytes(r.K, r.N, parts) + 1023) / 1024 * 1024;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// weight-constant precompute
// ---------------------------------------------------------------------------------------------------------------
static int precompute_encoder_constants(gw_plan* p, cudaStream_t st) {
  p->cur_tag = TAG_CONST;
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge;
  const int N = p->n_in_cur;
  RowSrc none;
  // e_enc = edge_encoder(edge_attr)                                              encoder.py:206
  {
    const Mlp& m = p->enc_edge_enc;
    GemmOp f = first_op(N, 1, src_stream(p->enc_attr.p, d.enc_edge_attr_dim, d.enc_edge_attr_dim, N), none, m.W[0],
                        m.in[0], m.in[0], m.b[0]);
    GW_TRY(run_mlp(p, m, f, false, true, none, p->e_enc.p, De, st));
  }
  // C1_enc[p] = W1e e_enc[p] + W1d xm0[mesh(p)] + b1                              layer 1 of graph_net_block.py:131-133
  {
    const Mlp& m = p->enc_blk_edge;
    GemmOp t;  // tmpP = xm0 . W1d^T   [H, He]
    t.rows_per_sample = d.n_mesh, t.batch = 1;
    t.a[0] = src_stream(p->xm0.p, Dn, Dn, d.n_mesh);
    t.W = m.W[0] + Dn, t.K = Dn, t.ldw = m.in[0], t.N = He;
    t.out = p->tmpP.p, t.ldo = He;
    GW_TRY(run_op(p, t, st));
    GemmOp c;
    c.rows_per_sample = N, c.batch = 1;
    c.a[0] = src_stream(p->e_enc.p, De, De, N);
    c.W = m.W[0] + 2 * Dn, c.K = De, c.ldw = m.in[0], c.N = He, c.bias = m.b[0];
    c.add[0] = src_bgather(p->tmpP.p, He, He, p->enc_mesh.p);
    c.out = p->C1_enc.p, c.ldo = He;
    GW_TRY(run_op(p, c, st));
  }
  if (is_tc(p)) {
    GW_TRY(raw_bound(p, SL_EENC, p->e_enc.p, (long long)N * De, st));
    GW_TRY(raw_bound(p, SL_C1ENC, p->C1_enc.p, (long long)N * He, st));
  }
  return 0;
}

static int precompute_constants(gw_plan* p, cudaStream_t st) {
  p->cur_tag = TAG_CONST;
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge;
  RowSrc none;
  if (p->w_enc) {
    // xm0 = node_encoder(h3_nodes)                                                encoder.py:199-205 (mesh rows)
    const Mlp& m = p->enc_node;
    GemmOp f = first_op(d.n_mesh, 1, src_stream(p->h3_nodes, d.in_dim, d.in_dim, d.n_mesh), none, m.W[0], m.in[0],
                        m.in[0], m.b[0]);
    GW_TRY(run_mlp(p, m, f, false, true, none, p->xm0.p, Dn, st));
  }
  if (p->w_enc && p->have_lat) {
    // e_lat = latent_edge_encoder(edge_attr)                                      encoder.py:235-241
    const Mlp& m = p->enc_lat_edge_enc;
    GemmOp f = first_op(d.n_lat_edges, 1, src_stream(p->lat_attr.p, 2, 2, d.n_lat_edges), none, m.W[0], m.in[0], m.in[0], m.b[0]);
    GW_TRY(run_mlp(p, m, f, false, true, none, p->e_lat.p, De, st));
  }
  if (p->w_dec && p->have_dec) {
    // e_dec = decoder.edge_encoder(edge_attr); E1_dec = W1e e_dec + b1            assimilator_decoder.py:175
    const Mlp& m = p->dec_edge_enc;
    GemmOp f = first_op(d.n_dec_edges, 1, src_stream(p->dec_attr.p, 2, 2, d.n_dec_edges), none, m.W[0], m.in[0], m.in[0], m.b[0]);
    GW_TRY(run_mlp(p, m, f, false, true, none, p->e_dec.p, De, st));
    const Mlp& e = p->dec_blk_edge;
    GemmOp c;
    c.rows_per_sample = d.n_dec_edges, c.batch = 1;
    c.a[0] = src_stream(p->e_dec.p, De, De, d.n_dec_edges);
    c.W = e.W[0] + 2 * Dn, c.K = De, c.ldw = e.in[0], c.N = He, c.bias = e.b[0];
    c.out = p->E1_dec.p, c.ldo = He;
    GW_TRY(run_op(p, c, st));
    if (is_tc(p) && p->S_dec.p)  // sum_e (e_dec[e] + LN(..)) = S_dec[point] + sum_e LN(..): graph_net_block.py:133,188 reassociated
      GW_CUDA(launch_segsum(p->e_dec.p, De, De, p->dec_ptr.p, nullptr, d.n_dec_edges, d.n_out, 1, p->S_dec.p, De, st));
  }
  if (p->w_enc && p->have_enc) GW_TRY(precompute_encoder_constants(p, st));
  if (is_tc(p)) {  // magnitude bounds of the constant tensors the chains read (operand range, gw_tc3.cu)
    if (p->w_enc) GW_TRY(raw_bound(p, SL_XM0, p->xm0.p, (long long)d.n_mesh * Dn, st));
    if (p->w_enc && p->have_lat) GW_TRY(raw_bound(p, SL_ELAT, p->e_lat.p, (long long)d.n_lat_edges * De, st));
    if (p->w_dec && p->have_dec) {
      GW_TRY(raw_bound(p, SL_EDEC, p->e_dec.p, (long long)d.n_dec_edges * De, st));
      GW_TRY(raw_bound(p, SL_E1DEC, p->E1_dec.p, (long long)d.n_dec_edges * He, st));
      if (p->S_dec.p) GW_TRY(raw_bound(p, SL_SDEC, p->S_dec.p, (long long)d.n_out * De, st));
    }
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// stages
// ---------------------------------------------------------------------------------------------------------------
// Encoder.forward (encoder.py:197-242) for `nb` samples of `features`; writes x_out [nb*H, Dn].
static int stage_encoder(gw_plan* p, const float* features, float* x_out, float* x_out_bound, int nb, cudaStream_t st) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, N = p->n_in_cur, H = d.n_mesh;
  RowSrc none;
  if (is_tc(p)) GW_CUDA(cudaMemsetAsync(sl(p, SL_FEAT), 0, sizeof(float), st));
  for (int s0 = 0; s0 < nb; s0 += p->chunk) {
    const int cb = std::min(p->chunk, nb - s0);
    const float* f = features + (size_t)s0 * N * d.in_dim;
    float* xg = p->rows_n.p;
    float* eprime = p->rows_e.p;
    if (is_tc(p)) {
      // chain 1 (lat/lon rows): node_encoder (3 layers + LN) -> edge MLP of the encoder block (W1s . h + C1, 2 layers + LN)
      // + e_enc residual -> e' rows.  Six GEMMs per row without leaving the SM.
      p->cur_tag = TAG_ENC_GRID;
      {
        TcChain ch;
        ch.rows_per_sample = N, ch.batch = cb;
        ch.K0 = p->tc_enc_node.w0.K;
        if ((d.in_dim & 63) || (reinterpret_cast<uintptr_t>(f) & 15)) {
          // widen the feature rows to K0 (zero padded, 16-byte aligned) so that stage 0 takes the 128-bit path; the
          // lat/lon row buffer is free here (the whole encoder block runs inside this chain).  The same pass takes the
          // absolute maximum of the raw features: the chain scales its fp16-split operands from it.
          TimedLaunch t(p, st);
          GW_CUDA(launch_pad_rows(f, d.in_dim, d.in_dim, xg, ch.K0, (long long)cb * N, sl(p, SL_FEAT), st));
          ch.a0[0] = bounded(src_stream(xg, ch.K0, ch.K0, N), sl(p, SL_FEAT));
        } else {
          TimedLaunch t(p, st);
          GW_CUDA(launch_absmax_flat(f, (long long)cb * N * d.in_dim, sl(p, SL_FEAT), st));
          ch.a0[0] = bounded(src_stream(f, d.in_dim, d.in_dim, N), sl(p, SL_FEAT));
        }
        const Mlp &mn = p->enc_node, &me = p->enc_blk_edge;
        ch.layer[0] = tc_layer(p->tc_enc_node.w0, &mn, 0, true, true);
        ch.layer[1] = tc_layer(p->tc_enc_node.w1, &mn, 1, true, true);
        ch.layer[2] = tc_layer(p->tc_enc_node.w2, &mn, 2, false, true);
        tc_ln(ch.layer[2], mn, none);
        ch.layer[3] = tc_layer(p->tc_enc_edge.w0, nullptr, -1, true, true);
        ch.layer[3].add[0] = bounded(src_bcast(p->C1_enc.p, He, He), sl(p, SL_C1ENC));
        ch.layer[4] = tc_layer(p->tc_enc_edge.w1, &me, 1, true, true);
        ch.layer[5] = tc_layer(p->tc_enc_edge.w2, &me, 2, false, false);
        tc_ln(ch.layer[5], me, bounded(src_bcast(p->e_enc.p, De, De), sl(p, SL_EENC)));
        tc_out(ch.layer[5], eprime, De, De, sl(p, SL_ROWS_E));
        ch.n_layers = 6;
        GW_TRY(run_chain(p, ch, st));
      }
      // chain 2 (mesh rows): [xm0 | sum of incoming e'] -> node MLP + LN + residual -> x
      p->cur_tag = TAG_ENC_MESH;
      {
        TcChain ch;
        ch.rows_per_sample = H, ch.batch = cb;
        {  // the lat/lon -> mesh segments are very skewed (a polar cell collects thousands of points): reduced by their own kernel
          TimedLaunch t(p, st);
          if (De == 256 && p->enc_partial.p)
            GW_CUDA(launch_segsum_chunked(eprime, De, p->enc_ptr.p, p->enc_perm.p, N, H, cb, p->enc_chunk_seg.p, p->enc_chunk_j0.p,
                                          p->enc_seg_chunk0.p, p->enc_max_chunks, p->enc_partial.p, p->agg_mesh.p, De, st));
          else
            GW_CUDA(launch_segsum(eprime, De, De, p->enc_ptr.p, p->enc_perm.p, N, H, cb, p->agg_mesh.p, De, st));
        }
        ch.a0[0] = bounded(src_bcast(p->xm0.p, Dn, Dn), sl(p, SL_XM0));
        ch.a0[1] = bounded(src_stream(p->agg_mesh.p, De, De, H), sl(p, SL_ROWS_E));
        ch.a0[1].bound_mul_i = p->enc_deg.p;  // a sum of up to (longest lat/lon -> mesh segment) rows
        ch.K0 = Dn + De;
        const Mlp& m = p->enc_blk_node;
        ch.layer[0] = tc_layer(p->tc_enc_mnode.w0, &m, 0, true, true);
        ch.layer[1] = tc_layer(p->tc_enc_mnode.w1, &m, 1, true, true);
        ch.layer[2] = tc_layer(p->tc_enc_mnode.w2, &m, 2, false, false);
        tc_ln(ch.layer[2], m, bounded(src_bcast(p->xm0.p, Dn, Dn), sl(p, SL_XM0)));
        tc_out(ch.layer[2], x_out + (size_t)s0 * H * Dn, Dn, Dn, x_out_bound);
        ch.n_layers = 3;
        GW_TRY(run_chain(p, ch, st));
      }
      continue;
    }
    // node_encoder on the lat/lon rows (encoder.py:205); the mesh rows are the constant xm0
    p->cur_tag = TAG_ENC_GRID;
    {
      const Mlp& m = p->enc_node;
      GemmOp fo = first_op(N, cb, src_stream(f, d.in_dim, d.in_dim, N), none, m.W[0], m.in[0], m.in[0], m.b[0]);
      GW_TRY(run_mlp(p, m, fo, false, true, none, xg, Dn, st));
    }
    // edge update e' = LN(MLP([x_src ; x_dst ; e])) + e   (graph_net_block.py:131-135); dst and e terms are in C1_enc
    {
      const Mlp& m = p->enc_blk_edge;
      GemmOp fo = first_op(N, cb, src_stream(xg, Dn, Dn, N), none, m.W[0], Dn, m.in[0], nullptr);
      fo.add[0] = src_bcast(p->C1_enc.p, He, He);
      GW_TRY(run_mlp(p, m, fo, false, true, src_bcast(p->e_enc.p, De, De), eprime, De, st));
    }
    // mesh node update x' = LN(MLP([x ; sum_in e'])) + x   (graph_net_block.py:184-191), mesh rows only
    p->cur_tag = TAG_ENC_MESH;
    {
      const Mlp& m = p->enc_blk_node;
      GemmOp fo = first_op(H, cb, src_bcast(p->xm0.p, Dn, Dn),
                           src_segsum(eprime, De, De, p->enc_ptr.p, p->enc_perm.p, N), m.W[0], m.in[0], m.in[0], m.b[0]);
      GW_TRY(run_mlp(p, m, fo, false, true, src_bcast(p->xm0.p, Dn, Dn), x_out + (size_t)s0 * H * Dn, Dn, st));
    }
  }
  return 0;
}

// Processor.forward (processor.py:123-128): num_blocks message-passing blocks.  x_in [nb*H, Dn] -> x_out [nb*H, Dn].
// The graph (H nodes, El target-sorted edges) is shared by the nb samples.  e0 is the initial edge state:
// broadcast (one copy for every sample: the constant e_lat of encoder.py:235-241) or per-sample [nb*El, De].
struct ProcGraph {
  int H, El;
  const int32_t *src, *dst, *ptr;
  const float* e0;
  bool e0_broadcast;
  int maxdeg, mindeg;    // longest / shortest per-node segment of incoming edges
  const float* e0_bound; // magnitude bound of e0
};
static int stage_processor(gw_plan* p, const ProcGraph& g, const float* x_in, float* x_out, int x_in_slot, int x_out_slot, int nb,
                           cudaStream_t st) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = g.H, El = g.El;
  const float* x_cur = x_in;
  float* xb[2] = {p->xbuf0.p, p->xbuf1.p};
  float* eb[2] = {p->ebuf0.p, p->ebuf1.p};
  const float* e_cur = nullptr;  // null: block 0 reads e0
  bool p_ready = false;          // P of the coming block was produced by the previous block's node chain
  auto xs = [&](const float* buf) { return sl(p, buf == xb[0] ? SL_X0 : (buf == xb[1] ? SL_X1 : (buf == x_in ? x_in_slot : x_out_slot))); };
  auto es = [&](const float* buf) { return sl(p, buf == eb[0] ? SL_E0 : SL_E1); };
  // the per-node sums of e' are produced by the edge chain itself when every node collects at most 8 edges (icosahedral
  // meshes: 6 or 7); longer segments (arbitrary caller graphs) keep the separate reduction kernel
  const bool fuse = is_tc(p) && p->fuse_seg && g.maxdeg >= 1 && g.maxdeg <= 8;
  for (int k = 0; k < d.num_blocks; ++k) {
    const Mlp& me = p->proc_edge[k];
    const Mlp& mn = p->proc_node[k];
    if (is_tc(p)) {
      const bool last = k == d.num_blocks - 1;
      float* e_next = eb[k & 1];
      float* x_next = last ? x_out : xb[k & 1];
      if (x_next == x_cur) x_next = xb[(k & 1) ^ 1];
      const RowSrc e_src = e_cur ? bounded(src_stream(e_cur, De, De, El), es(e_cur))
                                 : bounded(g.e0_broadcast ? src_bcast(g.e0, De, De) : src_stream(g.e0, De, De, El), g.e0_bound);
      if (!p_ready) {  // P = x [W1s ; W1d]^T : two products of the same operand (block 0; later blocks: see the node chain)
        p->cur_tag = TAG_PROC_P;
        TcChain ch;
        ch.rows_per_sample = H, ch.batch = nb;
        ch.a0[0] = bounded(src_stream(x_cur, Dn, Dn, H), xs(x_cur));
        ch.K0 = Dn;
        ch.layer[0] = tc_layer(p->tc_proc_edge[k].w0, nullptr, -1, false, false);
        tc_out(ch.layer[0], p->P.p, 2 * He, He, sl(p, SL_P));
        ch.layer[1] = tc_layer(p->tc_proc_edge[k].w0b, nullptr, -1, false, false);
        ch.layer[1].reuse_a = 1;
        tc_out(ch.layer[1], p->P.p + He, 2 * He, He, sl(p, SL_P));
        ch.n_layers = 2;
        GW_TRY(run_chain(p, ch, st));
      }
      p->cur_tag = TAG_PROC_EDGE;
      {  // e' = LN(W3 relu(W2 relu(W1e e + b1 + P_s[src] + P_d[dst]) + b2) + b3) + e   (+ per-node sums of e' when fused)
        TcChain ch;
        ch.rows_per_sample = El, ch.batch = nb;
        ch.a0[0] = e_src;
        ch.K0 = De;
        ch.layer[0] = tc_layer(p->tc_proc_edge[k].w0c, &me, 0, true, true);
        ch.layer[0].add[0] = bounded(src_gather(p->P.p, 2 * He, He, g.src, H, 0), sl(p, SL_P));
        ch.layer[0].add[1] = bounded(src_gather(p->P.p, 2 * He, He, g.dst, H, He), sl(p, SL_P));
        ch.layer[1] = tc_layer(p->tc_proc_edge[k].w1, &me, 1, true, true);
        ch.layer[2] = tc_layer(p->tc_proc_edge[k].w2, &me, 2, false, false);
        tc_ln(ch.layer[2], me, e_src);
        if (!(fuse && last)) tc_out(ch.layer[2], e_next, De, De, es(e_next));  // (the last block's e' is only ever summed)
        if (fuse) {
          TcLayer& L = ch.layer[2];
          L.seg_dst = g.dst, L.seg_out = p->agg_mesh.p, L.seg_ld = De, L.seg_rows = H, L.seg_carry = p->seg_carry.p;
          L.seg_maxdeg = (float)g.maxdeg, L.seg_bound = sl(p, SL_AGG_MESH);
          if (g.mindeg == 0) GW_CUDA(cudaMemsetAsync(p->agg_mesh.p, 0, (size_t)nb * H * De * sizeof(float), st));  // nodes without edges
        }
        ch.n_layers = 3;
        GW_TRY(run_chain(p, ch, st));
      }
      p->cur_tag = TAG_PROC_NODE;
      if (fuse) {  // (timed with its consumer, like round 1's segment-sum launch: it completes the node chain's aggregate input)
        TimedLaunch t(p, st);
        GW_CUDA(launch_seg_carry(p->seg_carry.p, g.dst, El, H, nb, p->agg_mesh.p, De, st));
      }
      {  // x' = LN(MLP([x ; sum_in e'])) + x
        TcChain ch;
        ch.rows_per_sample = H, ch.batch = nb;
        if (!fuse) {  // per-node sum of incoming e' rows (contiguous CSR segments): coalesced reduction kernel
          TimedLaunch t(p, st);
          GW_CUDA(launch_segsum(e_next, De, De, g.ptr, nullptr, El, H, nb, p->agg_mesh.p, De, st));
        }
        ch.a0[0] = bounded(src_stream(x_cur, Dn, Dn, H), xs(x_cur));
        ch.a0[1] = fuse ? bounded(src_stream(p->agg_mesh.p, De, De, H), sl(p, SL_AGG_MESH))
                        : bounded(src_stream(p->agg_mesh.p, De, De, H), es(e_next), (float)std::max(g.maxdeg, 1));
        ch.K0 = Dn + De;
        ch.layer[0] = tc_layer(p->tc_proc_node[k].w0, &mn, 0, true, true);
        ch.layer[1] = tc_layer(p->tc_proc_node[k].w1, &mn, 1, true, true);
        ch.layer[2] = tc_layer(p->tc_proc_node[k].w2, &mn, 2, false, false);
        tc_ln(ch.layer[2], mn, bounded(src_stream(x_cur, Dn, Dn, H), xs(x_cur)));
        tc_out(ch.layer[2], x_next, Dn, Dn, xs(x_next));
        ch.n_layers = 3;
        p_ready = false;
        if (k + 1 < d.num_blocks && He == Dn) {
          // the next block's P = x' [W1s ; W1d]^T needs exactly the rows this chain has just produced: two more products
          // of the same operand, and the separate P launches (and their re-read of x') disappear
          ch.layer[2].feeds_next = 1;
          ch.layer[3] = tc_layer(p->tc_proc_edge[k + 1].w0, nullptr, -1, false, false);
          tc_out(ch.layer[3], p->P.p, 2 * He, He, sl(p, SL_P));
          ch.layer[4] = tc_layer(p->tc_proc_edge[k + 1].w0b, nullptr, -1, false, false);
          ch.layer[4].reuse_a = 1;
          tc_out(ch.layer[4], p->P.p + He, 2 * He, He, sl(p, SL_P));
          ch.n_layers = 5;
          p_ready = true;
        }
        GW_TRY(run_chain(p, ch, st));
      }
      x_cur = x_next;
      e_cur = e_next;
      continue;
    }
    // P = x [W1s ; W1d]^T   (two column slices of the edge MLP's first Linear)
    p->cur_tag = TAG_PROC_P;
    for (int h = 0; h < 2; ++h) {
      GemmOp t;
      t.rows_per_sample = H, t.batch = nb;
      t.a[0] = src_stream(x_cur, Dn, Dn, H);
      t.W = me.W[0] + h * Dn, t.K = Dn, t.ldw = me.in[0], t.N = He;
      t.out = p->P.p + h * He, t.ldo = 2 * He;
      GW_TRY(run_op(p, t, st));
    }
    float* e_next = eb[k & 1];
    p->cur_tag = TAG_PROC_EDGE;
    {
      RowSrc e_src = e_cur ? src_stream(e_cur, De, De, El)
                           : (g.e0_broadcast ? src_bcast(g.e0, De, De) : src_stream(g.e0, De, De, El));
      GemmOp fo = first_op(El, nb, e_src, RowSrc(), me.W[0] + 2 * Dn, De, me.in[0], me.b[0]);
      fo.add[0] = src_gather(p->P.p, 2 * He, He, g.src, H, 0);
      fo.add[1] = src_gather(p->P.p, 2 * He, He, g.dst, H, He);
      GW_TRY(run_mlp(p, me, fo, false, true, e_src, e_next, De, st));
    }
    float* x_next = (k == d.num_blocks - 1) ? x_out : xb[k & 1];
    if (x_next == x_cur) x_next = xb[(k & 1) ^ 1];  // never update in place: node and edge passes both read old x
    p->cur_tag = TAG_PROC_NODE;
    {
      GemmOp fo = first_op(H, nb, src_stream(x_cur, Dn, Dn, H), src_segsum(e_next, De, De, g.ptr, nullptr, El),
                           mn.W[0], mn.in[0], mn.in[0], mn.b[0]);
      GW_TRY(run_mlp(p, mn, fo, false, true, src_stream(x_cur, Dn, Dn, H), x_next, Dn, st));
    }
    x_cur = x_next;
    e_cur = e_next;
  }
  if (x_cur != x_out) GW_CUDA(cudaMemcpyAsync(x_out, x_cur, (size_t)nb * H * Dn * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}
static ProcGraph latent_graph_of(gw_plan* p) {
  return ProcGraph{p->d.n_mesh, p->d.n_lat_edges, p->lat_src.p, p->lat_dst.p, p->lat_ptr.p, p->e_lat.p, true,
                   p->lat_maxdeg, p->lat_mindeg, sl(p, SL_ELAT)};
}

// AssimilatorDecoder.forward (assimilator_decoder.py:173-200) + Decoder residual (decoder.py:92-94).
// multi-GPU loss boundary: the chain that stores the forecast also stores it into every GPU's gather buffer (gw_tc3.cu out_mode)
static void apply_out_peers(gw_plan* p, TcChain& ch) {
  if (p->out_mode == 0) return;
  char* o = reinterpret_cast<char*>(ch.layer[ch.n_layers - 1].out);
  ch.out_mode = p->out_mode, ch.n_out_peers = p->n_out_peers;
  if (p->out_mode == 1) ch.out_mc = reinterpret_cast<float*>(o + p->out_delta[0]);
  for (int j = 0; j < p->n_out_peers && j < 8; ++j) ch.out_peer[j] = reinterpret_cast<float*>(o + p->out_delta[j]);
}

// e' rows of the decoder block are only materialised by the CUDA-core path and by the unfused fallback: allocated on demand
static int ensure_rows_e(gw_plan* p, size_t floats) {
  if (p->rows_e.n >= floats) return 0;
  GW_CUDA(cudaDeviceSynchronize());
  return p->rows_e.alloc(floats);
}

static int stage_decoder(gw_plan* p, const float* x_in, int x_in_slot, const float* start, int start_ld, float* out, int out_ld, int nb,
                         cudaStream_t st) {
  const gw_dims& d = p->d;
  const int Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, H = d.n_mesh, Ed = d.n_dec_edges, No = d.n_out;
  RowSrc none;
  const bool fuse = is_tc(p) && p->fuse_seg && p->dec_maxdeg >= 1 && p->dec_maxdeg <= 8;
  GW_CHECK(p->out_mode == 0 || (is_tc(p) && p->tc_dec_out_ok), "the fused loss-boundary gather needs the tensor-core output chain");
  if (!fuse) GW_TRY(ensure_rows_e(p, (size_t)p->chunk * std::max((size_t)p->d.n_in, (size_t)Ed) * De));
  for (int s0 = 0; s0 < nb; s0 += p->chunk) {
    const int cb = std::min(p->chunk, nb - s0);
    const float* x = x_in + (size_t)s0 * H * Dn;
    float* Pd = p->P.p;  // [cb*H, He]
    float* eprime = p->rows_e.p;
    float* xg = p->rows_n.p;
    const Mlp& me = p->dec_blk_edge;
    if (is_tc(p)) {
      const Mlp& mn = p->dec_blk_node;
      p->cur_tag = TAG_DEC_P;
      {
        TcChain ch;
        ch.rows_per_sample = H, ch.batch = cb;
        ch.a0[0] = bounded(src_stream(x, Dn, Dn, H), sl(p, x_in_slot));
        ch.K0 = Dn;
        ch.layer[0] = tc_layer(p->tc_dec_edge.w0, nullptr, -1, false, false);
        tc_out(ch.layer[0], Pd, He, He, sl(p, SL_P));
        ch.n_layers = 1;
        GW_TRY(run_chain(p, ch, st));
      }
      p->cur_tag = TAG_DEC_EDGE;
      {  // layer 1 = relu(Pd[src] + E1) is the operand assembly; layers 2, 3 + LN + e_dec residual on the tensor cores; the rows
         // are summed per lat/lon point in the epilogue (fused): e' is never written (the reference discards it too: `out, _ =`)
        TcChain ch;
        ch.rows_per_sample = Ed, ch.batch = cb;
        ch.a0[0] = bounded(src_gather_bcast_relu(Pd, He, He, p->dec_src.p, H, p->E1_dec.p, He), sl(p, SL_P));
        ch.a0[0].bound2 = sl(p, SL_E1DEC);
        ch.K0 = He;
        ch.layer[0] = tc_layer(p->tc_dec_edge.w1, &me, 1, true, true);
        ch.layer[1] = tc_layer(p->tc_dec_edge.w2, &me, 2, false, false);
        // (fused sums: the constant residual e_dec is not read per edge -- its per-point sum S_dec joins each finished sum)
        tc_ln(ch.layer[1], me, fuse && p->S_dec.p ? none : bounded(src_bcast(p->e_dec.p, De, De), sl(p, SL_EDEC)));
        if (fuse) {
          TcLayer& L = ch.layer[1];
          if (p->S_dec.p) L.seg_add = p->S_dec.p, L.seg_add_bound = sl(p, SL_SDEC);
          L.seg_dst = p->dec_dst.p, L.seg_out = p->agg_grid.p, L.seg_ld = De, L.seg_rows = No, L.seg_carry = p->seg_carry.p;
          L.seg_maxdeg = (float)p->dec_maxdeg, L.seg_bound = sl(p, SL_AGG_GRID);
          if (p->dec_mindeg == 0) GW_CUDA(cudaMemsetAsync(p->agg_grid.p, 0, (size_t)cb * No * De * sizeof(float), st));
        } else {
          tc_out(ch.layer[1], eprime, De, De, sl(p, SL_ROWS_E));
        }
        ch.n_layers = 2;
        GW_TRY(run_chain(p, ch, st));
      }
      p->cur_tag = TAG_DEC_NODE;
      if (fuse) {
        TimedLaunch t(p, st);
        GW_CUDA(launch_seg_carry(p->seg_carry.p, p->dec_dst.p, Ed, No, cb, p->agg_grid.p, De, st));
      }
      {  // lat/lon node update (x == 0, so only the aggregate half of W1 and no residual)
        TcChain ch;
        ch.rows_per_sample = No, ch.batch = cb;
        if (!fuse) {
          TimedLaunch t(p, st);
          GW_CUDA(launch_segsum(eprime, De, De, p->dec_ptr.p, nullptr, Ed, No, cb, p->agg_grid.p, De, st));
        }
        ch.a0[0] = fuse ? bounded(src_stream(p->agg_grid.p, De, De, No), sl(p, SL_AGG_GRID))
                        : bounded(src_stream(p->agg_grid.p, De, De, No), sl(p, SL_ROWS_E), (float)std::max(p->dec_maxdeg, 1));
        ch.K0 = De;
        ch.layer[0] = tc_layer(p->tc_dec_node.w0, &mn, 0, true, true);
        ch.layer[1] = tc_layer(p->tc_dec_node.w1, &mn, 1, true, true);
        ch.layer[2] = tc_layer(p->tc_dec_node.w2, &mn, 2, false, false);
        tc_ln(ch.layer[2], mn, none);
        if (p->tc_dec_out_ok) {  // node_decoder (256->128->128->out, no norm) + start-feature residual in the same chain
          const Mlp& m = p->dec_node_dec;
          ch.layer[2].feeds_next = 1;
          ch.layer[3] = tc_layer(p->tc_dec_out.w0, &m, 0, true, true);
          ch.layer[4] = tc_layer(p->tc_dec_out.w1, &m, 1, true, true);
          {  // the whole decoder tail as ONE lean chain when the output layer qualifies for the lean path's narrow epilogue (even
             // out_dim, 8-byte aligned rows, no fused multi-GPU boundary): no hidden-row round trip, no general-path chain
            TcChain c6 = ch;
            c6.layer[5] = tc_layer(p->tc_dec_out.w2, &m, 2, false, false);
            if (start && d.residual_dim > 0)
              c6.layer[5].residual = src_stream(start + (size_t)s0 * No * start_ld, start_ld, d.out_dim, No);
            tc_out(c6.layer[5], out + (size_t)s0 * No * out_ld, out_ld, d.out_dim);
            c6.n_layers = 6;
            apply_out_peers(p, c6);
            if (tc3_chain_is_lean(c6)) {
              GW_TRY(run_chain(p, c6, st));
              continue;
            }
          }
          if (p->tc_dec_out.w1.N <= Dn && !(p->tc_dec_out.w1.N & 63)) {
            // the narrow output layer (78 of 80 columns, 8-byte aligned rows) would take the whole chain off the lean
            // path: run it as a chain of its own on the hidden rows h
            ch.layer[4].feeds_next = 0;
            const int Hd = p->tc_dec_out.w1.N;
            tc_out(ch.layer[4], xg, Hd, Hd, sl(p, SL_ROWS_N));
            ch.n_layers = 5;
            GW_TRY(run_chain(p, ch, st));
            TcChain c2;
            c2.rows_per_sample = No, c2.batch = cb;
            c2.a0[0] = bounded(src_stream(xg, Hd, Hd, No), sl(p, SL_ROWS_N));
            c2.K0 = Hd;
            c2.layer[0] = tc_layer(p->tc_dec_out.w2, &m, 2, false, false);
            if (start && d.residual_dim > 0)
              c2.layer[0].residual = src_stream(start + (size_t)s0 * No * start_ld, start_ld, d.out_dim, No);
            tc_out(c2.layer[0], out + (size_t)s0 * No * out_ld, out_ld, d.out_dim);
            c2.n_layers = 1;
            apply_out_peers(p, c2);
            GW_TRY(run_chain(p, c2, st));
            continue;
          }
          ch.layer[5] = tc_layer(p->tc_dec_out.w2, &m, 2, false, false);
          if (start && d.residual_dim > 0)
            ch.layer[5].residual = src_stream(start + (size_t)s0 * No * start_ld, start_ld, d.out_dim, No);
          tc_out(ch.layer[5], out + (size_t)s0 * No * out_ld, out_ld, d.out_dim);
          ch.n_layers = 6;
          apply_out_peers(p, ch);
          GW_TRY(run_chain(p, ch, st));
          continue;
        }
        tc_out(ch.layer[2], xg, Dn, Dn, sl(p, SL_ROWS_N));
        ch.n_layers = 3;
        GW_TRY(run_chain(p, ch, st));
      }
      for (int b = 0; b < cb; ++b) {  // node_decoder on the CUDA cores when its shape does not fit the chain kernel (sample by
                                      // sample: the tensor-core plan's ping-pong scratch holds one sample)
        const Mlp& m = p->dec_node_dec;
        GemmOp fo = first_op(No, 1, src_stream(xg + (size_t)b * No * Dn, Dn, Dn, No), none, m.W[0], m.in[0], m.in[0], m.b[0]);
        RowSrc res;
        if (start && d.residual_dim > 0) res = src_stream(start + (size_t)(s0 + b) * No * start_ld, start_ld, d.out_dim, No);
        GW_TRY(run_mlp(p, m, fo, false, m.ln_g != nullptr, res, out + (size_t)(s0 + b) * No * out_ld, out_ld, st));
      }
      continue;
    }
    p->cur_tag = TAG_DEC_P;
    {  // Pd = x W1s^T ; the dst operand (lat/lon nodes) is identically zero, assimilator_decoder.py:84,189-193
      GemmOp t;
      t.rows_per_sample = H, t.batch = cb;
      t.a[0] = src_stream(x, Dn, Dn, H);
      t.W = me.W[0], t.K = Dn, t.ldw = me.in[0], t.N = He;
      t.out = Pd, t.ldo = He;
      GW_TRY(run_op(p, t, st));
    }
    p->cur_tag = TAG_DEC_EDGE;
    {  // edge MLP: layer 1 output = relu(Pd[src] + E1_dec) is assembled on the fly as the A operand of layer 2
      GemmOp fo;
      fo.rows_per_sample = Ed, fo.batch = cb;
      fo.a[0] = src_gather_bcast_relu(Pd, He, He, p->dec_src.p, H, p->E1_dec.p, He);
      fo.W = me.W[1], fo.K = me.in[1], fo.ldw = me.in[1], fo.bias = me.b[1];
      GW_TRY(run_mlp(p, me, fo, true, true, src_bcast(p->e_dec.p, De, De), eprime, De, st));
    }
    p->cur_tag = TAG_DEC_NODE;
    {  // lat/lon node update: cat([0 ; agg]) -> only the agg half of W1 contributes; residual x == 0
      const Mlp& mn = p->dec_blk_node;
      GemmOp fo = first_op(No, cb, src_segsum(eprime, De, De, p->dec_ptr.p, nullptr, Ed), none, mn.W[0] + Dn, De, mn.in[0], mn.b[0]);
      GW_TRY(run_mlp(p, mn, fo, false, true, none, xg, Dn, st));
    }
    {  // node_decoder (no norm) + start-feature residual (decoder.py:93)
      const Mlp& m = p->dec_node_dec;
      GemmOp fo = first_op(No, cb, src_stream(xg, Dn, Dn, No), none, m.W[0], m.in[0], m.in[0], m.b[0]);
      RowSrc res;
      if (start && d.residual_dim > 0) res = src_stream(start + (size_t)s0 * No * start_ld, start_ld, d.out_dim, No);
      GW_TRY(run_mlp(p, m, fo, false, m.ln_g != nullptr, res, out + (size_t)s0 * No * out_ld, out_ld, st));
    }
  }
  return 0;
}

// longest / shortest segment of a CSR (and, optionally, the target of every entry); synchronises `st` (graph upload time)
static int csr_stats(gw_plan* p, const int32_t* ptr, int n, int32_t* dst, int* maxdeg, int* mindeg, cudaStream_t st) {
  const int init[2] = {0, 0x7fffffff};
  int got[2] = {0, 0};
  GW_CUDA(cudaMemcpyAsync(p->deg_stats.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
  GW_CUDA(launch_csr_expand(ptr, n, dst, p->deg_stats.p, st));
  GW_CUDA(cudaMemcpyAsync(got, p->deg_stats.p, sizeof(got), cudaMemcpyDeviceToHost, st));
  GW_CUDA(cudaStreamSynchronize(st));
  *maxdeg = got[0], *mindeg = n > 0 ? got[1] : 0;
  return 0;
}

// longest lat/lon -> mesh segment of the current encoder graph, left on the device (it scales a magnitude bound): no sync
static int encoder_degree(gw_plan* p, cudaStream_t st) {
  static const int init[2] = {0, 0x7fffffff};
  GW_CUDA(cudaMemcpyAsync(p->enc_deg.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
  GW_CUDA(launch_csr_expand(p->enc_ptr.p, p->d.n_mesh, nullptr, p->enc_deg.p, st));
  if (p->enc_chunk_seg.p)  // chunk table of the two-level segment sum follows the graph
    GW_CUDA(launch_seg_chunks(p->enc_ptr.p, p->d.n_mesh, p->enc_chunk_seg.p, p->enc_chunk_j0.p, p->enc_seg_chunk0.p, st));
  return 0;
}

}  // namespace gw
#include "gw_train.inl"
namespace gw {

enum { NEED_ENC = 1, NEED_PROC = 2, NEED_DEC = 4, NEED_INFER = 8 };
static int check_ready(gw_plan* p, int batch, int need) {
  GW_CHECK(p != nullptr, "null plan");
  if (need & NEED_INFER)
    GW_CHECK(!p->train_only, "this plan was made by gw_plan_create_train: it holds no inference scratch (use a gw_plan_create plan to run forwards)");
  if (need & NEED_ENC) GW_CHECK(p->have_enc && p->have_lat && p->w_enc, "encoder stage needs the encoder + latent graphs and encoder.* weights");
  if (need & NEED_PROC) GW_CHECK(p->w_proc, "processor stage needs processor.* weights");
  if (need & NEED_DEC) GW_CHECK(p->have_dec && p->w_dec, "decoder stage needs the decoder graph and decoder.* weights");
  GW_CHECK(batch >= 1 && batch <= p->d.max_batch, "batch out of range [1, max_batch]");
  GW_CUDA(cudaSetDevice(p->device));
  return 0;
}

}  // namespace gw

// ===================================================================================================================
// C ABI
// ===================================================================================================================
extern "C" {

int gw_abi_version(void) { return GW_ABI_VERSION; }
const char* gw_last_error(void) { return gw::g_err.c_str(); }
int64_t gw_launch_count(void) { return gw::g_launches; }
void gw_launch_count_reset(void) { gw::g_launches = 0; }

// inference scratch and weight constants of a plan (gw_plan_create; a training-only plan holds none of it)
static int alloc_inference_scratch(gw_plan* p, size_t chunk) {
  const gw_dims& d = p->d;
  const bool tc = d.precision != GW_PREC_FP32_SIMT;
  const size_t Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, Hn = d.hidden_node;
  const size_t max_hid = std::max({Dn, De, He, Hn, (size_t)d.hidden_dec, (size_t)d.out_dim});
  const size_t max_rows = std::max({(size_t)d.n_in, (size_t)d.n_out, (size_t)d.n_mesh, (size_t)d.n_lat_edges, (size_t)d.n_dec_edges});
  const size_t n_io = std::max((size_t)d.n_in, (size_t)d.n_out);
  const size_t dec_tiles = ((size_t)d.n_dec_edges + 127) / 128, lat_tiles = ((size_t)d.n_lat_edges + 127) / 128;
  const size_t B = d.max_batch;
  int rc = 0;
  rc |= p->e_enc.alloc((size_t)d.n_in * De) | p->xm0.alloc((size_t)d.n_mesh * Dn) | p->C1_enc.alloc((size_t)d.n_in * He);
  rc |= p->e_lat.alloc((size_t)d.n_lat_edges * De) | p->e_dec.alloc((size_t)d.n_dec_edges * De);
  rc |= p->E1_dec.alloc((size_t)d.n_dec_edges * He) | p->tmpP.alloc((size_t)d.n_mesh * He);
  if (tc && d.n_out > 0 && d.n_dec_edges > 0) rc |= p->S_dec.alloc((size_t)d.n_out * De);
  {  // hidden-activation ping-pong of run_mlp: every stage on the CUDA-core path, the one-off constant precompute
     // (one sample's worth of rows) on the tensor-core path
    size_t pp = (tc ? 1 : chunk) * max_rows * max_hid;
    if (!tc && B * std::max((size_t)d.n_lat_edges, (size_t)d.n_mesh) > chunk * max_rows) pp = B * max_rows * max_hid;
    rc |= p->bufA.alloc(pp) | p->bufB.alloc(pp);
  }
  rc |= p->rows_n.alloc(chunk * n_io * Dn);
  rc |= p->rows_e.alloc(chunk * (tc ? (size_t)d.n_in : std::max((size_t)d.n_in, (size_t)d.n_dec_edges)) * De);
  rc |= p->xbuf0.alloc(B * d.n_mesh * Dn) | p->xbuf1.alloc(B * d.n_mesh * Dn);
  rc |= p->ebuf0.alloc(B * d.n_lat_edges * De) | p->ebuf1.alloc(B * d.n_lat_edges * De);
  rc |= p->P.alloc(B * d.n_mesh * 2 * He);
  rc |= p->agg_mesh.alloc(B * d.n_mesh * De);
  if (tc && d.n_in > 0) {
    p->enc_max_chunks = gw::seg_chunk_bound(d.n_mesh, d.n_in);
    rc |= p->enc_chunk_seg.alloc(p->enc_max_chunks) | p->enc_chunk_j0.alloc(p->enc_max_chunks) | p->enc_seg_chunk0.alloc(d.n_mesh + 1);
    rc |= p->enc_partial.alloc(chunk * (size_t)p->enc_max_chunks * 256);
  }
  if (tc) {
    rc |= p->agg_grid.alloc(chunk * d.n_out * De);
    rc |= p->seg_carry.alloc(std::max(chunk * dec_tiles, B * (lat_tiles + 1)) * 2048);  // [samples][tiles][8 row groups][256]
  }
  return rc;
}

static int plan_create(const gw_dims* dims, gw_plan** out_plan, bool train_only) {
  GW_CHECK(dims && out_plan, "null argument");
  const gw_dims& d = *dims;
  GW_CHECK(d.n_in >= 0 && d.n_out >= 0 && d.n_mesh > 0 && d.n_lat_edges >= 0 && d.n_dec_edges >= 0,
           "graph sizes must be non-negative (n_mesh positive); a standalone sub-module leaves the parts it lacks at 0");
  GW_CHECK(d.in_dim > 0 && d.out_dim > 0 && d.node_dim > 0 && d.edge_dim > 0, "feature sizes must be positive");
  GW_CHECK(d.hidden_layers_node >= 1 && d.hidden_layers_edge >= 1 && d.hidden_layers_dec >= 1, "hidden_layers must be >= 1");
  GW_CHECK(d.residual_dim == 0 || d.residual_dim == d.out_dim,
           "residual_dim must equal out_dim (the reference adds start features of the same width, decoder.py:93)");
  GW_CHECK(d.max_batch >= 1, "max_batch must be >= 1");
  GW_CHECK(d.precision == GW_PREC_FP32_SIMT || d.precision == GW_PREC_FP32_TC || d.precision == GW_PREC_BF16_TC, "unknown precision");
  if (d.precision != GW_PREC_FP32_SIMT) {
    GW_CHECK(d.node_dim == 256 && d.edge_dim == 256 && d.hidden_node == 256 && d.hidden_edge == 256,
             "the tensor-core chains are built for 256-wide node/edge/hidden dims (the reference default); use fp32_simt otherwise");
    GW_CHECK(d.hidden_layers_node == 2 && d.hidden_layers_edge == 2, "the tensor-core chains are built for hidden_layers = 2");
    int cc_major = 0, cc_minor = 0, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
    GW_CHECK(cc_major == 9 && cc_minor == 0, "the tensor-core chains need an sm_90a device (wgmma)");
  }
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) {
    gw::set_error("no CUDA device available (libgwb200 has no CPU fallback)");
    return 1;
  }
  gw_plan* p = new gw_plan();
  p->d = d;
  p->train_only = train_only;
  // every failure after this point releases the plan and whatever it already holds
#define GW_CUDA_P(expr)                                                          \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) {                                                     \
      std::string _m = std::string(#expr) + ": " + cudaGetErrorString(_e);       \
      gw_plan_destroy(p);                                                        \
      gw::set_error(_m);                                                         \
      return 1;                                                                  \
    }                                                                            \
  } while (0)
  GW_CUDA_P(cudaGetDevice(&p->device));
  const size_t Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, Hn = d.hidden_node;
  const size_t max_hid = std::max({Dn, De, He, Hn, (size_t)d.hidden_dec, (size_t)d.out_dim});
  const size_t max_rows = std::max({(size_t)d.n_in, (size_t)d.n_out, (size_t)d.n_mesh, (size_t)d.n_lat_edges, (size_t)d.n_dec_edges});
  // chunking: keep the per-pass scratch of the lat/lon-sized stages under ~24 GB (an 80 GB H100 also holds the caller's tensors).  The tensor-core path never writes the
  // decoder's e' rows (their per-point sums are formed in the edge chain's epilogue), and its hidden activations stay on
  // the SM, so its per-sample scratch is three lat/lon-sized row buffers; the CUDA-core path also needs e' and the ping-pong.
  const bool tc = d.precision != GW_PREC_FP32_SIMT;
  const size_t n_io = std::max((size_t)d.n_in, (size_t)d.n_out);
  const size_t dec_tiles = ((size_t)d.n_dec_edges + 127) / 128;
  const size_t per_sample = tc ? (n_io * Dn + (size_t)d.n_in * De + (size_t)d.n_out * De + dec_tiles * 2048) * sizeof(float)
                               : (2 * max_rows * max_hid + std::max((size_t)d.n_in, (size_t)d.n_dec_edges) * De + n_io * Dn) * sizeof(float);
  size_t chunk = std::max<size_t>(1, std::min<size_t>(d.max_batch, (24ull << 30) / std::max<size_t>(per_sample, 1)));
  if (const char* force = getenv("GW_B200_CHUNK")) {  // test knob: exercise the chunked stage loops on small grids
    const long v = atol(force);
    if (v >= 1) chunk = std::min<size_t>((size_t)v, (size_t)d.max_batch);
  }
  p->chunk = (int)chunk;
  p->fuse_seg = tc && !getenv("GW_TC3_NOSEG");  // diagnostics: GW_TC3_NOSEG=1 keeps the separate segment-sum kernels
  if (const char* pts = getenv("GW_B200_TRAIN_CHUNK")) {  // test knob: many chunks of the bounded-memory training step on small grids
    const long v = atol(pts);
    if (v >= 1) p->train_chunk_pts = (int)std::min<long>(v, 1l << 30);
  }
  int rc = 0;
  rc |= p->enc_mesh.alloc(d.n_in) | p->enc_perm.alloc(d.n_in) | p->enc_ptr.alloc(d.n_mesh + 1);
  rc |= p->enc_attr.alloc((size_t)d.n_in * d.enc_edge_attr_dim);
  rc |= p->lat_src.alloc(d.n_lat_edges) | p->lat_dst.alloc(d.n_lat_edges) | p->lat_ptr.alloc(d.n_mesh + 1);
  rc |= p->lat_attr.alloc((size_t)d.n_lat_edges * 2);
  rc |= p->dec_src.alloc(d.n_dec_edges) | p->dec_ptr.alloc(d.n_out + 1) | p->dec_attr.alloc((size_t)d.n_dec_edges * 2);
  rc |= p->dec_dst.alloc(d.n_dec_edges) | p->deg_stats.alloc(2) | p->enc_deg.alloc(2) | p->bounds.alloc(gw::SL_COUNT);
  rc |= p->zeros_h3.alloc((size_t)d.n_mesh * d.in_dim);
  if (!train_only) rc |= alloc_inference_scratch(p, chunk);
  if (rc) {
    std::string keep = gw::g_err;
    gw_plan_destroy(p);
    gw::set_error(keep);
    return 1;
  }
  GW_CUDA_P(cudaMemset(p->zeros_h3.p, 0, p->zeros_h3.bytes()));
  GW_CUDA_P(cudaMemset(p->bounds.p, 0, p->bounds.bytes()));
  GW_CUDA_P(cudaHostAlloc((void**)&p->tc_status_host, 64 * sizeof(int32_t), cudaHostAllocMapped));
  std::memset(p->tc_status_host, 0, 64 * sizeof(int32_t));
  GW_CUDA_P(cudaHostGetDevicePointer((void**)&p->tc_status_dev, p->tc_status_host, 0));
#undef GW_CUDA_P
  p->n_in_cur = d.n_in;
  *out_plan = p;
  return 0;
}

int gw_plan_create(const gw_dims* dims, gw_plan** out_plan) { return plan_create(dims, out_plan, false); }
int gw_plan_create_train(const gw_dims* dims, gw_plan** out_plan) { return plan_create(dims, out_plan, true); }

int gw_plan_destroy(gw_plan* p) {
  if (!p) return 0;
  for (DevBuf<int32_t>* b : {&p->enc_mesh, &p->enc_perm, &p->enc_ptr, &p->lat_src, &p->lat_dst, &p->lat_ptr, &p->dec_src, &p->dec_ptr})
    b->release();
  for (DevBuf<float>* b : {&p->enc_attr, &p->lat_attr, &p->dec_attr, &p->wbuf, &p->zeros_h3, &p->e_enc, &p->xm0, &p->C1_enc,
                           &p->e_lat, &p->e_dec, &p->E1_dec, &p->S_dec, &p->tmpP, &p->bufA, &p->bufB, &p->rows_n, &p->rows_e, &p->xbuf0,
                           &p->xbuf1, &p->ebuf0, &p->ebuf1, &p->P})
    b->release();
  p->tc_packed.release(), p->tc_absmax.release(), p->agg_mesh.release(), p->agg_grid.release();
  p->bounds.release(), p->dec_dst.release(), p->seg_carry.release(), p->deg_stats.release(), p->enc_deg.release();
  p->h3_frames.release(), p->h3_lat.release(), p->h3_lng.release(), p->h3_cell_of.release(), p->h3_slot.release(), p->obs_ws.release();
  p->enc_chunk_seg.release(), p->enc_chunk_j0.release(), p->enc_seg_chunk0.release(), p->enc_partial.release();
  if (p->train) {
    for (gw_tape* k : p->train->tapes) {  // every live tape's memory goes with the plan; the tapes stay as dead handles
      gw::tape_release(p->train, k, p->train->st);
      k->plan = nullptr;
    }
    p->train->tapes.clear();
    p->train->wT.release(), p->train->gbuf.release(), p->train->lat_perm_src.release(), p->train->lat_ptr_src.release();
    p->train->dec_perm_src.release(), p->train->dec_ptr_src.release(), p->train->iota.release(), p->train->sort_ws.release();
    p->train->enc_slot_sorted.release(), p->train->dec_cperm.release(), p->train->dec_cptr.release();
    p->train->bslots.release(), p->train->wg_ws.release();
    for (auto& kv : p->train->images) kv.second.img.release(), kv.second.amax.release();
    delete p->train;
    p->train = nullptr;
  }
  if (p->tc_status_host) cudaFreeHost(p->tc_status_host);
  for (cudaEvent_t e : p->ev_pool) cudaEventDestroy(e);
  delete p;
  return 0;
}

int64_t gw_plan_device_bytes(const gw_plan* p) {
  if (!p) return 0;
  size_t t = 0;
  for (const DevBuf<int32_t>* b : {&p->enc_mesh, &p->enc_perm, &p->enc_ptr, &p->lat_src, &p->lat_dst, &p->lat_ptr, &p->dec_src, &p->dec_ptr})
    t += b->bytes();
  for (const DevBuf<float>* b : {&p->enc_attr, &p->lat_attr, &p->dec_attr, &p->wbuf, &p->zeros_h3, &p->e_enc, &p->xm0, &p->C1_enc,
                                 &p->e_lat, &p->e_dec, &p->E1_dec, &p->S_dec, &p->tmpP, &p->bufA, &p->bufB, &p->rows_n, &p->rows_e,
                                 &p->xbuf0, &p->xbuf1, &p->ebuf0, &p->ebuf1, &p->P})
    t += b->bytes();
  t += p->tc_packed.bytes() + p->agg_mesh.bytes() + p->agg_grid.bytes() + p->seg_carry.bytes() + p->dec_dst.bytes();
  return (int64_t)t;
}

int gw_plan_set_encoder_graph(gw_plan* p, int32_t n_in, const int32_t* enc_mesh, const int32_t* perm, const int32_t* ptr,
                              const float* attr, void* stream) {
  GW_CHECK(p && enc_mesh && perm && ptr && attr, "null argument");
  GW_CHECK(n_in >= 1 && n_in <= p->d.n_in, "n_in exceeds the plan's capacity (gw_dims.n_in)");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  GW_CUDA(cudaMemcpyAsync(p->enc_mesh.p, enc_mesh, (size_t)n_in * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->enc_perm.p, perm, (size_t)n_in * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->enc_ptr.p, ptr, (size_t)(p->d.n_mesh + 1) * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->enc_attr.p, attr, (size_t)n_in * p->d.enc_edge_attr_dim * 4, cudaMemcpyDeviceToDevice, st));
  p->n_in_cur = n_in;
  p->have_enc = true;
  ++p->enc_graph_gen;
  GW_TRY(gw::encoder_degree(p, st));
  if (p->w_enc && !p->train_only) GW_TRY(gw::precompute_encoder_constants(p, st));  // per-call graphs (assimilator_encoder.py:118)
  return 0;
}

int gw_plan_set_h3_tables(gw_plan* p, int32_t res, int32_t n_cells, int32_t lattice_n, const double* face_frames, const int32_t* cell_of,
                          const int32_t* cell_slot, const double* cell_lat, const double* cell_lng, double scale, double rot_cos,
                          double rot_sin, void* stream) {
  GW_CHECK(p && face_frames && cell_of && cell_slot && cell_lat && cell_lng, "null argument");
  GW_CHECK(n_cells == p->d.n_mesh, "the H3 tables must describe the plan's mesh (n_cells == n_mesh)");
  GW_CHECK(lattice_n > 0 && res >= 0, "bad table sizes");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  const size_t w = 2 * (size_t)lattice_n + 1;
  GW_TRY(p->h3_frames.alloc(180));
  GW_TRY(p->h3_cell_of.alloc(20 * w * w));
  GW_TRY(p->h3_slot.alloc(n_cells));
  GW_TRY(p->h3_lat.alloc(n_cells));
  GW_TRY(p->h3_lng.alloc(n_cells));
  GW_CUDA(cudaMemcpyAsync(p->h3_frames.p, face_frames, 180 * sizeof(double), cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->h3_cell_of.p, cell_of, 20 * w * w * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->h3_slot.p, cell_slot, (size_t)n_cells * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->h3_lat.p, cell_lat, (size_t)n_cells * sizeof(double), cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->h3_lng.p, cell_lng, (size_t)n_cells * sizeof(double), cudaMemcpyDeviceToDevice, st));
  gw::H3Tables& t = p->h3;
  t.res = res, t.n_cells = n_cells, t.lat_n = lattice_n;
  t.frames = p->h3_frames.p, t.cell_of = p->h3_cell_of.p, t.cell_slot = p->h3_slot.p, t.cell_lat = p->h3_lat.p, t.cell_lng = p->h3_lng.p;
  t.scale = scale, t.cr = rot_cos, t.sr = rot_sin;
  return 0;
}

int gw_plan_build_obs_graph(gw_plan* p, const float* lat_lon_heights, int32_t n_obs, void* stream) {
  GW_CHECK(p && lat_lon_heights, "null argument");
  GW_CHECK(p->h3.res >= 0, "gw_plan_set_h3_tables must be called first");
  GW_CHECK(p->d.enc_edge_attr_dim == 3, "the observation graph carries 3 edge attributes (sin d, cos d, height)");
  GW_CHECK(n_obs >= 1 && n_obs <= p->d.n_in, "n_obs exceeds the plan's capacity (gw_dims.n_in)");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  const size_t need = gw::obs_graph_workspace_bytes(p->d.n_in);
  if (p->obs_ws.n < need) GW_TRY(p->obs_ws.alloc(need));
  GW_CUDA(gw::launch_obs_graph(p->h3, lat_lon_heights, n_obs, p->d.n_mesh, p->enc_mesh.p, p->enc_perm.p, p->enc_ptr.p, p->enc_attr.p,
                               p->obs_ws.p, p->obs_ws.n, p->tc_status_dev, st));
  p->n_in_cur = n_obs;
  p->have_enc = true;
  ++p->enc_graph_gen;
  GW_TRY(gw::encoder_degree(p, st));
  if (p->w_enc && !p->train_only) GW_TRY(gw::precompute_encoder_constants(p, st));  // per-call graphs (assimilator_encoder.py:118)
  return 0;
}

int gw_plan_set_latent_graph(gw_plan* p, const int32_t* src, const int32_t* dst, const int32_t* ptr, const float* attr, void* stream) {
  GW_CHECK(p && src && dst && ptr && attr, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  const size_t El = p->d.n_lat_edges;
  GW_CUDA(cudaMemcpyAsync(p->lat_src.p, src, El * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->lat_dst.p, dst, El * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->lat_ptr.p, ptr, (size_t)(p->d.n_mesh + 1) * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->lat_attr.p, attr, El * 2 * 4, cudaMemcpyDeviceToDevice, st));
  GW_TRY(gw::csr_stats(p, p->lat_ptr.p, p->d.n_mesh, nullptr, &p->lat_maxdeg, &p->lat_mindeg, st));
  p->have_lat = true;
  p->w_enc = p->w_proc = p->w_dec = false;  // constants depend on the graphs: weights must be (re)uploaded after
  return 0;
}

int gw_plan_set_decoder_graph(gw_plan* p, const int32_t* src, const int32_t* ptr, const float* attr, void* stream) {
  GW_CHECK(p && src && ptr && attr, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  const size_t Ed = p->d.n_dec_edges;
  GW_CUDA(cudaMemcpyAsync(p->dec_src.p, src, Ed * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->dec_ptr.p, ptr, (size_t)(p->d.n_out + 1) * 4, cudaMemcpyDeviceToDevice, st));
  GW_CUDA(cudaMemcpyAsync(p->dec_attr.p, attr, Ed * 2 * 4, cudaMemcpyDeviceToDevice, st));
  GW_TRY(gw::csr_stats(p, p->dec_ptr.p, p->d.n_out, p->dec_dst.p, &p->dec_maxdeg, &p->dec_mindeg, st));
  p->have_dec = true;
  p->w_enc = p->w_proc = p->w_dec = false;
  return 0;
}

int gw_plan_set_weights(gw_plan* p, const gw_param* params, int32_t n, void* stream) {
  GW_CHECK(p && params && n > 0, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  size_t total = 0;
  for (int i = 0; i < n; ++i) {
    GW_CHECK(params[i].name && params[i].data && params[i].rows > 0 && params[i].cols > 0, "malformed gw_param entry");
    total += ((size_t)params[i].rows * params[i].cols + 63) / 64 * 64;  // 256-byte aligned slices
  }
  ++p->wgen;  // (even a failed upload has replaced what a tape's backward would differentiate)
  if (p->wbuf.n != total) GW_TRY(p->wbuf.alloc(total));
  p->params.clear();
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    size_t cnt = (size_t)params[i].rows * params[i].cols;
    GW_CUDA(cudaMemcpyAsync(p->wbuf.p + off, params[i].data, cnt * 4, cudaMemcpyDeviceToDevice, st));
    p->params[params[i].name] = {p->wbuf.p + off, {params[i].rows, params[i].cols}};
    off += (cnt + 63) / 64 * 64;
  }
  GW_TRY(gw::bind_all(p));
  if (p->train_only) return 0;  // (the training step packs its own weight images and computes the constants it needs)
  if (gw::is_tc(p)) GW_TRY(gw::pack_tc_weights(p, st));
  GW_TRY(gw::precompute_constants(p, st));
  return 0;
}

int gw_encoder_forward(gw_plan* p, const float* features, float* x_out, int32_t batch, void* stream) {
  GW_TRY(gw::check_ready(p, batch, gw::NEED_ENC | gw::NEED_INFER));
  GW_CHECK(features && x_out, "null argument");
  return gw::stage_encoder(p, features, x_out, gw::sl(p, gw::SL_XOUT), batch, (cudaStream_t)stream);
}

int gw_processor_forward(gw_plan* p, const float* x_in, float* x_out, int32_t batch, void* stream) {
  GW_TRY(gw::check_ready(p, batch, gw::NEED_PROC | gw::NEED_INFER));
  GW_CHECK(x_in && x_out, "null argument");
  GW_CHECK(p->have_lat && p->w_enc, "gw_processor_forward uses the plan's latent graph and encoded latent edges; "
                                    "use gw_processor_forward_graph for caller-supplied graphs");
  cudaStream_t st = (cudaStream_t)stream;
  if (gw::is_tc(p)) GW_TRY(gw::raw_bound(p, gw::SL_XIN, x_in, (long long)batch * p->d.n_mesh * p->d.node_dim, st));
  return gw::stage_processor(p, gw::latent_graph_of(p), x_in, x_out, gw::SL_XIN, gw::SL_XOUT, batch, st);
}

int gw_processor_forward_graph(gw_plan* p, const float* x_in, float* x_out, const float* edge_attr, int32_t n_nodes,
                               int32_t n_edges, const int32_t* src, const int32_t* dst, const int32_t* ptr, void* stream) {
  GW_TRY(gw::check_ready(p, 1, gw::NEED_PROC | gw::NEED_INFER));
  GW_CHECK(x_in && x_out && edge_attr && src && dst && ptr, "null argument");
  GW_CHECK(n_nodes >= 1 && (size_t)n_nodes <= (size_t)p->d.max_batch * p->d.n_mesh, "n_nodes exceeds max_batch*n_mesh");
  GW_CHECK(n_edges >= 1 && (size_t)n_edges <= (size_t)p->d.max_batch * p->d.n_lat_edges, "n_edges exceeds max_batch*n_lat_edges");
  cudaStream_t st = (cudaStream_t)stream;
  gw::ProcGraph g{n_nodes, n_edges, src, dst, ptr, edge_attr, false, 0, 0, gw::sl(p, gw::SL_EIN)};
  if (gw::is_tc(p)) {
    GW_TRY(gw::csr_stats(p, ptr, n_nodes, nullptr, &g.maxdeg, &g.mindeg, st));  // decides whether the per-node sums can be fused
    GW_TRY(gw::raw_bound(p, gw::SL_XIN, x_in, (long long)n_nodes * p->d.node_dim, st));
    GW_TRY(gw::raw_bound(p, gw::SL_EIN, edge_attr, (long long)n_edges * p->d.edge_dim, st));
  }
  return gw::stage_processor(p, g, x_in, x_out, gw::SL_XIN, gw::SL_XOUT, 1, st);
}

int gw_decoder_forward(gw_plan* p, const float* x_in, const float* start, int32_t start_ld, float* out, int32_t batch, void* stream) {
  GW_TRY(gw::check_ready(p, batch, gw::NEED_DEC | gw::NEED_INFER));
  GW_CHECK(x_in && out, "null argument");
  GW_CHECK(p->d.residual_dim == 0 || (start && start_ld >= p->d.residual_dim), "start features required (decoder.py:93)");
  cudaStream_t st = (cudaStream_t)stream;
  if (gw::is_tc(p)) GW_TRY(gw::raw_bound(p, gw::SL_XIN, x_in, (long long)batch * p->d.n_mesh * p->d.node_dim, st));
  return gw::stage_decoder(p, x_in, gw::SL_XIN, start, start_ld, out, p->d.out_dim, batch, st);
}

int gw_forward(gw_plan* p, const float* features, float* out, int32_t batch, void* stream) {
  return gw_forward_strided(p, features, out, p ? p->d.out_dim : 0, batch, stream);
}

int gw_forward_strided(gw_plan* p, const float* features, float* out, int32_t out_ld, int32_t batch, void* stream) {
  GW_TRY(gw::check_ready(p, batch, gw::NEED_ENC | gw::NEED_PROC | gw::NEED_DEC | gw::NEED_INFER));
  GW_CHECK(features && out, "null argument");
  GW_CHECK(out_ld >= p->d.out_dim, "out_ld must be at least out_dim");
  cudaStream_t st = (cudaStream_t)stream;
  // x lives in xbuf0 between stages
  GW_TRY(gw::stage_encoder(p, features, p->xbuf0.p, gw::sl(p, gw::SL_X0), batch, st));
  GW_TRY(gw::stage_processor(p, gw::latent_graph_of(p), p->xbuf0.p, p->xbuf0.p, gw::SL_X0, gw::SL_X0, batch, st));
  return gw::stage_decoder(p, p->xbuf0.p, gw::SL_X0, p->d.residual_dim > 0 ? features : nullptr, p->d.in_dim, out, out_ld, batch, st);
}

// the plan's training state, made on first use with its built-in tape registered
static gw::TrainState* train_state(gw_plan* p) {
  if (!p->train) {
    p->train = new gw::TrainState();
    p->train->own.plan = p;
    p->train->tapes.insert(&p->train->own);
  }
  return p->train;
}

int gw_tape_create(gw_plan* p, gw_tape** out) {
  GW_CHECK(p && out, "null argument");
  gw::TrainState* T = train_state(p);
  gw_tape* k = new gw_tape();
  k->plan = p;
  T->tapes.insert(k);
  *out = k;
  return 0;
}

int gw_tape_destroy(gw_tape* k, void* stream) {
  if (!k) return 0;
  if (gw_plan* p = k->plan) {
    GW_CHECK(k != &p->train->own, "gw_tape_destroy: the plan's built-in tape goes with the plan");
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

int gw_train_forward(gw_plan* p, const float* features, float* out, int32_t batch, void* stream) {
  GW_CHECK(p != nullptr, "null plan");
  return gw_train_forward_tape(p, &train_state(p)->own, features, out, batch, stream);
}

int gw_train_backward_tape(gw_plan* p, gw_tape* k, const float* grad_out, float* grad_features, const gw_param* grads, int32_t n, void* stream) {
  GW_TRY(check_tape(p, k));
  GW_CHECK(grad_out && (n == 0 || grads), "null argument");
  GW_CUDA(cudaSetDevice(p->device));
  cudaStream_t st = (cudaStream_t)stream;
  GW_TRY(gw::train_backward(p, p->train, k, grad_out, grad_features, st));
  for (int i = 0; i < n; ++i) {  // gradients are handed out under the reference's parameter names, shaped like the parameters
    GW_CHECK(grads[i].name && grads[i].data, "malformed gw_param entry");
    auto it = p->params.find(grads[i].name);
    GW_CHECK(it != p->params.end(), std::string("gw_train_backward: unknown parameter '") + grads[i].name + "'");
    const size_t cnt = (size_t)it->second.second.first * it->second.second.second;
    GW_CHECK((size_t)grads[i].rows * grads[i].cols == cnt, std::string("gw_train_backward: shape of '") + grads[i].name + "' differs");
    GW_CUDA(cudaMemcpyAsync(const_cast<float*>(grads[i].data), p->train->gbuf.p + (it->second.first - p->wbuf.p), cnt * sizeof(float),
                            cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

int gw_train_backward(gw_plan* p, const float* grad_out, float* grad_features, const gw_param* grads, int32_t n, void* stream) {
  GW_CHECK(p != nullptr, "null argument");
  GW_CHECK(p->train != nullptr, "gw_train_backward needs a preceding gw_train_forward");
  return gw_train_backward_tape(p, &p->train->own, grad_out, grad_features, grads, n, stream);
}

int64_t gw_train_peak_bytes(const gw_plan* p) { return (p && p->train) ? (int64_t)p->train->peak_bytes : 0; }

int gw_plan_set_output_peers(gw_plan* p, int32_t mode, int32_t n, const int64_t* deltas_bytes) {
  GW_CHECK(p != nullptr, "null plan");
  GW_CHECK(mode == 0 || (mode == 1 && n == 1 && deltas_bytes) || (mode == 2 && n >= 1 && n <= 8 && deltas_bytes), "bad mode / count");
  p->out_mode = mode, p->n_out_peers = mode == 2 ? n : 0;
  for (int j = 0; j < 8; ++j) p->out_delta[j] = (mode != 0 && j < n) ? deltas_bytes[j] : 0;
  return 0;
}

int gw_latent_edge_features(gw_plan* p, float* edge_attr_out, void* stream) {
  GW_CHECK(p && edge_attr_out, "null argument");
  GW_CHECK(!p->train_only, "this plan was made by gw_plan_create_train: it holds no encoded latent edges");
  GW_CHECK(p->w_enc && p->have_lat, "needs the latent graph and encoder.* weights");
  GW_CUDA(cudaMemcpyAsync(edge_attr_out, p->e_lat.p, p->e_lat.bytes(), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

int gw_plan_status(gw_plan* p, int32_t* status_out, void* stream) {
  GW_CHECK(p && status_out, "null argument");
  cudaSetDevice(p->device);
  cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
  volatile int32_t* h = p->tc_status_host;
  *status_out = h[0];
  if (e != cudaSuccess) {  // e.g. a trap: report what the device recorded (the block is host memory, still readable)
    gw::set_error(std::string("device fault: ") + cudaGetErrorString(e) + "; status word " + std::to_string(h[0]) +
                  " (per-warp wait records: gw_plan_debug)");
    return 1;
  }
  if (h[0]) h[0] = 0;
  return 0;
}

int gw_plan_status_peek(gw_plan* p, int32_t* status_out) {
  GW_CHECK(p && status_out, "null argument");
  *status_out = ((volatile int32_t*)p->tc_status_host)[0];  // host-mapped word: no CUDA call, no synchronisation
  return 0;
}

int gw_debug_trace_next(gw_plan* p, int32_t tag, int64_t* device_buf) {
  GW_CHECK(p != nullptr, "null plan");
  p->trace_buf = (long long*)device_buf;
  p->trace_tag = tag;
  return 0;
}

int gw_plan_debug(gw_plan* p, int32_t* out16) {
  GW_CHECK(p && out16, "null argument");
  for (int i = 0; i < 64; ++i) out16[i] = ((volatile int32_t*)p->tc_status_host)[i];
  return 0;
}

int gw_timing_enable(gw_plan* p, int32_t on) {
  GW_CHECK(p != nullptr, "null plan");
  p->timing = on != 0;
  p->stamps.clear();
  p->ev_used = 0;
  return 0;
}

int32_t gw_timing_num_tags(void) { return gw::TAG_COUNT; }
const char* gw_timing_tag_name(int32_t tag) { return (tag >= 0 && tag < gw::TAG_COUNT) ? gw::kTagNames[tag] : ""; }

int gw_timing_read(gw_plan* p, int64_t* launches, double* ms, void* stream) {
  GW_CHECK(p && launches && ms, "null argument");
  GW_CUDA(cudaSetDevice(p->device));
  GW_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  for (int t = 0; t < gw::TAG_COUNT; ++t) launches[t] = 0, ms[t] = 0.0;
  for (const auto& s : p->stamps) {
    float f = 0.f;
    GW_CUDA(cudaEventElapsedTime(&f, s.a, s.b));
    launches[s.tag] += 1;
    ms[s.tag] += f;
  }
  p->stamps.clear();
  p->ev_used = 0;
  return 0;
}

}  // extern "C"
