// gw_plan.h -- what the translation units of libgwb200.so's host side share: the error macros, the plan (struct gw_plan), row-source
// constructors, magnitude-bound slots, per-launch timing, and the functions one unit calls in another.  gw_forward.cu holds the
// weights, the weight constants and the inference stages; gw_train.cu the training step (TrainState and gw_tape are its own: the
// plan keeps an opaque pointer); gw_api.cu the C ABI of include/gw_b200.h around them.
#pragma once

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

struct TrainState;  // gw_train.cu

}  // namespace gw

using namespace gw;

struct gw_plan {
  gw::TrainState* train = nullptr;  // training step state (gw_train.cu), created on first use, torn down by train_destroy
  bool train_only = false;          // gw_plan_create_train: graphs, weights and the bounded-memory (chunked) training step only
  int train_chunk_pts = 0;          // GW_B200_TRAIN_CHUNK: points per chunk of that step (0: from the shapes, gw_train.cu)
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

inline RowSrc src_stream(const float* base, int ld, int width, int rows_per_sample, int col0 = 0) {
  RowSrc s;
  s.kind = SRC_STREAM, s.base = base, s.ld = ld, s.width = width, s.src_rows = rows_per_sample, s.col0 = col0;
  return s;
}
inline RowSrc src_bcast(const float* base, int ld, int width, int col0 = 0) {
  RowSrc s;
  s.kind = SRC_BCAST, s.base = base, s.ld = ld, s.width = width, s.col0 = col0;
  return s;
}
inline RowSrc src_gather(const float* base, int ld, int width, const int32_t* idx, int src_rows, int col0 = 0) {
  RowSrc s;
  s.kind = SRC_GATHER, s.base = base, s.ld = ld, s.width = width, s.idx = idx, s.src_rows = src_rows, s.col0 = col0;
  return s;
}
inline RowSrc src_bgather(const float* base, int ld, int width, const int32_t* idx) {
  RowSrc s;
  s.kind = SRC_BGATHER, s.base = base, s.ld = ld, s.width = width, s.idx = idx;
  return s;
}
inline RowSrc src_segsum(const float* base, int ld, int width, const int32_t* ptr, const int32_t* perm, int src_rows) {
  RowSrc s;
  s.kind = SRC_SEGSUM, s.base = base, s.ld = ld, s.width = width, s.ptr = ptr, s.perm = perm, s.src_rows = src_rows;
  return s;
}
inline RowSrc src_gather_bcast_relu(const float* base, int ld, int width, const int32_t* idx, int src_rows,
                                    const float* base2, int ld2) {
  RowSrc s;
  s.kind = SRC_GATHER_BCAST_RELU, s.base = base, s.ld = ld, s.width = width, s.idx = idx, s.src_rows = src_rows;
  s.base2 = base2, s.ld2 = ld2;
  return s;
}

// magnitude-bound slots (gw_plan::bounds)
enum BoundSlot { SL_FEAT = 0, SL_XIN, SL_XOUT, SL_X0, SL_X1, SL_E0, SL_E1, SL_EIN, SL_P, SL_AGG_MESH, SL_AGG_GRID, SL_ROWS_N, SL_ROWS_E,
                 SL_EENC, SL_C1ENC, SL_XM0, SL_ELAT, SL_EDEC, SL_E1DEC, SL_SDEC, SL_COUNT };
inline float* sl(gw_plan* p, int i) { return p->bounds.p + i; }
inline RowSrc bounded(RowSrc s, const float* b, float mul = 1.f) {
  s.bound = b, s.bound_mul = mul;
  return s;
}
// |x| of a raw caller tensor -> slot (the slot is reset first: absmax accumulates with atomicMax)
inline int raw_bound(gw_plan* p, int slot, const float* x, long long n, cudaStream_t st) {
  GW_CUDA(cudaMemsetAsync(sl(p, slot), 0, sizeof(float), st));
  GW_CUDA(launch_absmax_flat(x, n, sl(p, slot), st));
  return 0;
}

// (the training step's phases, gw_train.cu: taped forward products, data gradients, weight gradients, operand bounds, the
// memory-bound rest -- LayerNorm backward, segment sums, gathers, batch reductions -- and the per-weight work done once per weight
// upload: transposes and weight images)
enum KernelTag { TAG_CONST = 0, TAG_ENC_GRID, TAG_ENC_MESH, TAG_PROC_P, TAG_PROC_EDGE, TAG_PROC_NODE, TAG_DEC_P, TAG_DEC_EDGE,
                 TAG_DEC_NODE, TAG_TRAIN_FWD, TAG_TRAIN_DGRAD, TAG_TRAIN_WGRAD, TAG_TRAIN_PACK, TAG_TRAIN_OTHER, TAG_TRAIN_WEIGHTS,
                 TAG_COUNT };
static const char* const kTagNames[TAG_COUNT] = {"const", "enc_grid", "enc_mesh", "proc_p", "proc_edge", "proc_node", "dec_p",
                                                 "dec_edge", "dec_node", "train_fwd", "train_dgrad", "train_wgrad", "train_pack",
                                                 "train_other", "train_weights"};

inline cudaEvent_t take_event(gw_plan* p) {
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

inline GemmOp first_op(int rows, int batch, const RowSrc& a0, const RowSrc& a1, const float* W, int K, int ldw,
                       const float* bias) {
  GemmOp op;
  op.rows_per_sample = rows, op.batch = batch;
  op.a[0] = a0, op.a[1] = a1;
  op.W = W, op.K = K, op.ldw = ldw, op.bias = bias;
  return op;
}

// the graph stage_processor runs on (gw_forward.cu describes it)
struct ProcGraph {
  int H, El;
  const int32_t *src, *dst, *ptr;
  const float* e0;
  bool e0_broadcast;
  int maxdeg, mindeg;    // longest / shortest per-node segment of incoming edges
  const float* e0_bound; // magnitude bound of e0
};

// gw_forward.cu
int run_op(gw_plan* p, const GemmOp& op, cudaStream_t st);
int run_chain(gw_plan* p, TcChain& ch, cudaStream_t st);
bool is_tc(const gw_plan* p);
int bind_all(gw_plan* p);
int pack_tc_weights(gw_plan* p, cudaStream_t st);
int precompute_encoder_constants(gw_plan* p, cudaStream_t st);
int precompute_constants(gw_plan* p, cudaStream_t st);
int stage_encoder(gw_plan* p, const float* features, float* x_out, float* x_out_bound, int nb, cudaStream_t st);
int stage_processor(gw_plan* p, const ProcGraph& g, const float* x_in, float* x_out, int x_in_slot, int x_out_slot, int nb,
                    cudaStream_t st);
ProcGraph latent_graph_of(gw_plan* p);
int stage_decoder(gw_plan* p, const float* x_in, int x_in_slot, const float* start, int start_ld, float* out, int out_ld, int nb,
                  cudaStream_t st);
int csr_stats(gw_plan* p, const int32_t* ptr, int n, int32_t* dst, int* maxdeg, int* mindeg, cudaStream_t st);
int encoder_degree(gw_plan* p, cudaStream_t st);

// gw_api.cu: the plan holds what the stages in `need` read, and `batch` fits it; makes the plan's device current
enum { NEED_ENC = 1, NEED_PROC = 2, NEED_DEC = 4, NEED_INFER = 8 };
int check_ready(gw_plan* p, int batch, int need);

// gw_train.cu: releases the plan's training state for gw_plan_destroy; live tapes lose their memory and stay as dead handles
void train_destroy(gw_plan* p);

}  // namespace gw
