// gw_api.cu -- the C ABI of libgwb200.so (include/gw_b200.h) outside the training step: version, errors, launch count, plan
// create / destroy, graph and weight upload, the forward entry points (gw_forward.cu), output peers, status, debug, timing.
#include "gw_plan.h"

#include <memory>

namespace gw {

static thread_local std::string g_err;
static thread_local long long g_launches = 0;
void set_error(const std::string& msg) { g_err = msg; }
void count_launch(int n) { g_launches += n; }

int check_ready(gw_plan* p, int batch, int need) {
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

// the training state first (its live tapes are released and left dead), then the host resources; the device buffers go with
// their members
gw_plan::~gw_plan() {
  gw::train_destroy(this);
  if (tc_status_host) cudaFreeHost(tc_status_host);
  for (cudaEvent_t e : ev_pool) cudaEventDestroy(e);
}

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
  const bool tc = gw::is_fused(p);  // (a layer-by-layer plan has the CUDA-core path's scratch, and its assembled operands)
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
  if (p->layered)  // [x ; per-node sums of e'] of the encoder / processor node MLPs, per-point sums of the decoder's
    rc |= p->cat.alloc(std::max(B * d.n_mesh * (Dn + De), chunk * d.n_out * De));
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
  // tensor-core plans: the fused chains for the reference's default trunk (256-wide node / edge / hidden, 2 hidden layers), and
  // for a trunk at least 256 wide with a width above 256 (train/run.py's 1024-wide model), a plan that runs the forward layer by
  // layer as tensor-core column blocks, any number of hidden layers
  const int trunk[4] = {d.node_dim, d.edge_dim, d.hidden_node, d.hidden_edge};
  const bool wide = *std::min_element(trunk, trunk + 4) >= 256 && *std::max_element(trunk, trunk + 4) > 256;
  if (d.precision != GW_PREC_FP32_SIMT) {
    GW_CHECK(wide || (d.node_dim == 256 && d.edge_dim == 256 && d.hidden_node == 256 && d.hidden_edge == 256),
             "the tensor-core precisions need node/edge/hidden dims of 256 (the reference default) or a trunk at least 256 wide with "
             "one width above 256; use fp32_simt otherwise");
    GW_CHECK(wide || (d.hidden_layers_node == 2 && d.hidden_layers_edge == 2),
             "the tensor-core chains of the 256-wide trunk are built for hidden_layers = 2");
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
  std::unique_ptr<gw_plan> p(new gw_plan());  // a failure below frees the plan and whatever it already holds
  p->d = d;
  p->train_only = train_only;
  p->layered = d.precision != GW_PREC_FP32_SIMT && wide;
  p->row_images.tag = gw::TAG_CONST;
  GW_CHECK(!(train_only && p->layered), "the training step's tensor-core precisions need the 256-wide trunk; use fp32_simt");
  GW_CUDA(cudaGetDevice(&p->device));
  const size_t Dn = d.node_dim, De = d.edge_dim, He = d.hidden_edge, Hn = d.hidden_node;
  const size_t max_hid = std::max({Dn, De, He, Hn, (size_t)d.hidden_dec, (size_t)d.out_dim});
  const size_t max_rows = std::max({(size_t)d.n_in, (size_t)d.n_out, (size_t)d.n_mesh, (size_t)d.n_lat_edges, (size_t)d.n_dec_edges});
  // chunking: keep the per-pass scratch of the lat/lon-sized stages under ~24 GB (an 80 GB H100 also holds the caller's tensors).  The tensor-core path never writes the
  // decoder's e' rows (their per-point sums are formed in the edge chain's epilogue), and its hidden activations stay on
  // the SM, so its per-sample scratch is three lat/lon-sized row buffers; the CUDA-core path also needs e' and the ping-pong.
  const bool tc = gw::is_fused(p.get());
  const size_t n_io = std::max((size_t)d.n_in, (size_t)d.n_out);
  const size_t dec_tiles = ((size_t)d.n_dec_edges + 127) / 128;
  const size_t per_sample = tc ? (n_io * Dn + (size_t)d.n_in * De + (size_t)d.n_out * De + dec_tiles * 2048) * sizeof(float)
                               : (2 * max_rows * max_hid + std::max((size_t)d.n_in, (size_t)d.n_dec_edges) * De + n_io * Dn +
                                  (p->layered ? (size_t)d.n_out * De : 0)) * sizeof(float);
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
  if (!train_only) rc |= alloc_inference_scratch(p.get(), chunk);
  GW_TRY(rc);
  {  // zeroed on a private non-blocking stream and complete on return: the plan's first call may come from any stream, also one
     // not ordered against the legacy default stream (cudaDeviceSynchronize would instead wait for whatever the caller queued there)
    cudaStream_t zs = nullptr;
    GW_CUDA(cudaStreamCreateWithFlags(&zs, cudaStreamNonBlocking));
    cudaError_t e = cudaMemsetAsync(p->zeros_h3.p, 0, p->zeros_h3.bytes(), zs);
    if (e == cudaSuccess) e = cudaMemsetAsync(p->bounds.p, 0, p->bounds.bytes(), zs);
    if (e == cudaSuccess) e = cudaStreamSynchronize(zs);
    cudaStreamDestroy(zs);
    GW_CUDA(e);
  }
  GW_CUDA(cudaHostAlloc((void**)&p->tc_status_host, 64 * sizeof(int32_t), cudaHostAllocMapped));
  std::memset(p->tc_status_host, 0, 64 * sizeof(int32_t));
  GW_CUDA(cudaHostGetDevicePointer((void**)&p->tc_status_dev, p->tc_status_host, 0));
  p->n_in_cur = d.n_in;
  *out_plan = p.release();
  return 0;
}

int gw_plan_create(const gw_dims* dims, gw_plan** out_plan) { return plan_create(dims, out_plan, false); }
int gw_plan_create_train(const gw_dims* dims, gw_plan** out_plan) { return plan_create(dims, out_plan, true); }

int gw_plan_destroy(gw_plan* p) {
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
  ++p->graph_gen;
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
  ++p->graph_gen;
  p->w_enc = p->w_proc = p->w_dec = false;
  return 0;
}

int gw_plan_set_h3_nodes(gw_plan* p, const float* rows, void* stream) {
  GW_CHECK(p && rows, "null argument");
  auto it = p->params.find("encoder.h3_nodes");
  GW_CHECK(it != p->params.end() && p->b_enc && p->h3_nodes == it->second.first,
           "gw_plan_set_h3_nodes: the plan's weights bind no encoder.h3_nodes (gw_plan_set_weights first, with an encoder.* group)");
  cudaStream_t st = (cudaStream_t)stream;
  GW_CUDA(cudaSetDevice(p->device));
  GW_CUDA(cudaMemcpyAsync(const_cast<float*>(p->h3_nodes), rows, (size_t)p->d.n_mesh * p->d.in_dim * 4, cudaMemcpyDeviceToDevice, st));
  ++p->graph_gen;  // (a tape's backward differentiates the rows its forward read)
  p->w_enc = p->b_enc, p->w_proc = p->b_proc, p->w_dec = p->b_dec;  // the views stay valid: only the constants follow the graphs
  if (!p->train_only) GW_TRY(gw::precompute_constants(p, st));
  return 0;
}

int gw_segment_sum(const float* rows, int64_t n_rows, int32_t width, const int32_t* perm, const int32_t* ptr, int32_t n_seg, float* out,
                   void* stream) {
  GW_CHECK(rows && perm && ptr && out, "null argument");
  GW_CHECK(n_rows >= 0 && n_rows <= INT32_MAX && width >= 1 && n_seg >= 1, "bad sizes");
  GW_CUDA(gw::launch_segsum(rows, width, width, ptr, perm, (int)n_rows, n_seg, 1, out, width, (cudaStream_t)stream));
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
  if (gw::is_fused(p)) GW_TRY(gw::pack_tc_weights(p, st));
  if (p->layered) p->row_images.new_weights(p->wbuf.p);  // (packed on their first use, by the constants below)
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
