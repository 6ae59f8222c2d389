// gw_forward.cu -- the plan's weights (lookup, binding, tensor-core weight images), the weight-constant precompute, and the
// encode-process-decode forward expressed as chains of gw::GemmOp row ops.
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
#include "gw_plan.h"

namespace gw {

int run_op(gw_plan* p, const GemmOp& op, cudaStream_t st) {
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

int run_chain(gw_plan* p, TcChain& ch, cudaStream_t st) {
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
bool is_tc(const gw_plan* p) { return p->d.precision != GW_PREC_FP32_SIMT; }

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

int bind_all(gw_plan* p) {
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
int pack_tc_weights(gw_plan* p, cudaStream_t st) {
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
int precompute_encoder_constants(gw_plan* p, cudaStream_t st) {
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

int precompute_constants(gw_plan* p, cudaStream_t st) {
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
int stage_encoder(gw_plan* p, const float* features, float* x_out, float* x_out_bound, int nb, cudaStream_t st) {
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
int stage_processor(gw_plan* p, const ProcGraph& g, const float* x_in, float* x_out, int x_in_slot, int x_out_slot, int nb,
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
ProcGraph latent_graph_of(gw_plan* p) {
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

int stage_decoder(gw_plan* p, const float* x_in, int x_in_slot, const float* start, int start_ld, float* out, int out_ld, int nb,
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
int csr_stats(gw_plan* p, const int32_t* ptr, int n, int32_t* dst, int* maxdeg, int* mindeg, cudaStream_t st) {
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
int encoder_degree(gw_plan* p, cudaStream_t st) {
  static const int init[2] = {0, 0x7fffffff};
  GW_CUDA(cudaMemcpyAsync(p->enc_deg.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
  GW_CUDA(launch_csr_expand(p->enc_ptr.p, p->d.n_mesh, nullptr, p->enc_deg.p, st));
  if (p->enc_chunk_seg.p)  // chunk table of the two-level segment sum follows the graph
    GW_CUDA(launch_seg_chunks(p->enc_ptr.p, p->d.n_mesh, p->enc_chunk_seg.p, p->enc_chunk_j0.p, p->enc_seg_chunk0.p, st));
  return 0;
}

}  // namespace gw
