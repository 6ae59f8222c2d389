/* gw_b200.h -- C ABI of libgwb200.so: the H100 (sm_90a) encode-process-decode forward of graph_weather.
 *
 * The reference is pure Python (SURVEY.md section 2a: no native code, no FFI), so there is no existing C interface
 * to mirror; each entry point below names the reference Python call it replaces.  A maintainer binds this library
 * from Python with ctypes (INTEGRATION.md shows the stub); graph_weather_b200/_capi.py is that binding.
 *
 * Conventions
 *   - plain pointers and sizes only; device pointers unless the name says host; all floating point is fp32,
 *     row-major contiguous; indices are int32 (the reference's int64 edge_index is narrowed by the caller).
 *   - every function returns 0 on success, non-zero on failure; gw_last_error() gives the message
 *     (thread-local).  Nothing throws across the ABI.  There is NO CPU fallback: every compute entry point
 *     fails if no CUDA device / kernel image is available.
 *   - the caller owns every buffer it passes.  The plan owns only its scratch, packed weights and the
 *     weight-constant tensors it precomputes.  No global state; plans are independent (one per GPU rank).
 *   - `stream` is a cudaStream_t passed as void*, and may be any stream of the plan's device, also a non-blocking one.  A call
 *     does all its device work on that stream; the only exception is gw_plan_create, which zeroes the new plan's buffers on a
 *     private stream and waits for that before it returns.  Calls on one plan share its scratch: when they come from
 *     different streams, the caller orders each after the previous one (graph_weather_b200/_capi.py does, with an event per
 *     plan).
 */
#ifndef GW_B200_H
#define GW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GW_ABI_VERSION 2

/* arithmetic mode of the MLP contractions */
#define GW_PREC_FP32_SIMT 0 /* fp32 FFMA on CUDA cores (exact fp32; any hidden size)                              */
#define GW_PREC_FP32_TC 1   /* wgmma f16, each fp32 operand split hi+lo (2x fp16), 3 MMAs, fp32 accumulate         */
#define GW_PREC_BF16_TC 2   /* wgmma bf16 operands, single MMA, fp32 accumulate (configs 3/4)                       */

typedef struct gw_plan gw_plan; /* opaque */

/* Sizes of one model + graph set.  Mirrors the constructor arguments of GraphWeatherForecaster (forecast.py:64-84)
 * and GraphWeatherAssimilator (analysis.py:55-72) plus the graph sizes the reference derives from lat_lons. */
typedef struct gw_dims {
  int32_t n_in;        /* input lat/lon (or observation) points: encoder.num_latlons                 */
  int32_t n_out;       /* output lat/lon points: decoder.num_latlons (== n_in for the forecaster)    */
  int32_t n_mesh;      /* H3 cells: 2+120*7^res (5882 at res 2)                                      */
  int32_t n_lat_edges; /* latent edges (41162 at res 2)                                              */
  int32_t n_dec_edges; /* decoder edges (~7*n_out)                                                   */
  int32_t in_dim;      /* feature_dim+aux_dim (102) / observation_dim (2)                            */
  int32_t enc_edge_attr_dim; /* 2 (forecaster) or 3 (assimilator: + height)                          */
  int32_t out_dim;     /* output_dim (78) / analysis_dim                                             */
  int32_t residual_dim;/* >0: out += features[..., :residual_dim] (decoder.py:93); 0: none           */
  int32_t node_dim, edge_dim;                 /* 256, 256 */
  int32_t hidden_node, hidden_edge;           /* hidden_dim_processor_{node,edge}: 256 */
  int32_t hidden_layers_node, hidden_layers_edge; /* 2, 2 */
  int32_t hidden_dec, hidden_layers_dec;      /* 128, 2 */
  int32_t num_blocks;                         /* processor blocks: 9 */
  int32_t precision;                          /* GW_PREC_* */
  int32_t max_batch;                          /* scratch is sized for this many samples per call */
} gw_dims;

/* One named fp32 parameter tensor; `name` is the reference state_dict key
 * (e.g. "processor.graph_processor.blocks.3.edge_model.edge_mlp.model.0.weight", [256,768] row-major). */
typedef struct gw_param {
  const char* name;
  const float* data; /* device */
  int64_t rows, cols; /* 1-D tensors: rows = n, cols = 1 */
} gw_param;

int gw_abi_version(void);
const char* gw_last_error(void);

/* Replaces: GraphWeatherForecaster.__init__ / GraphWeatherAssimilator.__init__ module construction
 * (forecast.py:129-170, analysis.py:96-134).  Allocates scratch for dims->max_batch samples on the current device. */
int gw_plan_create(const gw_dims* dims, gw_plan** out_plan);
int gw_plan_destroy(gw_plan* plan);
/* A plan for training only (GraphWeatherForecaster(use_checkpointing=True)): graphs, weights and the training state, none of
 * the inference scratch, packed inference weights or weight constants.  gw_plan_set_weights on it binds the weights only;
 * gw_forward, gw_forward_strided, the stage entry points and gw_latent_edge_features on it fail.  Its training step (the
 * whole network's, and the standalone encoder's and decoder's, gw_train_{encoder,decoder}_*_tape) is the
 * bounded-memory one: gw_train_forward_tape keeps only the mesh-sized activations and the output, and gw_train_backward_tape recomputes
 * the grid-sized stages (the encoder's lat/lon side, the decoder) chunk by chunk with the forward's own ops, releasing each
 * chunk's temporaries before the next.  Its peak working memory grows with the grid by at most one chunk.  Chunks hold a fixed
 * working-set budget divided by the batch, chosen from the shapes alone (never from free device memory): encoder chunks are whole
 * mesh slots, decoder chunks runs of consecutive points.  The forward equals the taped step's bit for bit in GW_PREC_FP32_SIMT and
 * GW_PREC_BF16_TC (GW_PREC_FP32_TC scales each chunk's operands from the chunk); gradients equal it up to fp32 summation order. */
int gw_plan_create_train(const gw_dims* dims, gw_plan** out_plan);
/* bytes of device memory the plan holds (scratch + packed weights + constants) */
int64_t gw_plan_device_bytes(const gw_plan* plan);

/* Graph upload (all device int32 / fp32 arrays, copied into the plan).
 * Replaces the graphs built at encoder.py:76-109,244-268 and assimilator_decoder.py:69-106.
 *   encoder : one edge per input point p -> mesh slot enc_mesh[p] in [0,n_mesh); attr [n_in, enc_edge_attr_dim];
 *             perm[n_in] = points sorted by mesh slot (ties in point order), ptr[n_mesh+1] = CSR over slots into perm.
 *             n_in may be smaller than gw_dims.n_in (the assimilator rebuilds this graph per call,
 *             assimilator_encoder.py:118,170-216); if weights are loaded its constants are refreshed.
 *   latent  : edges SORTED BY TARGET: src[j], dst[j] (non-decreasing), ptr[n_mesh+1] CSR over dst; attr [El,2]
 *   decoder : edges grouped by output point: src[j] mesh slot, ptr[n_out+1]; attr [Ed,2]                      */
int gw_plan_set_encoder_graph(gw_plan* plan, int32_t n_in, const int32_t* enc_mesh, const int32_t* perm,
                              const int32_t* ptr, const float* attr, void* stream);
/* Device-side construction of the assimilator's per-call observation graph
 * (AssimilatorEncoder.create_input_graph, assimilator_encoder.py:170-216: h3.latlng_to_cell + great_circle_distance per
 * observation in a Python loop).  gw_plan_set_h3_tables uploads, once, the hexagonal-grid tables of the plan's resolution
 * (all DEVICE pointers, copied): face_frames [20][9] = centre, i-axis, j-axis unit vectors of every icosahedron face;
 * cell_of [20][(2 lattice_n + 1)^2] = canonical cell of each face-lattice point or -1; cell_slot [n_cells] = mesh slot of the
 * cell (H-1-rank, the encoder's numbering, encoder.py:80-84); cell_lat / cell_lng [n_cells] radians; scale, rot_cos,
 * rot_sin: gnomonic plane -> lattice transform of the resolution.  gw_plan_build_obs_graph then replaces
 * gw_plan_set_encoder_graph for every forward: lat_lon_heights [n_obs, 3] fp32 degrees / degrees / height on the device ->
 * mesh slot, [sin d, cos d, height] edge attributes, slot-sorted permutation and CSR inside the plan; no host copy, no
 * synchronisation. */
int gw_plan_set_h3_tables(gw_plan* plan, int32_t res, int32_t n_cells, int32_t lattice_n, const double* face_frames, const int32_t* cell_of,
                          const int32_t* cell_slot, const double* cell_lat, const double* cell_lng, double scale, double rot_cos,
                          double rot_sin, void* stream);
int gw_plan_build_obs_graph(gw_plan* plan, const float* lat_lon_heights, int32_t n_obs, void* stream);

int gw_plan_set_latent_graph(gw_plan* plan, const int32_t* src, const int32_t* dst, const int32_t* ptr,
                             const float* attr, void* stream);
int gw_plan_set_decoder_graph(gw_plan* plan, const int32_t* src, const int32_t* ptr, const float* attr, void* stream);

/* Replaces: load_state_dict on the reference module.  Looks parameters up by reference key name, packs them for
 * the selected precision, then recomputes every weight-constant tensor (edge encoders on the fixed graphs,
 * node_encoder(h3_nodes), the constant layer-1 terms).  Must follow the graph uploads; call again after any weight
 * or graph change.  `params` is a host array of n entries whose `data` are device pointers.  The table may hold
 * any subset of the groups "encoder.*", "processor.*", "decoder.*" (the reference's sub-modules can be built and
 * called on their own, tests/test_model.py:20-119); a stage whose group or graph is missing fails when called.
 * "decoder.node_decoder" may end in a LayerNorm ("...model.{2 L + 1}.weight/bias" present): the regional forecaster builds
 * its node decoder with the configured norm (regional_forecast.py:224-231), the forecaster / assimilator decoders without. */
int gw_plan_set_weights(gw_plan* plan, const gw_param* params, int32_t n, void* stream);

/* Plans whose graphs change between calls without a weight change (RegionalForecaster.forward_regions: a batch of regions run
 * as one graph, a new set of regions per call).  After the call's graph uploads, gw_plan_set_h3_nodes copies rows [n_mesh, in_dim]
 * (device) over the "encoder.h3_nodes" table gw_plan_set_weights bound, binds again the weight groups that upload bound (graph
 * uploads unbind them) and recomputes the weight constants on the new graphs -- without copying or re-packing any weight.  Like a
 * latent or decoder graph upload it moves the plan's graph generation: a training backward whose forward ran on the earlier
 * graphs or rows refuses.
 * gw_segment_sum: out[s, :] = sum of rows[perm[j], :] over j in [ptr[s], ptr[s+1]), in j order (rows [n_rows, width], perm, ptr
 * [n_seg + 1], out [n_seg, width]; all device).  A fixed-order sum without atomics: forward_regions adds the h3_nodes gradient
 * rows of a cell that several regions share into the cell's row of the table. */
int gw_plan_set_h3_nodes(gw_plan* plan, const float* rows, void* stream);
int gw_segment_sum(const float* rows, int64_t n_rows, int32_t width, const int32_t* perm, const int32_t* ptr, int32_t n_seg, float* out,
                   void* stream);

/* Replaces: GraphWeatherForecaster.forward (forecast.py:215-247, constraint_type="none") and
 * GraphWeatherAssimilator.forward (analysis.py:136-150) after its per-call input graph is uploaded.
 *   features [batch, n_in, in_dim]  ->  out [batch, n_out, out_dim];  batch <= max_batch.                     */
int gw_forward(gw_plan* plan, const float* features, float* out, int32_t batch, void* stream);

/* gw_forward with a caller-chosen row stride of `out` (floats, >= out_dim): an autoregressive rollout lets step t write its
 * forecast straight into the first out_dim columns of step t+1's feature rows (out = next_features, out_ld = in_dim), so
 * no concatenation pass exists between steps. */
int gw_forward_strided(gw_plan* plan, const float* features, float* out, int32_t out_ld, int32_t batch, void* stream);

/* Training step (SURVEY.md 8(f) row 2: "then backward"; every caller of the reference trains, train/run.py:508-543).  A tape holds
 * what one training forward saves for its backward.  gw_train_forward_tape is gw_forward that keeps the activations the backward
 * needs on `tape` (a second forward on the same tape replaces the first); gw_train_backward_tape consumes them: grad_out
 * [batch, n_out, out_dim] -> gradients of every parameter, copied into the caller's tensors named like the parameters (`grads`:
 * reference state_dict keys, device pointers, parameter shapes), and, if grad_features is not NULL, the gradient of the input
 * features [batch, n_in, in_dim].  One backward per forward.  LayerNorm MLPs, dims <= 256.  The plan's precision is the step's
 * arithmetic: GW_PREC_FP32_SIMT exact fp32 on CUDA cores (weight gradients accumulated with float atomics: repeatable to ~1e-7
 * relative, not bit for bit); GW_PREC_FP32_TC (fp16 hi/lo split, 3 MMAs per product) or GW_PREC_BF16_TC (bf16 operands) on wgmma
 * tensor cores with fp32 accumulation, fp32 tape and fp32 gradients -- 256-wide dims and 2 hidden layers, sm_90a; their weight
 * gradients of layers with more than 16 inputs are reduced in a fixed order (bit for bit repeatable).  Timing tags train_fwd,
 * train_dgrad, train_wgrad, train_pack (operand bounds), train_other and train_weights split a step (gw_timing_read).  The
 * per-weight work -- transposed weights and, on tensor cores, the weight images -- is done once per gw_plan_set_weights, by the
 * first step after it (tag train_weights).
 * Several tapes keep several forwards alive at once (a loss summed over a multi-step rollout, back-propagated once).  Tapes of one
 * plan share its weights, graphs and gradient buffer; their calls are ordered like every other call on the plan (Conventions).
 * Batches may differ between tapes.
 *   gw_tape_destroy releases the tape's memory stream-ordered on `stream` and frees the handle: from another stream than the
 *   tape's last forward or backward, the caller orders it after that call as it orders any call on the plan.
 *   gw_plan_destroy releases the memory of every tape of the plan and leaves them dead: a forward or backward on a dead tape
 *   fails (gw_tape_destroy still frees the handle).
 *   A backward fails when gw_plan_set_weights ran after the tape's forward (its gradient would be taken at other weights).
 *   gw_tape_bytes: the bytes the tape holds -- between its forward and backward, what the forward saved (shape-determined);
 *   0 after the backward. */
typedef struct gw_tape gw_tape; /* opaque */
int gw_tape_create(gw_plan* plan, gw_tape** out_tape);
int gw_tape_destroy(gw_tape* tape, void* stream);
int gw_train_forward_tape(gw_plan* plan, gw_tape* tape, const float* features, float* out, int32_t batch, void* stream);
int gw_train_backward_tape(gw_plan* plan, gw_tape* tape, const float* grad_out, float* grad_features, const gw_param* grads,
                           int32_t n, void* stream);
int64_t gw_tape_bytes(const gw_tape* tape);
/* The training step of one stage alone, on a tape of a plan that holds that stage (the reference's sub-modules are ordinary
 * differentiable modules, tests/test_model.py:20-119).  The encoder and decoder calls run the step of their plan: the taped step on
 * a gw_plan_create plan; on a gw_plan_create_train plan the bounded-memory step (Encoder / Decoder(use_checkpointing=True)), whose
 * forward keeps only the mesh-sized activations and whose backward recomputes the lat/lon side chunk by chunk, as the whole
 * network's.  The processor calls take a gw_plan_create plan only: the processor has no grid-sized work, and
 * gw_train_set_processor_segments bounds its memory.  Replaces the autograd backward of Encoder.forward (encoder.py:153-242)
 * and AssimilatorEncoder.forward (assimilator_encoder.py:118-168), Processor.forward (processor.py:83-128), Decoder.forward
 * (decoder.py:79-94) and AssimilatorDecoder.forward (assimilator_decoder.py:131-200).  The whole-network step above is these three
 * stages composed.  Conventions as for gw_train_forward_tape / gw_train_backward_tape: one backward per forward, on the tape of a
 * forward of the same stage; a backward after gw_plan_set_weights fails; gradients are copied into `grads` under the reference's
 * state_dict names; gw_tape_bytes and gw_train_peak_bytes keep their meaning; the processor calls follow
 * gw_train_set_processor_segments; GW_PREC_FP32_TC / GW_PREC_BF16_TC bound the caller's x_in and edge_attr as they bound features
 * (status bit 3 on an inf / NaN).  Inputs a forward reads (features, x_in, edge_attr, start_features) are read again by its
 * backward: the caller keeps them unchanged until it has run.  Mesh rows are in slot order, as for the stage entry points below.
 *   encoder    features [batch, n_in, in_dim] -> x_out [batch*n_mesh, node_dim] and e_lat_out [n_lat_edges, edge_dim]: one sample's
 *              latent edge features in the plan's target-sorted order, as gw_latent_edge_features returns them (the reference
 *              repeats them per sample).  Backward: grad_x, grad_e_lat (summed over the samples; NULL: zero) -> parameter gradients
 *              and, unless grad_features is NULL, the features' gradient.  A backward fails once the encoder graph was replaced
 *              after its forward (the assimilator's per-call observation graph).  On a training-only plan, a forward on a new
 *              encoder graph copies its slot CSR to the host once to cut the chunks (a stream synchronisation per observation set).
 *   processor  on a caller-supplied graph, as gw_processor_forward_graph (copied onto the tape with its source-sorted CSR, so it
 *              may change on every call); x_out must not alias x_in.  Backward: grad_x_out [n_nodes, node_dim] -> parameter
 *              gradients, grad_x_in [n_nodes, node_dim] and grad_edge_attr [n_edges, edge_dim] per edge (either may be NULL).
 *   decoder    x_in [batch*n_mesh, node_dim] (+ start_features [batch, n_out, start_ld] when the plan has a residual) -> out.
 *              Backward: grad_out [batch, n_out, out_dim] -> parameter gradients and grad_x_in (NULL: none).  The residual's
 *              gradient, grad_out itself, is the caller's to add to start_features' gradient.  On a training-only plan the backward
 *              reads x_in and start_features again chunk by chunk. */
int gw_train_encoder_forward_tape(gw_plan* plan, gw_tape* tape, const float* features, float* x_out, float* e_lat_out, int32_t batch,
                                  void* stream);
int gw_train_encoder_backward_tape(gw_plan* plan, gw_tape* tape, const float* grad_x, const float* grad_e_lat, float* grad_features,
                                   const gw_param* grads, int32_t n, void* stream);
int gw_train_processor_forward_tape(gw_plan* plan, gw_tape* tape, const float* x_in, float* x_out, const float* edge_attr, int32_t n_nodes,
                                    int32_t n_edges, const int32_t* src, const int32_t* dst, const int32_t* ptr, void* stream);
int gw_train_processor_backward_tape(gw_plan* plan, gw_tape* tape, const float* grad_x_out, float* grad_x_in, float* grad_edge_attr,
                                     const gw_param* grads, int32_t n, void* stream);
int gw_train_decoder_forward_tape(gw_plan* plan, gw_tape* tape, const float* x_in, const float* start_features, int32_t start_ld, float* out,
                                  int32_t batch, void* stream);
int gw_train_decoder_backward_tape(gw_plan* plan, gw_tape* tape, const float* grad_out, float* grad_x_in, const gw_param* grads, int32_t n,
                                   void* stream);
/* Replaces: Processor.set_checkpoint_segments (processor.py:70-81) and GraphCast.set_checkpoint_processor (graphcast/model.py:149-163,
 * 230-250).  Processor segments of the training forwards that start after this call, on either training step: 0 (the default) keeps
 * the processor's whole tape; N > 0 cuts segments of N blocks (0..N-1, N..2N-1, ..., a shorter last one); -1, or any N >=
 * num_blocks, makes the processor one segment.  A forward with segments keeps only each segment's first x and e rows and the
 * processor's output, and its backward recomputes one segment at a time with the forward's own ops before differentiating it:
 * outputs and gradients are those of segments = 0 bit for bit (GW_PREC_FP32_SIMT weight gradients up to its float atomics), at
 * the cost of one more processor forward.  Each tape records the value its forward ran with, and its backward follows that, so
 * changing it between a forward and its backward is harmless.  gw_tape_bytes and gw_train_peak_bytes depend on the shapes and
 * this value only.  Values below -1 fail. */
int gw_train_set_processor_segments(gw_plan* plan, int32_t segments);
/* Replaces: torch.use_deterministic_algorithms(True) for the training backward (the Python layer sets it from
 * torch.are_deterministic_algorithms_enabled() right before each backward).  on != 0: the backwards that start after this call,
 * on either training step, sum every parameter gradient in an order that follows from the shapes alone, so that the same inputs,
 * weights and plan give the same gradients bit for bit on every run.  It switches the CUDA-core weight gradient (every weight in
 * GW_PREC_FP32_SIMT, Linears with at most 16 inputs in the tensor-core precisions) and the LayerNorm backward (every precision) from
 * float atomics to per-slab / per-CTA partials in a plan-shared workspace of at most 32 MiB (allocated on first use, released by
 * gw_plan_destroy) that a second kernel adds in order.  Every other part of the step already sums in a fixed order, and the
 * forward has nothing to switch.  Off (the default): the atomic kernels, whose gradients repeat to ~1e-7 relative only.  The
 * results of the two modes are not bit-equal to each other. */
int gw_train_set_deterministic(gw_plan* plan, int32_t on);
/* Device bytes of that workspace now (0 before the first backward with the flag on). */
int64_t gw_train_deterministic_bytes(const gw_plan* plan);
/* High-water mark, in bytes, of the training step's stream-ordered working allocations -- every live tape plus the running step's
 * temporaries -- since a training forward last began while no other tape held memory (0 before the first step).  For one tape at
 * a time: over the last gw_train_forward_tape and the gw_train_backward_tape after it.  It depends on the shapes only, unlike device-wide
 * figures on a shared card. */
int64_t gw_train_peak_bytes(const gw_plan* plan);

/* Multi-GPU loss boundary fused into the forecast's last chain (SURVEY.md 8(e): the one gather of the outputs).  After this call
 * every gw_forward / gw_forward_strided / gw_decoder_forward stores its `out` rows, as the tiles leave the tensor cores, into
 * the gather buffers of every GPU of the job as well:
 *   mode 1  NVLink multicast: deltas_bytes[0] = (multicast alias of the caller's gather buffer) - (its local address); one
 *           multimem.st per value, the NVSwitch replicates it to all GPUs of the multicast group (this GPU included);
 *   mode 2  peer stores: deltas_bytes[j] = (mapping of GPU j's gather buffer in this process) - (local address), n <= 8 entries
 *           (this GPU's own buffer included): one store per GPU and value;
 *   mode 0  off (default).
 * `out` passed to the forward must lie inside the local gather buffer the deltas were taken from.  The caller orders the
 * exchange with its own cross-GPU barrier (graph_weather_b200/dist.py).  Tensor-core precisions only. */
int gw_plan_set_output_peers(gw_plan* plan, int32_t mode, int32_t n, const int64_t* deltas_bytes);

/* Stage entry points (the reference's sub-module API, tests/test_model.py:106-119):
 *   gw_encoder_forward   Encoder.forward   encoder.py:153-242        features -> x [batch*n_mesh, node_dim]
 *   gw_processor_forward Processor.forward processor.py:83-128       x -> x   (in place allowed)
 *   gw_decoder_forward   Decoder.forward   decoder.py:79-94 / AssimilatorDecoder.forward assimilator_decoder.py:131
 *                        x [batch*n_mesh,node_dim] (+ start features [batch,n_out,start_ld], first residual_dim used)
 * Mesh rows are in the encoder/decoder slot order (slot = H-1-rank), as in the reference.                       */
int gw_encoder_forward(gw_plan* plan, const float* features, float* x_out, int32_t batch, void* stream);
int gw_processor_forward(gw_plan* plan, const float* x_in, float* x_out, int32_t batch, void* stream);
int gw_decoder_forward(gw_plan* plan, const float* x_in, const float* start_features, int32_t start_ld, float* out,
                       int32_t batch, void* stream);
/* Processor.forward on a CALLER-SUPPLIED graph (processor.py:83 takes edge_index / edge_attr as arguments):
 * n_nodes x [n_nodes,node_dim], n_edges target-sorted edges (src, dst non-decreasing, ptr[n_nodes+1]) with initial
 * edge features edge_attr [n_edges, edge_dim].  The reference's batch-replicated graph is simply a larger graph;
 * capacity: n_nodes <= max_batch*n_mesh, n_edges <= max_batch*n_lat_edges. */
int gw_processor_forward_graph(gw_plan* plan, const float* x_in, float* x_out, const float* edge_attr, int32_t n_nodes,
                               int32_t n_edges, const int32_t* src, const int32_t* dst, const int32_t* ptr, void* stream);
/* The encoded latent edge features Encoder.forward also returns (encoder.py:235-241), one sample's worth
 * [n_lat_edges, edge_dim] in the plan's target-sorted edge order; copies into caller memory. */
int gw_latent_edge_features(gw_plan* plan, float* edge_attr_out, void* stream);

/* Synchronises `stream` and returns (then clears) the plan's device status word: 0 = ok;
 * bit 0: an activation left the fp16 range in GW_PREC_FP32_TC (results invalid: rerun with GW_PREC_FP32_SIMT);
 * bit 1: internal pipeline timeout; bit 2: shared-memory misalignment; bit 3: a magnitude bound is not finite: the features or
 * a weight matrix hold an inf / NaN (inference also checks every bias and LayerNorm parameter).  The tensor-core precisions,
 * GW_PREC_FP32_TC and GW_PREC_BF16_TC, refuse such inputs this way in inference and in both training steps; GW_PREC_FP32_SIMT
 * never sets it and propagates them as torch does; bit 4: an observation could not be located on the mesh (non-finite coordinates).  Non-zero must be treated as failure.  (Operands are range-scaled from rigorous per-tensor magnitude bounds, so
 * bit 0 is a guard that finite inputs cannot trip.) */
int gw_plan_status(gw_plan* plan, int32_t* status_out, void* stream);
/* Non-blocking read of the same word (it lives in host-mapped memory): reflects every kernel that has COMPLETED so far
 * and does not clear it.  The Python wrappers peek before and after every forward and escalate to gw_plan_status
 * (synchronise, clear, raise) when it is non-zero, so a fault is reported at the latest on the next call. */
int gw_plan_status_peek(gw_plan* plan, int32_t* status_out);
/* Raw copy of the plan's 64-word host-mapped status block (no CUDA call: usable after a device fault):
 * word 0 = status flags; words 4+3w.. = {barrier byte offset, parity, block} of the wait warp w timed out on. */
int gw_plan_debug(gw_plan* plan, int32_t* out64);
/* Debug: the next tensor-core chain launched for kernel class `tag` writes a clock64 event timeline of its CTA 0 into
 * device_buf ([8 roles][1024 events][2] int64, zero-initialised by the caller). */
int gw_debug_trace_next(gw_plan* plan, int32_t tag, int64_t* device_buf);

/* Per-launch device timing for bench.py's live roofline measurement.  When enabled, every kernel this library
 * launches for the plan is bracketed by a cudaEvent pair recorded on the launching stream and attributed to a kernel
 * class ("tag": enc_grid, enc_mesh, proc_p, proc_edge, proc_node, dec_p, dec_edge, dec_node, const).
 * gw_timing_read synchronises `stream`, returns launches[] and summed milliseconds[] per tag (arrays of
 * gw_timing_num_tags() entries) since the previous read, and resets the record. */
int gw_timing_enable(gw_plan* plan, int32_t on);
int32_t gw_timing_num_tags(void);
const char* gw_timing_tag_name(int32_t tag);
int gw_timing_read(gw_plan* plan, int64_t* launches, double* milliseconds, void* stream);

/* Loss boundary (SURVEY 8(f) row 2, forward): NormalizedMSELoss.forward, graph_weather/models/losses.py:46-94.
 *   *sum_out = sum over b < batch, n < n_nodes of  node_weight[n] * mean_f( (pred - target)^2 * inv_variance[f] )
 * pred / target: [batch, n_nodes, n_features] fp32 row-major device pointers; inv_variance: [n_features] (1 / feature_variance,
 * losses.py:70) or NULL when the reference's `normalize` is False; node_weight: [n_nodes] = cos(latitude) tiled as
 * losses.py:83-88.  The reference's value is *sum_out / (batch * n_nodes) (losses.py:94); data-parallel ranks add their sums
 * (one all-reduced scalar) and divide by the global row count.  workspace: gw_loss_workspace_bytes() device bytes.
 * Deterministic (fixed reduction tree), independent of any plan. */
int64_t gw_loss_workspace_bytes(void);
int gw_normalized_mse_loss_sum(const float* pred, const float* target, const float* inv_variance, const float* node_weight,
                               int64_t batch, int64_t n_nodes, int32_t n_features, double* sum_out, void* workspace, void* stream);

/* PhysicalConstraintLayer.forward (graph_weather/models/layers/constraint_layer.py:58-188) as GraphWeatherForecaster applies
 * it (forecast.py:231-246: upsampling_factor 1, one patch = the whole grid), on graph-ordered rows:
 *   hr  [batch, n_nodes, channels]      the decoder output;  lr [batch, n_nodes, lr_ld] its first lr_channels columns are the
 *   low-resolution reference (channel c of hr pairs with channel c % lr_channels: forecast.py:243-245);
 *   src [n_nodes] int32: the row that the reference's graph_to_grid / grid_to_graph round trip leaves at node n
 *   (forecast.py:178-213; the identity for a complete row-major grid);  out [batch, n_nodes, channels].
 * type: GW_CONSTRAINT_ADDITIVE y = hr + lr - mean(hr); _MULTIPLICATIVE y = hr * mean(lr) / (mean(hr) + 1e-8);
 * _SOFTMAX y = exp(f hr) * (lr * (1 / exp(f hr))).  Means run over the nodes, per sample and channel, deterministically.
 * workspace: gw_constraint_workspace_bytes(batch, channels) device bytes. */
#define GW_CONSTRAINT_ADDITIVE 1
#define GW_CONSTRAINT_MULTIPLICATIVE 2
#define GW_CONSTRAINT_SOFTMAX 3
int64_t gw_constraint_workspace_bytes(int64_t batch, int32_t channels);
int gw_constraint_apply(int32_t type, const float* hr, const float* lr, int32_t lr_ld, int32_t lr_channels, const int32_t* src,
                        float* out, int64_t batch, int64_t n_nodes, int32_t channels, float exp_factor, void* workspace, void* stream);
/* Backward of gw_constraint_apply (the reference trains through the layer: forecast.py:231-246 lies inside the forward that
 * loss.backward() walks).  dy [batch, n_nodes, channels] = d loss / d out; hr, lr, lr_ld, src, exp_factor: the forward's inputs.
 *   d_hr [batch, n_nodes, channels]  gradient of hr;  d_lr [batch, n_nodes, channels] (contiguous; NULL: not computed) gradient of
 *   lr's first `channels` columns.  Rows no node reads get 0; a row read by several nodes sums their terms in ascending node order.
 * lr_channels must equal channels.  Additive / multiplicative: column sums in double, fixed order (the multiplicative means are
 * recomputed by the forward's kernels, bit for bit); softmax: torch's autograd of constraint_layer.py:172-187 op by op in fp32.
 * No atomics: repeated calls give identical bits.  workspace: gw_constraint_backward_workspace_bytes(batch, n_nodes, channels). */
int64_t gw_constraint_backward_workspace_bytes(int64_t batch, int64_t n_nodes, int32_t channels);
int gw_constraint_backward(int32_t type, const float* dy, const float* hr, const float* lr, int32_t lr_ld, int32_t lr_channels, const int32_t* src,
                           float* d_hr, float* d_lr, int64_t batch, int64_t n_nodes, int32_t channels, float exp_factor, void* workspace,
                           void* stream);

/* Backward of the loss sum: grad_pred[b, n, f] = (*scale_dev) * scale * node_weight[n] * 2 (pred - target) * inv_variance[f] / n_features.
 * scale_dev (device float, may be NULL = 1) carries the upstream gradient; scale is a host factor (1 / global row count). */
int gw_normalized_mse_loss_grad(const float* pred, const float* target, const float* inv_variance, const float* node_weight, int64_t batch,
                                int64_t n_nodes, int32_t n_features, const float* scale_dev, float scale, float* grad_pred, void* stream);

/* Counters for bench.py: kernels launched by this library on the calling thread since the last reset. */
int64_t gw_launch_count(void);
void gw_launch_count_reset(void);

#ifdef __cplusplus
}
#endif
#endif /* GW_B200_H */
