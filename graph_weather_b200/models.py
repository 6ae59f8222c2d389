"""Drop-in host-side mirror of the reference's module API for the encode-process-decode path.

Same class names, constructor arguments, attribute names and state_dict keys as
    graph_weather/models/forecast.py:61-247           GraphWeatherForecaster
    graph_weather/models/analysis.py:52-150           GraphWeatherAssimilator
    graph_weather/models/layers/encoder.py:36-268     Encoder
    graph_weather/models/layers/processor.py:17-128   Processor
    graph_weather/models/layers/decoder.py:24-94      Decoder
    graph_weather/models/layers/assimilator_{encoder,decoder}.py
    graph_weather/models/layers/graph_net_block.py    MLP / EdgeProcessor / NodeProcessor / GraphProcessor
so `load_state_dict` / `from_pretrained` round-trip with the reference, and sub-modules are constructed in the
reference's order so that `torch.manual_seed(s)` gives the same initial weights.

These modules hold parameters and graphs only.  Every forward goes through libgwb200.so (graph_weather_b200._capi);
there is no eager-PyTorch or CPU execution path -- CPU tensors raise.
"""

from __future__ import annotations

import contextlib
import os
import weakref
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
from torch import nn

from . import _capi, graphs, h3lite
from .constraint import GridMapping, PhysicalConstraintLayer

try:  # the reference mixes this into both wrappers (forecast.py:61, analysis.py:52)
    from huggingface_hub import PyTorchModelHubMixin
except Exception:  # pragma: no cover

    class PyTorchModelHubMixin:  # type: ignore
        pass


def _no_host_path(what):
    raise RuntimeError(
        f"{what}: graph_weather_b200 executes only through its CUDA library on a CUDA device; "
        "there is no CPU / eager fallback. Move the module and inputs to the GPU."
    )


# ---------------------------------------------------------------------------------------------------------------
# parameter containers (graph_net_block.py)
# ---------------------------------------------------------------------------------------------------------------
class MLP(nn.Module):
    """Parameter container with the reference layout (graph_net_block.py:45-61): `model.{0,2,..}` Linear, last index LayerNorm."""

    def __init__(self, in_dim, out_dim=128, hidden_dim=128, hidden_layers=2, norm_type: Optional[str] = "LayerNorm",
                 use_checkpointing: bool = False):  # fmt: skip
        super().__init__()
        self.use_checkpointing = use_checkpointing
        layers = [nn.Linear(in_dim, hidden_dim), nn.ReLU()]
        for _ in range(hidden_layers - 1):
            layers += [nn.Linear(hidden_dim, hidden_dim), nn.ReLU()]
        layers.append(nn.Linear(hidden_dim, out_dim))
        if norm_type is not None:
            assert norm_type in ["LayerNorm", "GraphNorm", "InstanceNorm", "BatchNorm", "MessageNorm"]
            if norm_type != "LayerNorm":  # only LayerNorm resolves in the reference too (getattr(nn, ...), :58)
                raise NotImplementedError(f"norm_type={norm_type!r}: only 'LayerNorm' is supported on the CUDA path")
            layers.append(nn.LayerNorm(out_dim))
        self.model = nn.Sequential(*layers)
        self.in_dim, self.out_dim, self.hidden_dim, self.hidden_layers = in_dim, out_dim, hidden_dim, hidden_layers

    def forward(self, x):
        _no_host_path("MLP.forward")


class EdgeProcessor(nn.Module):
    def __init__(self, in_dim_node=128, in_dim_edge=128, hidden_dim=128, hidden_layers=2, norm_type="LayerNorm"):
        super().__init__()
        self.edge_mlp = MLP(2 * in_dim_node + in_dim_edge, in_dim_edge, hidden_dim, hidden_layers, norm_type)


class NodeProcessor(nn.Module):
    def __init__(self, in_dim_node=128, in_dim_edge=128, hidden_dim=128, hidden_layers=2, norm_type="LayerNorm"):
        super().__init__()
        self.node_mlp = MLP(in_dim_node + in_dim_edge, in_dim_node, hidden_dim, hidden_layers, norm_type)


class _MetaBlock(nn.Module):
    """Stands where the reference puts torch_geometric.nn.MetaLayer (graph_net_block.py:221-228): same child names."""

    def __init__(self, edge_model, node_model):
        super().__init__()
        self.edge_model = edge_model
        self.node_model = node_model


class GraphProcessor(nn.Module):
    def __init__(self, mp_iterations=15, in_dim_node=128, in_dim_edge=128, hidden_dim_node=128, hidden_dim_edge=128,
                 hidden_layers_node=2, hidden_layers_edge=2, norm_type="LayerNorm", use_checkpointing=False):  # fmt: skip
        super().__init__()
        if norm_type != "LayerNorm":
            raise NotImplementedError("the CUDA message-passing kernels implement LayerNorm MLPs (the reference default)")
        self.use_checkpointing = use_checkpointing
        self.blocks = nn.ModuleList()
        for _ in range(mp_iterations):
            self.blocks.append(
                _MetaBlock(
                    EdgeProcessor(in_dim_node, in_dim_edge, hidden_dim_edge, hidden_layers_edge, norm_type),
                    NodeProcessor(in_dim_node, in_dim_edge, hidden_dim_node, hidden_layers_node, norm_type),
                )
            )


# ---------------------------------------------------------------------------------------------------------------
# engine: one gw_plan + upload bookkeeping
# ---------------------------------------------------------------------------------------------------------------
def _params_fingerprint(named):
    return tuple((k, v.data_ptr(), v._version, tuple(v.shape)) for k, v in named)


def _tc_eligible(dims: dict) -> bool:
    """The tensor-core chains are built for the reference's default sizes: 256-wide node / edge / hidden, 2 hidden layers."""
    return (dims.get("node_dim") == 256 and dims.get("edge_dim") == 256 and dims.get("hidden_node") == 256
            and dims.get("hidden_edge") == 256 and dims.get("hidden_layers_node") == 2 and dims.get("hidden_layers_edge") == 2)  # fmt: skip


def _tc_layered(dims: dict) -> bool:
    """A trunk the tensor cores run layer by layer: every node / edge / hidden width at least 256 and one above 256 (train/run.py's
    1024-wide model), any number of hidden layers."""
    w = [dims.get(k, 0) for k in ("node_dim", "edge_dim", "hidden_node", "hidden_edge")]
    return min(w) >= 256 and max(w) > 256


def _validate_precision(precision: str, dims: dict):
    """Constructor-time check, so that an impossible request fails where the module is built, not at the first forward."""
    if precision not in ("auto",) + tuple(_capi.PRECISIONS):
        raise ValueError(f"precision={precision!r}: expected one of 'auto', {sorted(_capi.PRECISIONS)}")
    if precision in ("fp32", "fp32_tc", "bf16") and not (_tc_eligible(dims) or _tc_layered(dims)):
        raise ValueError(
            f"precision={precision!r} runs the tensor cores: the fused chains need node/edge/hidden dims of 256 and 2 hidden layers "
            "(the reference defaults), the layer-by-layer forward a trunk at least 256 wide with one width above 256; use "
            "precision='auto' (CUDA-core exact fp32 for other sizes) or 'fp32_simt'"
        )


TRAIN_PRECISIONS = ("fp32_simt", "fp32", "bf16")


def _validate_train_precision(train_precision: str, dims: dict):
    """`train_precision` of GraphWeatherForecaster, GraphCast and GraphWeatherAssimilator: the arithmetic of the training step (gw_train.cu).  'fp32_simt' exact fp32 on
    CUDA cores; 'fp32' fp16 hi/lo split on tensor cores (3 MMAs per product, fp32 accumulation); 'bf16' bf16 tensor-core
    operands (fp32 accumulation, fp32 master weights, gradients and tape)."""
    if train_precision not in TRAIN_PRECISIONS:
        raise ValueError(f"train_precision={train_precision!r}: expected one of {list(TRAIN_PRECISIONS)}")
    if train_precision != "fp32_simt" and not _tc_eligible(dims):
        raise ValueError(
            f"train_precision={train_precision!r} runs the tensor-core chains, which are built for node/edge/hidden dims of 256 and 2 "
            "hidden layers (the reference defaults); use train_precision='fp32_simt' for other sizes"
        )


def resolve_precision(precision: str, dims: dict, device) -> str:
    """'auto' (the default of every constructor): the fp32-faithful tensor-core (wgmma) path wherever it applies -- reference
    default sizes on an sm_90 device (H100) -- and the exact-fp32 CUDA-core path otherwise.  Explicit values are returned unchanged."""
    if precision != "auto":
        return precision
    if _tc_eligible(dims) and torch.cuda.get_device_capability(device) == (9, 0):
        return "fp32"
    return "fp32_simt"


class _Engine:
    """Creates the plan lazily on the device of the first input, uploads graphs once and weights whenever a parameter
    changed (in-place optimiser steps and load_state_dict bump tensor versions; .to() changes data pointers)."""

    def __init__(self, dims: dict, precision: str, train_only: bool = False):
        _validate_precision(precision, dims)
        self.dims = dict(dims)
        self.precision = precision
        self.train_only = train_only  # training-only plans (gw_plan_create_train): the bounded-memory training step
        self.resolved_precision: Optional[str] = None
        self.plan: Optional[_capi.Plan] = None
        self.graph_uploaders = []  # callables(plan)
        self.generation = 0  # bumped whenever a new plan is created: per-plan upload caches key on it, never on pointers
        self.obs_key = None  # the host-built observation graph the plan holds (AssimilatorEncoder._upload_obs)
        self.last_tape = None  # tape of the last training forward made outside multi_step(): the next one closes it (_TrainFn)
        self._wfp = None

    def _create(self, device, max_batch):
        if self.plan is not None:
            self.plan.close()
        d = dict(self.dims)
        d["max_batch"] = int(max_batch)
        self.resolved_precision = resolve_precision(self.precision, self.dims, device)
        d["precision"] = _capi.PRECISIONS[self.resolved_precision]
        self.plan = _capi.Plan(device, train_only=self.train_only, **d)
        self.generation += 1
        for up in self.graph_uploaders:
            up(self.plan)
        self._wfp = None

    def ensure(self, device, batch, named_params, grow: Optional[dict] = None):
        device = torch.device(device)
        if device.type != "cuda":
            _no_host_path("forward on a CPU tensor")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        need_new = self.plan is None or self.plan.device != device
        if grow:
            for k, v in grow.items():
                if v > self.dims.get(k, 0):
                    self.dims[k] = int(v)
                    need_new = True
        if not need_new and batch > self.plan.dims.max_batch:
            need_new = True
        if not need_new and self.plan.peek():
            self.plan.status()  # a kernel of an earlier call flagged a fault: synchronise, clear and raise now
        if need_new:
            self._create(device, max(batch, self.plan.dims.max_batch if self.plan is not None else 1))
        named = list(named_params)
        fp = _params_fingerprint(named)
        if fp != self._wfp:
            self.plan.set_weights(named)
            self._wfp = fp
        return self.plan

    def invalidate_weights(self):
        self._wfp = None


def _new_engine(dims: dict, precision: str, uploaders, train_only: bool = False) -> _Engine:
    eng = _Engine(dims, precision, train_only)
    eng.graph_uploaders += uploaders
    return eng


def _own_engine(module, dims=None) -> _Engine:
    """The engine of an Encoder, AssimilatorEncoder or decoder called on its own (created on first use)."""
    if module._engine is None:
        module._engine = _new_engine(module._dims if dims is None else dims, module._precision, [module._upload_graphs])
    return module._engine


def _maybe_check(plan):
    """Every forward ends with a non-blocking look at the plan's host-mapped status word; a non-zero word (fp16-range
    overflow, pipeline timeout, misalignment: include/gw_b200.h) escalates to the synchronising `plan.status()`, which
    raises.  Kernels still running when this returns are covered by the same look at the start of the next call
    (`_Engine.ensure`).  GW_B200_CHECK=1 synchronises after every forward (tests, debugging)."""
    if os.environ.get("GW_B200_CHECK", "0") == "1" or plan.peek():
        plan.status()


class _TrainFn(torch.autograd.Function):
    """autograd node of one training forward of a wrapper (GraphWeatherForecaster, GraphCast, GraphWeatherAssimilator,
    RegionalForecaster): forward = gw_train_forward_tape (activations kept on a tape, `_capi.Tape`), backward =
    gw_train_backward_tape (gradients of every bound parameter, and of the features when they require grad).  One backward per
    forward.  Every forward makes a tape that this node owns: its backward consumes it, and dropping the graph without a backward
    frees it.  Outside `multi_step()` a forward first closes the tape of the previous forward made outside a window
    (`_Engine.last_tape`), which replaces that forward's activations; inside it, a forward closes nothing.

    The wrapper supplies its training engine (`_training_engine()`), the tensors the plan uploads (`_named()`), its output shape
    (`_out_shape(batch)`) and `bindings`: what the step differentiates, one (name the plan binds, tensor uploaded under that name,
    parameter, gradient map) per entry of `params` (`_grad_bindings()`).  The step returns each gradient shaped like the uploaded
    tensor; the map turns it into the parameter's gradient (None: it is the parameter's already).  `obs` (the assimilator's
    lat_lon_heights, else None) is built into the training plan's observation graph for this call, as inference builds it for
    every call.  Under torch.use_deterministic_algorithms(True), read when the backward runs, the backward sums every parameter
    gradient in a fixed order (gw_train_set_deterministic): the same inputs and weights give the same gradients bit for bit."""

    @staticmethod
    def forward(ctx, model, features, obs, bindings, *params):
        B = features.shape[0]
        eng = model._training_engine()
        plan = eng.ensure(features.device, B, model._named(), grow=None if obs is None else dict(n_in=obs.shape[0]))
        if obs is not None:
            model.encoder._upload_obs(eng, plan, obs)
        f = features.detach().to(torch.float32).contiguous()
        out = torch.empty(model._out_shape(B), dtype=torch.float32, device=f.device)
        in_window = bool(model.__dict__.get("_multi_step", 0))
        if not in_window and eng.last_tape is not None:
            eng.last_tape.close()  # stream-ordered, ahead of this forward's allocations
            eng.last_tape = None
        plan.set_processor_segments(model._processor_segments())
        tape = plan.tape()
        try:
            tape.forward(f, out)
            _maybe_check(plan)
        except BaseException:
            tape.close()  # a refused forward leaves no tape
            raise
        if not in_window:
            eng.last_tape = tape
        tape.node = weakref.ref(ctx)  # alive while the graph that will run this backward is (`_pending_tape`)
        ctx.tape = tape
        ctx.model, ctx.plan, ctx.eng = model, plan, eng
        ctx.feat_shape, ctx.feat_grad = tuple(f.shape), bool(features.requires_grad)
        ctx.names = [name for name, _, _, _ in bindings]
        ctx.pshapes = [tuple(bound.shape) for _, bound, _, _ in bindings]
        ctx.maps = [to_param for _, _, _, to_param in bindings]
        ctx.pgrad = [bool(q.requires_grad) for q in params]
        ctx.keep = f  # the tape reads the features again in the backward (weight gradient of the first Linear)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if ctx.tape is None or not ctx.tape.handle.value:
            raise RuntimeError("graph_weather_b200: backward of a forward whose activations were consumed by an earlier backward or "
                               "replaced by a later training forward outside multi_step() (one backward per forward)")
        if ctx.eng.plan is not ctx.plan:
            raise RuntimeError("graph_weather_b200: backward of a forward whose plan was replaced (a switch of the training step, a "
                               "larger batch or .to()): its activations are gone (one backward per forward)")
        dev = grad_out.device
        g = grad_out.detach().to(torch.float32).contiguous()
        gfeat = torch.empty(ctx.feat_shape, dtype=torch.float32, device=dev) if ctx.feat_grad else None
        grads = [torch.empty(s, dtype=torch.float32, device=dev) for s in ctx.pshapes]
        ctx.plan.set_deterministic(torch.are_deterministic_algorithms_enabled())  # (its value when the backward runs counts)
        try:
            ctx.tape.backward(g, gfeat, list(zip(ctx.names, grads)))
        finally:  # consumed, or refused (weights replaced, plan closed): either way the tape is done
            ctx.tape.close()
            ctx.tape = None
        _maybe_check(ctx.plan)
        return (None, gfeat, None, None) + tuple((gr if to_param is None else to_param(gr)) if need else None
                                                 for gr, to_param, need in zip(grads, ctx.maps, ctx.pgrad))


class _Stage:
    """What `_StageFn` runs for one training forward of a standalone sub-module: its training engine and plan, the parameters it
    differentiates (bound names and shapes), and the sub-module's two calls on a tape -- forward(tape, *inputs) -> outputs and
    backward(tape, grad_outputs, named_grads) -> the inputs' gradients."""

    def __init__(self, eng, plan, named_params, forward, backward):
        self.eng, self.plan = eng, plan
        self.names = [k for k, _ in named_params]
        self.shapes = [tuple(q.shape) for _, q in named_params]
        self.forward, self.backward = forward, backward


class _StageFn(torch.autograd.Function):
    """autograd node of one training forward of a standalone Encoder, AssimilatorEncoder, Processor, Decoder or AssimilatorDecoder:
    forward = the stage's gw_train_*_forward_tape on a tape of its own, backward = its gw_train_*_backward_tape (gradients of the
    stage's inputs and of every parameter).  The node owns its tape until the backward consumes it or the graph is dropped (which
    frees it): the semantics of `multi_step()` without the window, so a stage applied twice in one graph back-propagates through
    both calls.  One backward per forward.  The first `n_in` tensors are the stage's inputs (the tape reads them again in the
    backward, so the node keeps them), the rest its parameters.  The backward follows torch.use_deterministic_algorithms as
    _TrainFn's does."""

    @staticmethod
    def forward(ctx, stage, n_in, *tensors):
        inputs = tuple(t.detach() for t in tensors[:n_in])
        tape = stage.plan.tape()
        try:
            outs = stage.forward(tape, *inputs)
            _maybe_check(stage.plan)
        except BaseException:
            tape.close()  # a refused forward leaves no tape
            raise
        tape.node = weakref.ref(ctx)  # alive while the graph that will run this backward is (`_pending_tape`)
        ctx.tape, ctx.stage, ctx.n_in, ctx.keep = tape, stage, n_in, inputs
        return outs

    @staticmethod
    def backward(ctx, *grad_outs):
        stage = ctx.stage
        if ctx.tape is None or not ctx.tape.handle.value:
            raise RuntimeError("graph_weather_b200: backward of a sub-module's training forward whose activations were consumed by an "
                               "earlier backward (one backward per forward)")
        if stage.eng.plan is not stage.plan:
            raise RuntimeError("graph_weather_b200: backward of a sub-module's training forward whose plan was replaced (a switch of the "
                               "training step, a larger batch or graph, or .to()): its activations are gone (one backward per forward)")
        g = [x.detach().to(torch.float32).contiguous() for x in grad_outs]
        grads = [torch.empty(s, dtype=torch.float32, device=g[0].device) for s in stage.shapes]
        stage.plan.set_deterministic(torch.are_deterministic_algorithms_enabled())
        try:
            gin = stage.backward(ctx.tape, g, list(zip(stage.names, grads)))
        finally:  # consumed, or refused: either way the tape is done
            ctx.tape.close()
            ctx.tape = None
        _maybe_check(stage.plan)
        need = ctx.needs_input_grad[2:]
        return (None, None) + tuple(gr if nd else None for gr, nd in zip(tuple(gin) + tuple(grads), need))


def _stage_wants_grad(module, *inputs):
    """A sub-module built with a `train_precision` takes its training step in train mode with autograd on and something to
    differentiate (an input or a parameter); without one it stays inference-only."""
    return (module.train_precision is not None and torch.is_grad_enabled() and module.training
            and (any(t is not None and t.requires_grad for t in inputs) or any(q.requires_grad for q in module.parameters())))  # fmt: skip


def _stage_engine(module, dims, uploaders, bounded=False) -> _Engine:
    """The training engine of a standalone sub-module, of precision `train_precision`; its inference engine stays as it is.
    `bounded` (the Encoder's and decoders' use_checkpointing, read at every training forward) selects the step as a wrapper's
    `_bounded_step()` does: a training-only plan whose step keeps only the mesh-sized activations and recomputes the lat/lon side
    chunk by chunk in the backward, or the taped step (the default).  One engine per step, each created on first use; switching
    closes the other's plan (`_switch_training_engine`).  The chosen engine is `module._train_engine`."""
    def make(b):
        return _new_engine(dims, module.train_precision, uploaders, train_only=b)

    eng = _switch_training_engine(module.__dict__.setdefault("_train_engines", {}), bool(bounded), make)
    module.__dict__["_train_engine"] = eng
    return eng


def _run_stage(eng, plan, prefix, module, inputs, forward, backward):
    """One training forward of `module` through `_StageFn`, differentiating its inputs and every parameter (bound as `prefix.name`)."""
    named = [(f"{prefix}.{k}", q) for k, q in module.named_parameters()]
    stage = _Stage(eng, plan, named, forward, backward)
    return _StageFn.apply(stage, len(inputs), *inputs, *[q for _, q in named])


def _check_train_precision(train_precision, dims):
    """`train_precision` of a sub-module: None (the default) keeps it inference-only; a value is checked as for the wrappers."""
    if train_precision is not None:
        _validate_train_precision(train_precision, dims)


def _pending_tape(engine) -> bool:
    """The engine's plan holds a tape that a backward still needs: made by a forward whose backward has not run, and whose autograd
    graph is still alive (a dropped graph's tape is only waiting to be closed)."""
    plan = engine.plan
    return plan is not None and any(getattr(t, "node", None) is not None and t.node() is not None for t in plan.live_tapes())


def _switch_training_engine(engines: dict, bounded: bool, make) -> _Engine:
    """engines[bounded], created by make(bounded) on first use; the other step's engine gives up its plan (see
    `_Wrapper._training_engine`)."""
    if bounded not in engines:
        engines[bounded] = make(bounded)
    other = engines.get(not bounded)
    if other is not None and other.plan is not None:
        other.plan.close()
        other.plan = None
    return engines[bounded]


def _wants_grad(model, features):
    """A wrapper's forward takes the training step in train mode with autograd on and something to differentiate."""
    return torch.is_grad_enabled() and model.training and (features.requires_grad or any(q.requires_grad for q in model.parameters()))


def _check_segments(segments):
    """A processor segment count is -1 (the whole processor), 0 (none) or a number of blocks: refused where it is set, not at the next
    training forward."""
    if segments < -1:
        raise ValueError(f"checkpoint segments must be -1 (the whole processor), 0 (none) or a positive number of blocks, got {segments}")


def _prefixed(prefix, module):
    return [(f"{prefix}.{k}", v) for k, v in module.state_dict(keep_vars=True).items() if torch.is_tensor(v)]


def _latlon_list(lat_lons):
    return [(float(p[0]), float(p[1])) for p in lat_lons]


# ---------------------------------------------------------------------------------------------------------------
# Encoder (encoder.py)
# ---------------------------------------------------------------------------------------------------------------
class Encoder(nn.Module):
    def __init__(self, lat_lons: list, resolution: int = 2, input_dim: int = 78, output_dim: int = 256, output_edge_dim: int = 256,
                 hidden_dim_processor_node=256, hidden_dim_processor_edge=256, hidden_layers_processor_node=2,
                 hidden_layers_processor_edge=2, mlp_norm_type="LayerNorm", use_checkpointing: bool = False,
                 efficient_batching: bool = False, precision: str = "auto", train_precision: Optional[str] = None):  # fmt: skip
        """encoder.py:36-151.  train_precision=None (the default) keeps the module inference-only: its output has no autograd graph.
        'fp32_simt' | 'fp32' | 'bf16' (as for GraphWeatherForecaster) make a train-mode call with autograd on run the encoder's
        training step, so that `x` and `edge_attr` carry gradients to the features and every parameter.  use_checkpointing, read
        at every training forward, selects the step as for GraphWeatherForecaster: False (the default) the taped step, True the
        bounded-memory step, which keeps only the mesh-sized activations and recomputes the lat/lon side chunk by chunk in the
        backward (the 0.25 degree grid trains on one 80 GB card)."""
        super().__init__()
        self.use_checkpointing = use_checkpointing  # with a train_precision: the bounded-memory training step (_stage_engine)
        self.efficient_batching = efficient_batching
        self.output_dim = output_dim
        self.num_latlons = len(lat_lons)
        self.resolution = resolution
        self._g_enc = graphs.build_encoder_graph(lat_lons, resolution)
        self._g_lat = graphs.build_mesh_graph(resolution)
        self.num_h3 = self._g_lat.num_h3
        self.h3_nodes = nn.Parameter(torch.zeros((h3lite.get_num_cells(resolution), input_dim), dtype=torch.float))
        self.node_encoder = MLP(input_dim, output_dim, hidden_dim_processor_node, hidden_layers_processor_node, mlp_norm_type)
        self.edge_encoder = MLP(2, output_edge_dim, hidden_dim_processor_edge, hidden_layers_processor_edge, mlp_norm_type)
        self.latent_edge_encoder = MLP(2, output_edge_dim, hidden_dim_processor_edge, hidden_layers_processor_edge, mlp_norm_type)
        self.graph_processor = GraphProcessor(1, output_dim, output_edge_dim, hidden_dim_processor_node, hidden_dim_processor_edge,
                                              hidden_layers_processor_node, hidden_layers_processor_edge, mlp_norm_type)  # fmt: skip
        self._dims = dict(
            n_in=self.num_latlons, n_out=0, n_mesh=self.num_h3, n_lat_edges=self._g_lat.edge_index.shape[1], n_dec_edges=0,
            in_dim=input_dim, enc_edge_attr_dim=2, out_dim=1, residual_dim=0, node_dim=output_dim, edge_dim=output_edge_dim,
            hidden_node=hidden_dim_processor_node, hidden_edge=hidden_dim_processor_edge,
            hidden_layers_node=hidden_layers_processor_node, hidden_layers_edge=hidden_layers_processor_edge,
            hidden_dec=1, hidden_layers_dec=1, num_blocks=1,
        )  # fmt: skip
        self._engine = None
        _validate_precision(precision, self._dims)
        self._precision = precision
        _check_train_precision(train_precision, self._dims)
        self.train_precision = train_precision
        self._lat_edge_index_t = {}

    # graph uploads shared with the wrappers
    def _upload_graphs(self, plan):
        g, m = self._g_enc, self._g_lat
        plan.set_encoder_graph(g.mesh_local, g.perm, g.ptr, g.edge_attr)
        plan.set_latent_graph(m.src, m.dst, m.ptr, m.edge_attr[m.perm])

    def _latent_edge_index(self, batch, device):
        """edge_index [2,B*El] int64 in the reference's order and replication (encoder.py:224-242)."""
        m = self._g_lat
        key = (str(device), batch)
        if key not in self._lat_edge_index_t:
            ei = graphs.replicate_edge_index(m.edge_index, batch) if not self.efficient_batching else m.edge_index
            self._lat_edge_index_t = {key: torch.from_numpy(ei).to(device)}
        return self._lat_edge_index_t[key]

    def _latent_outputs(self, plan, batch, device):
        """(edge_index [2,B*El] int64, edge_attr [B*El,De]) in the reference's order and replication (encoder.py:224-242)."""
        m = self._g_lat
        El = m.edge_index.shape[1]
        ei = self._latent_edge_index(batch, device)
        sorted_attr = torch.empty((El, self._dims["edge_dim"]), dtype=torch.float32, device=device)
        plan.latent_edge_features(sorted_attr)
        ref_attr = torch.empty_like(sorted_attr)
        ref_attr[torch.from_numpy(m.perm).to(device)] = sorted_attr
        if not self.efficient_batching:
            ref_attr = ref_attr.repeat(batch, 1)
        return ei, ref_attr

    def _train_encode(self, features, lat_lon_heights):
        """The training step of Encoder.forward / AssimilatorEncoder.forward (`_StageFn`): x [B*H, Dn] and edge_attr as in inference,
        both differentiable.  edge_attr is formed from the sorted latent edge features by torch ops (the inverse of the plan's
        edge order, then one copy per sample), so autograd sums the copies' gradients.  lat_lon_heights gets no gradient."""
        B = features.shape[0]
        eng = _stage_engine(self, self._dims, [self._upload_graphs], self.use_checkpointing)
        grow = None if lat_lon_heights is None else dict(n_in=lat_lon_heights.shape[0])
        plan = eng.ensure(features.device, B, _prefixed("encoder", self), grow=grow)
        if lat_lon_heights is not None:
            self._upload_obs(eng, plan, lat_lon_heights)
        m = self._g_lat
        El, f_shape = m.edge_index.shape[1], tuple(features.shape)

        def forward(tape, f):
            x = torch.empty((B * self.num_h3, self.output_dim), dtype=torch.float32, device=f.device)
            e = torch.empty((El, self._dims["edge_dim"]), dtype=torch.float32, device=f.device)
            tape.encoder_forward(f, x, e)
            return x, e

        def backward(tape, g, named):
            gf = torch.empty(f_shape, dtype=torch.float32, device=g[0].device)
            tape.encoder_backward(g[0], g[1], gf, named)
            return (gf,)

        f = features.to(torch.float32).contiguous()
        x, sorted_attr = _run_stage(eng, plan, "encoder", self, (f,), forward, backward)
        inv = torch.from_numpy(np.argsort(m.perm)).to(f.device)  # ref_attr[perm] = sorted_attr, as a gather autograd can reverse
        ref_attr = sorted_attr[inv]
        if not self.efficient_batching:
            ref_attr = ref_attr.repeat(B, 1)
        return x, self._latent_edge_index(B, f.device), ref_attr

    def _encode(self, features, what, lat_lon_heights=None):
        """Encoder.forward and AssimilatorEncoder.forward; the assimilator's observation graph is uploaded for every call."""
        if features.device.type != "cuda":
            _no_host_path(what)
        if _stage_wants_grad(self, features):
            return self._train_encode(features, lat_lon_heights)
        B = features.shape[0]
        eng = _own_engine(self)
        if lat_lon_heights is None:
            plan = eng.ensure(features.device, B, _prefixed("encoder", self))
        else:
            plan = eng.ensure(features.device, B, _prefixed("encoder", self), grow=dict(n_in=lat_lon_heights.shape[0]))
            self._upload_obs(eng, plan, lat_lon_heights)
        f = features.detach().to(torch.float32).contiguous()
        x = torch.empty((B * self.num_h3, self.output_dim), dtype=torch.float32, device=f.device)
        plan.encoder_forward(f, x)
        _maybe_check(plan)
        ei, ea = self._latent_outputs(plan, B, f.device)
        return x, ei, ea

    def forward(self, features: torch.Tensor):
        return self._encode(features, "Encoder.forward")


# ---------------------------------------------------------------------------------------------------------------
# Processor (processor.py)
# ---------------------------------------------------------------------------------------------------------------
class Processor(nn.Module):
    def __init__(self, input_dim: int = 256, edge_dim: int = 256, num_blocks: int = 9, hidden_dim_processor_node: int = 256,
                 hidden_dim_processor_edge: int = 256, hidden_layers_processor_node: int = 2, hidden_layers_processor_edge: int = 2,
                 mlp_norm_type: str = "LayerNorm", use_thermalizer: bool = False, use_checkpointing: bool = False,
                 precision: str = "auto", train_precision: Optional[str] = None):  # fmt: skip
        """processor.py:17-68.  train_precision=None (the default) keeps the module inference-only.  'fp32_simt' | 'fp32' | 'bf16'
        make a train-mode call with autograd on run the processor's training step on the call's graph: `x`, `edge_attr` (in the
        caller's edge order) and every parameter get gradients, with `checkpoint_segments` read at every call.  Each call keeps its
        own tape, so a processor applied several times in one graph back-propagates through every call.  The processor has no
        grid-sized work: it always takes the taped step, and `set_checkpoint_segments` bounds its memory (use_checkpointing is
        passed on to the GraphProcessor, as in the reference)."""
        super().__init__()
        if use_thermalizer:
            raise NotImplementedError("use_thermalizer=True: the stochastic ThermalizerLayer is outside the accelerated path")
        self.input_dim = input_dim
        self.use_thermalizer = use_thermalizer
        self.checkpoint_segments = 0
        self.graph_processor = GraphProcessor(num_blocks, input_dim, edge_dim, hidden_dim_processor_node, hidden_dim_processor_edge,
                                              hidden_layers_processor_node, hidden_layers_processor_edge, mlp_norm_type,
                                              use_checkpointing)  # fmt: skip
        self._cfg = dict(node_dim=input_dim, edge_dim=edge_dim, hidden_node=hidden_dim_processor_node,
                         hidden_edge=hidden_dim_processor_edge, hidden_layers_node=hidden_layers_processor_node,
                         hidden_layers_edge=hidden_layers_processor_edge, num_blocks=num_blocks)  # fmt: skip
        _validate_precision(precision, self._cfg)
        self._precision = precision
        _check_train_precision(train_precision, self._cfg)
        self.train_precision = train_precision
        self._engine = None

    def set_checkpoint_segments(self, checkpoint_segments: int):
        """processor.py:70-81.  The training step of the wrapper this processor belongs to, or of this processor alone (a
        `train_precision`), recomputes the processor in its backward:
        0 (the default) keeps the processor's whole tape; N > 0 recomputes segments of N blocks, keeping only each segment's first
        node and edge rows; -1 recomputes the whole processor as one segment.  Outputs and gradients do not change, only the memory a
        training forward keeps and the time of its backward (gw_train_set_processor_segments).  Read at every training forward."""
        _check_segments(checkpoint_segments)
        self.checkpoint_segments = checkpoint_segments

    def _sorted_graph(self, edge_index, n_nodes):
        """Target-sorted int32 view of a caller-supplied graph.  Rebuilt on every call, as the reference re-reads its
        edge_index argument every call (processor.py:83-128): a cache keyed on the tensor's address would go stale when the
        allocator recycles it.  No host synchronisation: sort + searchsorted on the device."""
        dst_sorted, order = torch.sort(edge_index[1], stable=True)
        src = edge_index[0][order].to(torch.int32).contiguous()
        ptr = torch.searchsorted(dst_sorted, torch.arange(n_nodes + 1, device=edge_index.device, dtype=dst_sorted.dtype)).to(torch.int32)
        return src, dst_sorted.to(torch.int32).contiguous(), ptr.contiguous(), order

    def _plan_dims(self, n_nodes, n_edges):
        return dict(n_in=0, n_out=0, n_mesh=n_nodes, n_lat_edges=n_edges, n_dec_edges=0, in_dim=1, enc_edge_attr_dim=2, out_dim=1,
                    residual_dim=0, hidden_dec=1, hidden_layers_dec=1, **self._cfg)  # fmt: skip

    def forward(self, x: torch.Tensor, edge_index, edge_attr, t: int = 0, batch_size: int = None, efficient_batching: bool = False):
        if x.device.type != "cuda":
            _no_host_path("Processor.forward")
        train = _stage_wants_grad(self, x, edge_attr)
        x = x.to(torch.float32).contiguous() if train else x.detach().to(torch.float32).contiguous()
        n_nodes = x.shape[0]
        if efficient_batching and batch_size is not None and batch_size > 1:
            # shared graph, per-sample loop in the reference (processor.py:106-122) == block-diagonal replication
            per = n_nodes // batch_size
            edge_index = torch.cat([edge_index + i * per for i in range(batch_size)], dim=1)
            edge_attr = edge_attr.repeat(batch_size, 1)
        src, dst, ptr, order = self._sorted_graph(edge_index, n_nodes)
        if train:
            return self._train_forward(x, edge_attr.to(torch.float32)[order].contiguous(), src, dst, ptr)
        ea = edge_attr.detach().to(torch.float32)[order].contiguous()
        if self._engine is None:
            self._engine = _Engine(self._plan_dims(n_nodes, int(src.numel())), self._precision)
        plan = self._engine.ensure(x.device, 1, _prefixed("processor", self), grow=dict(n_mesh=n_nodes, n_lat_edges=int(src.numel())))
        out = torch.empty_like(x)
        plan.processor_forward_graph(x, out, ea, src, dst, ptr)
        _maybe_check(plan)
        return out

    def _train_forward(self, x, ea, src, dst, ptr):
        """The training step of Processor.forward (`_StageFn`) on the target-sorted graph; ea is edge_attr in that order, gathered by
        a torch op so that autograd returns its gradient in the caller's order."""
        n_nodes, n_edges = x.shape[0], int(src.numel())
        eng = _stage_engine(self, self._plan_dims(n_nodes, n_edges), [])
        plan = eng.ensure(x.device, 1, _prefixed("processor", self), grow=dict(n_mesh=n_nodes, n_lat_edges=n_edges))
        plan.set_processor_segments(self.checkpoint_segments)
        x_shape, e_shape = tuple(x.shape), tuple(ea.shape)

        def forward(tape, xi, e):
            out = torch.empty_like(xi)
            tape.processor_forward(xi, out, e, src, dst, ptr)
            return out

        def backward(tape, g, named):
            gx = torch.empty(x_shape, dtype=torch.float32, device=g[0].device)
            ge = torch.empty(e_shape, dtype=torch.float32, device=g[0].device)
            tape.processor_backward(g[0], gx, ge, named)
            return gx, ge

        return _run_stage(eng, plan, "processor", self, (x, ea), forward, backward)


# ---------------------------------------------------------------------------------------------------------------
# Decoders (assimilator_decoder.py, decoder.py)
# ---------------------------------------------------------------------------------------------------------------
class AssimilatorDecoder(nn.Module):
    def __init__(self, lat_lons: list, resolution: int = 2, input_dim: int = 256, output_dim: int = 78, output_edge_dim: int = 256,
                 hidden_dim_processor_node: int = 256, hidden_dim_processor_edge: int = 256, hidden_layers_processor_node: int = 2,
                 hidden_layers_processor_edge: int = 2, mlp_norm_type: str = "LayerNorm", hidden_dim_decoder: int = 128,
                 hidden_layers_decoder: int = 2, use_checkpointing: bool = False, efficient_batching: bool = False,
                 precision: str = "auto", train_precision: Optional[str] = None):  # fmt: skip
        """assimilator_decoder.py:36-129 (Decoder: decoder.py:24-77).  train_precision=None (the default) keeps the module
        inference-only.  'fp32_simt' | 'fp32' | 'bf16' make a train-mode call with autograd on run the decoder's training step:
        processor_features, start_features (the Decoder's residual) and every parameter get gradients.  use_checkpointing, read at
        every training forward, selects the step as for Encoder: True keeps only the mesh-sized activations and recomputes the
        decoder chunk by chunk in the backward."""
        super().__init__()
        self.use_checkpointing = use_checkpointing
        self.efficient_batching = efficient_batching
        self.num_latlons = len(lat_lons)
        self.resolution = resolution
        self._g_dec = graphs.build_decoder_graph(lat_lons, resolution)
        self.num_h3 = self._g_dec.num_h3
        self.output_dim = output_dim
        self.edge_encoder = MLP(2, output_edge_dim, hidden_dim_processor_edge, 2, mlp_norm_type)
        self.graph_processor = GraphProcessor(1, input_dim, output_edge_dim, hidden_dim_processor_node, hidden_dim_processor_edge,
                                              hidden_layers_processor_node, hidden_layers_processor_edge, mlp_norm_type)  # fmt: skip
        self.node_decoder = MLP(input_dim, output_dim, hidden_dim_decoder, hidden_layers_decoder, None)
        self._residual = False
        self._dims = dict(
            n_in=0, n_out=self.num_latlons, n_mesh=self.num_h3, n_lat_edges=0, n_dec_edges=int(self._g_dec.src.size),
            in_dim=1, enc_edge_attr_dim=2, out_dim=output_dim, residual_dim=0, node_dim=input_dim, edge_dim=output_edge_dim,
            hidden_node=hidden_dim_processor_node, hidden_edge=hidden_dim_processor_edge,
            hidden_layers_node=hidden_layers_processor_node, hidden_layers_edge=hidden_layers_processor_edge,
            hidden_dec=hidden_dim_decoder, hidden_layers_dec=hidden_layers_decoder, num_blocks=1,
        )  # fmt: skip
        _validate_precision(precision, self._dims)
        self._precision = precision
        _check_train_precision(train_precision, self._dims)
        self.train_precision = train_precision
        self._engine = None

    def _upload_graphs(self, plan):
        g = self._g_dec
        plan.set_decoder_graph(g.src, g.ptr, g.edge_attr)

    def _run(self, processor_features, batch_size, start_features):
        if processor_features.device.type != "cuda":
            _no_host_path("Decoder.forward")
        if _stage_wants_grad(self, processor_features, start_features):
            return self._train_run(processor_features, batch_size, start_features)
        x = processor_features.detach().to(torch.float32).contiguous()
        start = None if start_features is None else start_features.detach().to(torch.float32).contiguous()
        eng = _own_engine(self, dict(self._dims, residual_dim=self.output_dim if self._residual else 0))
        plan = eng.ensure(x.device, batch_size, _prefixed("decoder", self))
        out = torch.empty((batch_size, self.num_latlons, self.output_dim), dtype=torch.float32, device=x.device)
        plan.decoder_forward(x, start, out, batch_size)
        _maybe_check(plan)
        return out

    def _train_run(self, processor_features, batch_size, start_features):
        """The training step of the decoder's forward (`_StageFn`).  The residual's gradient is the output's gradient itself."""
        x = processor_features.to(torch.float32).contiguous()
        if x.numel() != batch_size * self.num_h3 * self._dims["node_dim"]:
            raise RuntimeError(f"processor_features: expected {batch_size} x {self.num_h3} mesh rows of width {self._dims['node_dim']}, "
                               f"got {tuple(processor_features.shape)}")  # fmt: skip
        eng = _stage_engine(self, dict(self._dims, residual_dim=self.output_dim if self._residual else 0), [self._upload_graphs],
                            self.use_checkpointing)  # fmt: skip
        plan = eng.ensure(x.device, batch_size, _prefixed("decoder", self))
        out_shape, x_shape = (batch_size, self.num_latlons, self.output_dim), tuple(x.shape)

        def forward(tape, xi, *start):
            out = torch.empty(out_shape, dtype=torch.float32, device=xi.device)
            tape.decoder_forward(xi, start[0] if start else None, out, batch_size)
            return out

        def backward(tape, g, named):
            gx = torch.empty(x_shape, dtype=torch.float32, device=g[0].device)
            tape.decoder_backward(g[0], gx, named)
            return (gx, g[0]) if start_features is not None else (gx,)

        inputs = (x,) if start_features is None else (x, start_features.to(torch.float32).contiguous())
        return _run_stage(eng, plan, "decoder", self, inputs, forward, backward)

    def forward(self, processor_features: torch.Tensor, batch_size: int) -> torch.Tensor:
        return self._run(processor_features, batch_size, None)


class Decoder(AssimilatorDecoder):
    def __init__(self, lat_lons, resolution: int = 2, input_dim: int = 256, output_dim: int = 78, output_edge_dim: int = 256,
                 hidden_dim_processor_node: int = 256, hidden_dim_processor_edge: int = 256, hidden_layers_processor_node: int = 2,
                 hidden_layers_processor_edge: int = 2, mlp_norm_type: str = "LayerNorm", hidden_dim_decoder: int = 128,
                 hidden_layers_decoder: int = 2, use_checkpointing: bool = False, efficient_batching: bool = False,
                 precision: str = "auto", train_precision: Optional[str] = None):  # fmt: skip
        super().__init__(lat_lons, resolution, input_dim, output_dim, output_edge_dim, hidden_dim_processor_node,
                         hidden_dim_processor_edge, hidden_layers_processor_node, hidden_layers_processor_edge, mlp_norm_type,
                         hidden_dim_decoder, hidden_layers_decoder, use_checkpointing, efficient_batching, precision,
                         train_precision)  # fmt: skip
        self._residual = True

    def forward(self, processor_features: torch.Tensor, start_features: torch.Tensor, t: int = 0) -> torch.Tensor:
        if start_features.shape[-1] != self.output_dim:  # same failure point as the reference's broadcast add (decoder.py:93)
            raise RuntimeError(
                f"The size of tensor a ({self.output_dim}) must match the size of tensor b ({start_features.shape[-1]}) "
                "at non-singleton dimension 2"
            )
        return self._run(processor_features, start_features.shape[0], start_features)


# ---------------------------------------------------------------------------------------------------------------
# AssimilatorEncoder (assimilator_encoder.py)
# ---------------------------------------------------------------------------------------------------------------
class AssimilatorEncoder(nn.Module):
    def __init__(self, resolution: int = 2, input_dim: int = 2, output_dim: int = 256, output_edge_dim: int = 256,
                 hidden_dim_processor_node: int = 256, hidden_dim_processor_edge: int = 256, hidden_layers_processor_node: int = 2,
                 hidden_layers_processor_edge: int = 2, mlp_norm_type: str = "LayerNorm", use_checkpointing: bool = False,
                 precision: str = "auto", train_precision: Optional[str] = None):  # fmt: skip
        """assimilator_encoder.py:36-168.  train_precision as for Encoder: None keeps the module inference-only; a value makes a
        train-mode call with autograd on differentiable in the observation values and every parameter (not in lat_lon_heights).
        The observation graph belongs to the plan, so of two training forwards alive at once only the later one can run its
        backward (the earlier one's raises).  use_checkpointing selects the bounded-memory step as for Encoder; as the observation
        graph changes with every call, each bounded step copies its slot table to the host once to cut the chunks."""
        super().__init__()
        self.use_checkpointing = use_checkpointing
        self.output_dim = output_dim
        self.input_dim = input_dim
        self.resolution = resolution
        self._g_lat = graphs.build_mesh_graph(resolution)
        self.num_h3 = self._g_lat.num_h3
        self.h3_nodes = torch.zeros((h3lite.get_num_cells(resolution), input_dim), dtype=torch.float)  # plain tensor, :80
        self.node_encoder = MLP(input_dim, output_dim, hidden_dim_processor_node, hidden_layers_processor_node, mlp_norm_type)
        self.edge_encoder = MLP(3, output_edge_dim, hidden_dim_processor_edge, hidden_layers_processor_edge, mlp_norm_type)
        self.latent_edge_encoder = MLP(2, output_edge_dim, hidden_dim_processor_edge, hidden_layers_processor_edge, mlp_norm_type)
        self.graph_processor = GraphProcessor(1, output_dim, output_edge_dim, hidden_dim_processor_node, hidden_dim_processor_edge,
                                              hidden_layers_processor_node, hidden_layers_processor_edge, mlp_norm_type)  # fmt: skip
        self._dims = dict(
            n_in=1, n_out=0, n_mesh=self.num_h3, n_lat_edges=self._g_lat.edge_index.shape[1], n_dec_edges=0, in_dim=input_dim,
            enc_edge_attr_dim=3, out_dim=1, residual_dim=0, node_dim=output_dim, edge_dim=output_edge_dim,
            hidden_node=hidden_dim_processor_node, hidden_edge=hidden_dim_processor_edge,
            hidden_layers_node=hidden_layers_processor_node, hidden_layers_edge=hidden_layers_processor_edge,
            hidden_dec=1, hidden_layers_dec=1, num_blocks=1,
        )  # fmt: skip
        _validate_precision(precision, self._dims)
        self._precision = precision
        _check_train_precision(train_precision, self._dims)
        self.train_precision = train_precision
        self._engine = None
        self.efficient_batching = False
        self._lat_edge_index_t = {}

    def _upload_graphs(self, plan):
        m = self._g_lat
        plan.set_latent_graph(m.src, m.dst, m.ptr, m.edge_attr[m.perm])
        plan.set_h3_tables(h3lite.device_tables(self.resolution))  # for the device-side observation graph

    def _upload_obs(self, engine, plan, lat_lon_heights):
        """The reference rebuilds the observation graph on every forward (assimilator_encoder.py:118,170-216).  Here the
        upload is skipped only when the observation set is provably the same: the key is the CONTENT of lat_lon_heights
        (it is copied to the host to build the graph anyway) plus the engine's plan generation, never a tensor address.  The key
        is kept per engine: the inference and training engines hold different plans."""
        if lat_lon_heights.is_cuda and os.environ.get("GW_B200_HOST_OBS_GRAPH", "0") != "1":
            # the observation graph is rebuilt ON THE DEVICE for every call, as the reference rebuilds it for every call
            # (assimilator_encoder.py:118): point location, edge attributes, slot-sorted CSR -- no host copy, no synchronisation
            plan.build_obs_graph(lat_lon_heights.detach().to(device=plan.device, dtype=torch.float32).contiguous())
            engine.obs_key = None
            return
        llh = lat_lon_heights.detach().to(device="cpu", dtype=torch.float64).contiguous().numpy()
        key = (engine.generation, llh.shape, hash(llh.tobytes()))
        if key != engine.obs_key:
            g = graphs.build_encoder_graph(llh[:, :2], self.resolution, heights=llh[:, 2])
            plan.set_encoder_graph(g.mesh_local, g.perm, g.ptr, g.edge_attr)
            engine.obs_key = key

    _latent_edge_index = Encoder._latent_edge_index
    _latent_outputs = Encoder._latent_outputs
    _train_encode = Encoder._train_encode
    _encode = Encoder._encode

    def forward(self, features: torch.Tensor, lat_lon_heights: torch.Tensor):
        return self._encode(features, "AssimilatorEncoder.forward", lat_lon_heights)


# ---------------------------------------------------------------------------------------------------------------
# wrappers (forecast.py, analysis.py)
# ---------------------------------------------------------------------------------------------------------------
class _Wrapper(nn.Module):
    """What GraphWeatherForecaster, GraphCast and GraphWeatherAssimilator share: one inference engine over the whole network
    (encoder -> processor -> decoder in one plan), the training engines of `_TrainFn`, and the dispatch between the two."""

    def _init_engine(self, out_dim, residual_dim, num_blocks, precision, train_precision):
        """The network's plan dims from the encoder's and decoder's, the inference engine, and the `train_precision` check."""
        dec = self.decoder._dims
        dims = dict(self.encoder._dims)
        dims.update(n_out=self.decoder.num_latlons, n_dec_edges=dec["n_dec_edges"], out_dim=out_dim, residual_dim=residual_dim,
                    hidden_dec=dec["hidden_dec"], hidden_layers_dec=dec["hidden_layers_dec"], num_blocks=num_blocks)  # fmt: skip
        self._engine = _new_engine(dims, precision, [self.encoder._upload_graphs, self.decoder._upload_graphs])
        _validate_train_precision(train_precision, dims)
        if dec["edge_dim"] != dims["edge_dim"]:
            # GraphCast(hidden_dim != 256): the reference's decoder keeps its default 256-wide edges (graphcast/model.py:97-111
            # passes no output_edge_dim) while the encoder and processor edges are hidden_dim wide
            raise NotImplementedError(
                f"decoder edge width {dec['edge_dim']} differs from the encoder's {dims['edge_dim']}: the CUDA plan runs one edge width "
                "through the whole network, so this model is not supported (GraphCast runs with hidden_dim=256 only)")
        self.train_precision = train_precision

    def _named(self):
        return [(k, v) for k, v in self.state_dict(keep_vars=True).items()]

    def _grad_bindings(self):
        """`_TrainFn`'s bindings: every parameter under its own name, its gradient as the step returns it."""
        return [(k, q, q, None) for k, q in self.named_parameters()]

    def _out_shape(self, batch):
        return (batch, self.decoder.num_latlons, self.decoder.output_dim)

    def _bounded_step(self) -> bool:
        return bool(self.use_checkpointing)

    def _processor_segments(self) -> int:
        """Processor segments of a training forward (`Processor.set_checkpoint_segments`), read at every training forward."""
        return self.processor.checkpoint_segments

    def _training_engine(self):
        """The plan the training step runs on, of precision `train_precision`; the inference engine stays as it is.  A
        tensor-core training precision needs an sm_90 device: elsewhere the first training forward raises.

        `_bounded_step()` (use_checkpointing=True, forecast.py:81; GraphCast adds its checkpoint controls), read at every training
        forward, selects the step: a training-only plan whose step keeps only the mesh-sized activations and recomputes the
        grid-sized stages chunk by chunk in the backward -- its working memory does not grow with the grid beyond one chunk (the
        0.25 degree grid trains on one 80 GB card) -- or the taped step (the default), which is faster where it fits.  Each
        engine is created on first use.  Only one holds a plan: switching closes the other's, so a backward of a forward made
        under the other step raises "one backward per forward"."""
        def make(bounded):
            return _new_engine(self._engine.dims, self.train_precision, [self.encoder._upload_graphs, self.decoder._upload_graphs],
                               train_only=bounded)  # fmt: skip

        eng = _switch_training_engine(self.__dict__.setdefault("_train_engines", {}), self._bounded_step(), make)
        self.__dict__["_train_engine"] = eng
        return eng

    def _inference_plan(self, features, obs=None):
        """The inference engine's plan for this batch (and for the assimilator, these observations) with the current weights."""
        if obs is None:
            return self._engine.ensure(features.device, features.shape[0], self._named())
        plan = self._engine.ensure(features.device, features.shape[0], self._named(), grow=dict(n_in=obs.shape[0]))
        self.encoder._upload_obs(self._engine, plan, obs)
        return plan

    def _infer(self, features, out, obs=None, out_ld=None):
        """One inference forward into `out` (a float32 tensor, or the shape of one to allocate)."""
        plan = self._inference_plan(features, obs)
        f = features.detach().to(torch.float32).contiguous()
        if not torch.is_tensor(out):
            out = torch.empty(out, dtype=torch.float32, device=f.device)
        plan.forward(f, out, out_ld=out_ld)
        _maybe_check(plan)
        return out

    @contextlib.contextmanager
    def multi_step(self):
        """Training forwards made inside this window each keep a tape of their own, so a loss summed over an autoregressive
        rollout back-propagates through every step with one `backward()`:

            with model.multi_step():
                y1 = model(x0)
                y2 = model(torch.cat([y1, aux1], -1))
            (crit(y1, t1) + crit(y2, t2)).backward()

        Each forward's autograd node owns its tape: the backward consumes it, and dropping the graph without a backward frees it.
        Tapes made inside stay valid after the window exits; exiting only changes what later forwards do (outside it, a training
        forward replaces the previous one's activations, as it always has).  A backward raises once its tape's plan was replaced
        (a switch between the taped and the bounded step, a larger batch, `.to()`) or the weights were re-uploaded after its
        forward (an optimiser step followed by another forward).  The memory of the window grows with the number of live tapes
        (tools/train_step_bench.py --rollout K reports it)."""
        depth = self.__dict__.get("_multi_step", 0)
        self.__dict__["_multi_step"] = depth + 1
        try:
            yield self
        finally:
            self.__dict__["_multi_step"] = depth

    def _train_or_infer(self, features, obs=None):
        """The training step in train mode with autograd on (`_wants_grad`), otherwise inference."""
        if _wants_grad(self, features):
            bindings = self._grad_bindings()
            return _TrainFn.apply(self, features, obs, bindings, *[q for _, _, q, _ in bindings])
        return self._infer(features, self._out_shape(features.shape[0]), obs)


@dataclass
class GraphWeatherForecasterConfig:
    """forecast.py:14-58"""

    lat_lons: list
    resolution: int = 2
    feature_dim: int = 78
    aux_dim: int = 24
    output_dim: Optional[int] = None
    node_dim: int = 256
    edge_dim: int = 256
    num_blocks: int = 9
    hidden_dim_processor_node: int = 256
    hidden_dim_processor_edge: int = 256
    hidden_layers_processor_node: int = 2
    hidden_layers_processor_edge: int = 2
    hidden_dim_decoder: int = 128
    hidden_layers_decoder: int = 2
    norm_type: str = "LayerNorm"
    use_checkpointing: bool = False
    constraint_type: str = "none"
    use_thermalizer: bool = False
    train_precision: str = "fp32_simt"

    def build(self) -> "GraphWeatherForecaster":
        return GraphWeatherForecaster(**self.__dict__)


class GraphWeatherForecaster(_Wrapper, PyTorchModelHubMixin):
    """GraphWeatherForecaster(lat_lons)(features): forecast.py:61-247, the main weather prediction model, optionally with physical
    constraints (constraint_type 'additive' | 'multiplicative' | 'softmax', upsampling factor 1); no thermalizer.  Inference and
    training (train mode with autograd on: `loss.backward()` runs the CUDA backward of the network and of the constraint layer)
    run on the device."""

    def __init__(self, lat_lons: list, resolution: int = 2, feature_dim: int = 78, aux_dim: int = 24, output_dim: Optional[int] = None,
                 node_dim: int = 256, edge_dim: int = 256, num_blocks: int = 9, hidden_dim_processor_node: int = 256,
                 hidden_dim_processor_edge: int = 256, hidden_layers_processor_node: int = 2, hidden_layers_processor_edge: int = 2,
                 hidden_dim_decoder: int = 128, hidden_layers_decoder: int = 2, norm_type: str = "LayerNorm",
                 use_checkpointing: bool = False, constraint_type: str = "none", use_thermalizer: bool = False,
                 precision: str = "auto", train_precision: str = "fp32_simt"):  # fmt: skip
        super().__init__()
        if use_thermalizer:
            raise NotImplementedError("use_thermalizer=True is outside the accelerated path (stochastic layer)")
        lat_lons = _latlon_list(lat_lons)
        graphs.validate_lat_lons(lat_lons)
        self.feature_dim = feature_dim
        self.constraint_type = constraint_type
        self.use_thermalizer = use_thermalizer
        self.use_checkpointing = use_checkpointing
        if output_dim is None:
            output_dim = self.feature_dim
        self.output_dim = output_dim
        # grid shape and the node -> (row, col) mapping of forecast.py:122-129,178-192
        self.original_lat_lons = list(lat_lons)
        self.__dict__["_grid_mapping"] = GridMapping(lat_lons)
        self.grid_shape = self._grid_mapping.grid_shape
        self.node_to_grid = self._grid_mapping.node_to_grid
        self.precision = precision
        self.encoder = Encoder(lat_lons=lat_lons, resolution=resolution, input_dim=feature_dim + aux_dim, output_dim=node_dim,
                               output_edge_dim=edge_dim, hidden_dim_processor_edge=hidden_dim_processor_edge,
                               hidden_layers_processor_node=hidden_layers_processor_node,
                               hidden_dim_processor_node=hidden_dim_processor_node,
                               hidden_layers_processor_edge=hidden_layers_processor_edge, mlp_norm_type=norm_type,
                               use_checkpointing=use_checkpointing, precision=precision)  # fmt: skip
        self.processor = Processor(input_dim=node_dim, edge_dim=edge_dim, num_blocks=num_blocks,
                                   hidden_dim_processor_edge=hidden_dim_processor_edge,
                                   hidden_layers_processor_node=hidden_layers_processor_node,
                                   hidden_dim_processor_node=hidden_dim_processor_node,
                                   hidden_layers_processor_edge=hidden_layers_processor_edge, mlp_norm_type=norm_type,
                                   use_thermalizer=use_thermalizer, precision=precision)  # fmt: skip
        self.decoder = Decoder(lat_lons=lat_lons, resolution=resolution, input_dim=node_dim, output_dim=output_dim,
                               output_edge_dim=edge_dim, hidden_dim_processor_edge=hidden_dim_processor_edge,
                               hidden_layers_processor_node=hidden_layers_processor_node,
                               hidden_dim_processor_node=hidden_dim_processor_node,
                               hidden_layers_processor_edge=hidden_layers_processor_edge, mlp_norm_type=norm_type,
                               hidden_dim_decoder=hidden_dim_decoder, hidden_layers_decoder=hidden_layers_decoder,
                               use_checkpointing=use_checkpointing, precision=precision)  # fmt: skip
        self._init_engine(output_dim, output_dim, num_blocks, precision, train_precision)
        if self.constraint_type != "none":  # forecast.py:162-170 (any other string fails at the first forward, as there)
            self.constraint = PhysicalConstraintLayer(model=self, grid_shape=self.grid_shape, constraint_type=constraint_type,
                                                      upsampling_factor=1)  # fmt: skip

    def graph_to_grid(self, graph_tensor: torch.Tensor) -> torch.Tensor:
        """[B, N, C] -> [B, C, H, W] (forecast.py:194-203)."""
        return self._grid_mapping.graph_to_grid(graph_tensor)

    def grid_to_graph(self, grid_tensor: torch.Tensor) -> torch.Tensor:
        """[B, C, H, W] -> [B, N, C] (forecast.py:205-213)."""
        return self._grid_mapping.grid_to_graph(grid_tensor)

    def _check_features(self, features):
        if features.device.type != "cuda":
            _no_host_path("GraphWeatherForecaster.forward")
        if features.shape[-1] < self.feature_dim or self.output_dim != self.feature_dim:
            # the reference fails at `out + start_features` (decoder.py:93) when output_dim != feature_dim
            raise RuntimeError(f"output_dim ({self.output_dim}) must equal feature_dim ({self.feature_dim}) for the residual add")

    def _constrain(self, out, f):
        """forecast.py:231-246: the decoder output, read as a row-major H x W grid, is corrected against the input's first
        feature_dim channels.  `rearrange(x, "b (h w) c -> b c h w")` only re-labels rows here: no layout pass exists."""
        return self.constraint.apply_rows(out, f, self._constraint_cell(out), self.feature_dim)

    def _constraint_cell(self, out):
        H, W = self.grid_shape
        if out.shape[1] != H * W:
            raise RuntimeError(f"Shape mismatch, can't divide axis of length {out.shape[1]} in chunks of {W}")  # einops' failure
        cell, _ = self._grid_mapping.tensors(out.device)
        return cell.to(torch.int32).contiguous()

    def forward(self, features: torch.Tensor, t: int = 0) -> torch.Tensor:
        self._check_features(features)
        # train mode with autograd on, like every training caller of the reference (train/run.py:508-543): the forward keeps
        # its activations and `loss.backward()` runs the CUDA backward.  Inference (`model.eval()` or `torch.no_grad()`) takes
        # the tensor-core path.
        out = self._train_or_infer(features)
        if self.constraint_type == "none":
            return out
        if out.requires_grad:
            # forecast.py:235-246 under autograd: the layer's backward adds the gradient of its `lr` input (the first
            # feature_dim features) to the residual and encoder paths of features.grad
            return self.constraint.constrain_rows(out, features[..., : self.feature_dim], self._constraint_cell(out))
        return self._constrain(out, features)

    def forward_into(self, features: torch.Tensor, out: torch.Tensor, peers=None) -> torch.Tensor:
        """forward(features) written into a caller-provided [B, N, output_dim] tensor.  `peers` = (mode, byte deltas) makes the
        chain that produces the forecast store it into every GPU's gather buffer as well (gw_plan_set_output_peers;
        graph_weather_b200.dist.BoundaryGather passes the aliases of its symmetric buffers): the multi-GPU loss-boundary gather,
        fused with the last GEMM.  Not available with a constraint layer (its correction follows the forecast)."""
        self._check_features(features)
        if self.constraint_type != "none":
            raise NotImplementedError("forward_into: the constraint layer post-processes the forecast; gather its output instead")
        if tuple(out.shape) != self._out_shape(features.shape[0]) or not out.is_contiguous() or out.dtype != torch.float32:
            raise RuntimeError("forward_into: `out` must be a contiguous float32 [B, N, output_dim] tensor")
        plan = self._inference_plan(features)
        f = features.detach().to(torch.float32).contiguous()
        if peers is not None:
            plan.set_output_peers(peers[0], peers[1])
        try:
            plan.forward(f, out, out_ld=self.output_dim)
        finally:
            if peers is not None:
                plan.set_output_peers(0)
        _maybe_check(plan)
        return out

    @torch.no_grad()
    def rollout(self, features: torch.Tensor, steps: int, aux=None, return_all: bool = True):
        """Autoregressive forecast: state_{t+1} = model([state_t | aux_t]) for `steps` steps (the loop every user of the
        reference writes around forecast.py:215-247; the reference has no helper for it).

        features [B, N, feature_dim + aux_dim] is step 0's input.  `aux` is None (the auxiliary columns of `features` are
        kept for every step), a tensor [steps, B, N, aux_dim] / [B, N, aux_dim], or a callable t -> [B, N, aux_dim].
        Every step writes its forecast straight into the first feature_dim columns of the next step's input rows
        (gw_forward_strided): no concatenation pass, no host round trip.  Returns [steps, B, N, feature_dim] (or the last
        state if return_all is False)."""
        self._check_features(features)
        B, N, Fin = features.shape
        plan = self._inference_plan(features)
        bufs = [features.detach().to(torch.float32).contiguous().clone(), None]
        bufs[1] = bufs[0].clone()  # aux columns are present in both from the start
        outs = torch.empty((steps if return_all else 1, B, N, self.output_dim), dtype=torch.float32, device=features.device)
        for t in range(steps):
            cur, nxt = bufs[t & 1], bufs[(t + 1) & 1]
            if aux is not None and Fin > self.feature_dim:
                a = aux(t) if callable(aux) else (aux[t] if aux.dim() == 4 else aux)
                cur[..., self.feature_dim :] = a.to(cur.dtype)
            if self.constraint_type == "none":
                plan.forward(cur, nxt, out_ld=Fin)  # forecast lands in nxt[..., :feature_dim]
                state = nxt[..., : self.output_dim]
            else:
                tmp = torch.empty((B, N, self.output_dim), dtype=torch.float32, device=cur.device)
                plan.forward(cur, tmp)
                state = self._constrain(tmp, cur)
                nxt[..., : self.output_dim] = state
            outs[t if return_all else 0] = state
        _maybe_check(plan)
        return outs if return_all else outs[0]


@dataclass
class GraphWeatherAssimilatorConfig:
    """analysis.py:11-49"""

    output_lat_lons: list
    resolution: int = 2
    observation_dim: int = 2
    analysis_dim: int = 78
    node_dim: int = 256
    edge_dim: int = 256
    num_blocks: int = 9
    hidden_dim_processor_node: int = 256
    hidden_dim_processor_edge: int = 256
    hidden_layers_processor_node: int = 2
    hidden_layers_processor_edge: int = 2
    hidden_dim_decoder: int = 128
    hidden_layers_decoder: int = 2
    norm_type: str = "LayerNorm"
    use_checkpointing: bool = False
    train_precision: str = "fp32_simt"

    def build(self) -> "GraphWeatherAssimilator":
        return GraphWeatherAssimilator(**self.__dict__)


class GraphWeatherAssimilator(_Wrapper, PyTorchModelHubMixin):
    """GraphWeatherAssimilator(output_lat_lons=..)(features, obs_lat_lon_heights): analysis.py:52-150.  Inference and training
    run on the device.  In train mode with autograd on, `loss.backward()` runs the CUDA backward (`train_precision`, as in
    GraphWeatherForecaster; use_checkpointing=True selects the bounded-memory step).  The observation graph is rebuilt for every
    training forward, as for every inference forward; `features.grad` is the gradient of the observation values, and
    `obs_lat_lon_heights` gets none (the reference builds the graph in numpy)."""

    def __init__(self, output_lat_lons: list, resolution: int = 2, observation_dim: int = 2, analysis_dim: int = 78,
                 node_dim: int = 256, edge_dim: int = 256, num_blocks: int = 9, hidden_dim_processor_node: int = 256,
                 hidden_dim_processor_edge: int = 256, hidden_layers_processor_node: int = 2, hidden_layers_processor_edge: int = 2,
                 hidden_dim_decoder: int = 128, hidden_layers_decoder: int = 2, norm_type: str = "LayerNorm",
                 use_checkpointing: bool = False, precision: str = "auto", train_precision: str = "fp32_simt"):  # fmt: skip
        super().__init__()
        output_lat_lons = _latlon_list(output_lat_lons)
        self.encoder = AssimilatorEncoder(resolution=resolution, input_dim=observation_dim, output_dim=node_dim,
                                          output_edge_dim=edge_dim, hidden_dim_processor_edge=hidden_dim_processor_edge,
                                          hidden_layers_processor_node=hidden_layers_processor_node,
                                          hidden_dim_processor_node=hidden_dim_processor_node,
                                          hidden_layers_processor_edge=hidden_layers_processor_edge, mlp_norm_type=norm_type,
                                          use_checkpointing=use_checkpointing, precision=precision)  # fmt: skip
        self.processor = Processor(input_dim=node_dim, edge_dim=edge_dim, num_blocks=num_blocks,
                                   hidden_dim_processor_edge=hidden_dim_processor_edge,
                                   hidden_layers_processor_node=hidden_layers_processor_node,
                                   hidden_dim_processor_node=hidden_dim_processor_node,
                                   hidden_layers_processor_edge=hidden_layers_processor_edge, mlp_norm_type=norm_type,
                                   precision=precision)  # fmt: skip
        self.decoder = AssimilatorDecoder(lat_lons=output_lat_lons, resolution=resolution, input_dim=node_dim, output_dim=analysis_dim,
                                          output_edge_dim=edge_dim, hidden_dim_processor_edge=hidden_dim_processor_edge,
                                          hidden_layers_processor_node=hidden_layers_processor_node,
                                          hidden_dim_processor_node=hidden_dim_processor_node,
                                          hidden_layers_processor_edge=hidden_layers_processor_edge, mlp_norm_type=norm_type,
                                          hidden_dim_decoder=hidden_dim_decoder, hidden_layers_decoder=hidden_layers_decoder,
                                          use_checkpointing=use_checkpointing, precision=precision)  # fmt: skip
        self.analysis_dim = analysis_dim
        self.use_checkpointing = use_checkpointing
        self._init_engine(analysis_dim, 0, num_blocks, precision, train_precision)

    def multi_step(self):
        raise NotImplementedError("GraphWeatherAssimilator.multi_step: the observation graph a training forward runs on belongs to the "
                                  "plan, not to the forward, so several forwards cannot stay differentiable at once")

    def forward(self, features: torch.Tensor, obs_lat_lon_heights: torch.Tensor) -> torch.Tensor:
        if features.device.type != "cuda":
            _no_host_path("GraphWeatherAssimilator.forward")
        return self._train_or_infer(features, obs_lat_lon_heights)


# ---------------------------------------------------------------------------------------------------------------
# GraphCast wrapper (graphcast/model.py)
# ---------------------------------------------------------------------------------------------------------------
class GraphCast(_Wrapper):
    """graph_weather/models/graphcast/model.py:21-285: Encoder + Processor + Decoder with hierarchical gradient-checkpoint
    controls and `efficient_batching`.  Efficient and replicated batching are the same computation -- the CUDA path always
    shares one graph across the batch (the reference proves the equivalence in tests/models/layers/test_efficient_batching.py).

    Inference and training run on the device.  In train mode with autograd on, `loss.backward()` runs the CUDA backward
    (`train_precision`, as in GraphWeatherForecaster; features.grad includes the residual path of the full input).  The
    checkpoint controls choose the training step, read at every training forward:
      * the bounded-memory step (a training-only plan that recomputes the grid-sized stages chunk by chunk in the backward) when
        use_checkpointing, set_checkpoint_model(True), set_checkpoint_encoder(True) or set_checkpoint_decoder(True) is set --
        GraphCastConfig.full_checkpointing and balanced_checkpointing;
      * the taped step otherwise.
    set_checkpoint_processor(segments) combines with either step: a non-zero value makes the backward recompute the processor in
    segments of that many blocks (-1: the whole processor as one) instead of keeping its tape -- GraphCastConfig.balanced_checkpointing
    and processor_only_checkpointing; 0 leaves the choice to processor.set_checkpoint_segments.  Checkpointing never changes the
    forward's result or the gradients, in the reference or here."""

    def __init__(self, lat_lons: list, resolution: int = 2, input_dim: int = 78, output_dim: int = 78, hidden_dim: int = 256,
                 num_processor_blocks: int = 9, hidden_layers: int = 2, mlp_norm_type: str = "LayerNorm",
                 use_checkpointing: bool = False, efficient_batching: bool = False, precision: str = "auto",
                 train_precision: str = "fp32_simt"):  # fmt: skip
        super().__init__()
        lat_lons = _latlon_list(lat_lons)
        self.lat_lons = lat_lons
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.efficient_batching = efficient_batching
        self.use_checkpointing = use_checkpointing
        self.encoder = Encoder(lat_lons=lat_lons, resolution=resolution, input_dim=input_dim, output_dim=hidden_dim,
                               output_edge_dim=hidden_dim, hidden_dim_processor_node=hidden_dim, hidden_dim_processor_edge=hidden_dim,
                               hidden_layers_processor_node=hidden_layers, hidden_layers_processor_edge=hidden_layers,
                               mlp_norm_type=mlp_norm_type, use_checkpointing=use_checkpointing,
                               efficient_batching=efficient_batching, precision=precision)  # fmt: skip
        self.processor = Processor(input_dim=hidden_dim, edge_dim=hidden_dim, num_blocks=num_processor_blocks,
                                   hidden_dim_processor_node=hidden_dim, hidden_dim_processor_edge=hidden_dim,
                                   hidden_layers_processor_node=hidden_layers, hidden_layers_processor_edge=hidden_layers,
                                   mlp_norm_type=mlp_norm_type, use_checkpointing=use_checkpointing, precision=precision)  # fmt: skip
        self.decoder = Decoder(lat_lons=lat_lons, resolution=resolution, input_dim=hidden_dim, output_dim=output_dim,
                               hidden_dim_processor_node=hidden_dim, hidden_dim_processor_edge=hidden_dim,
                               hidden_layers_processor_node=hidden_layers, hidden_layers_processor_edge=hidden_layers,
                               mlp_norm_type=mlp_norm_type, hidden_dim_decoder=hidden_dim, hidden_layers_decoder=hidden_layers,
                               use_checkpointing=use_checkpointing, efficient_batching=efficient_batching, precision=precision)  # fmt: skip
        self._checkpoint_model = False
        self._checkpoint_encoder = False
        self._checkpoint_processor_segments = 0
        self._checkpoint_decoder = False
        self._init_engine(output_dim, output_dim, num_processor_blocks, precision, train_precision)

    def _bounded_step(self) -> bool:
        return bool(self.use_checkpointing or self._checkpoint_model or self._checkpoint_encoder or self._checkpoint_decoder)

    def _processor_segments(self) -> int:
        return self._checkpoint_processor_segments or self.processor.checkpoint_segments

    # hierarchical checkpointing controls (model.py:118-174)
    def set_checkpoint_model(self, checkpoint_flag: bool):
        self._checkpoint_model = checkpoint_flag
        if checkpoint_flag:
            self._checkpoint_encoder = False
            self._checkpoint_processor_segments = 0
            self._checkpoint_decoder = False

    def set_checkpoint_encoder(self, checkpoint_flag: bool):
        self._checkpoint_encoder = checkpoint_flag

    def set_checkpoint_processor(self, checkpoint_segments: int):
        _check_segments(checkpoint_segments)
        self._checkpoint_processor_segments = checkpoint_segments

    def set_checkpoint_decoder(self, checkpoint_flag: bool):
        self._checkpoint_decoder = checkpoint_flag

    def forward(self, features: torch.Tensor) -> torch.Tensor:
        if features.device.type != "cuda":
            _no_host_path("GraphCast.forward")
        if features.shape[-1] != self.output_dim:  # the reference adds the full input as the residual (model.py:203, decoder.py:93)
            raise RuntimeError(f"The size of tensor a ({self.output_dim}) must match the size of tensor b ({features.shape[-1]}) "
                               "at non-singleton dimension 2")  # fmt: skip
        return self._train_or_infer(features)


class GraphCastConfig:
    """graphcast/model.py:288-345: pre-defined checkpointing strategies."""

    @staticmethod
    def no_checkpointing(model: GraphCast):
        model.set_checkpoint_model(False), model.set_checkpoint_encoder(False)
        model.set_checkpoint_processor(0), model.set_checkpoint_decoder(False)

    @staticmethod
    def full_checkpointing(model: GraphCast):
        model.set_checkpoint_model(True)

    @staticmethod
    def balanced_checkpointing(model: GraphCast):
        model.set_checkpoint_model(False), model.set_checkpoint_encoder(True)
        model.set_checkpoint_processor(-1), model.set_checkpoint_decoder(True)

    @staticmethod
    def processor_only_checkpointing(model: GraphCast):
        model.set_checkpoint_model(False), model.set_checkpoint_encoder(False)
        model.set_checkpoint_processor(-1), model.set_checkpoint_decoder(False)

    @staticmethod
    def fine_grained_checkpointing(model: GraphCast):
        model.set_checkpoint_model(False), model.set_checkpoint_encoder(False)
        model.set_checkpoint_processor(0), model.set_checkpoint_decoder(False)
