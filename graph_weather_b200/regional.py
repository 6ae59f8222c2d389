"""RegionalForecaster (graph_weather/models/regional_forecast.py:16-298): the encode-process-decode forward over a movable
high-resolution domain, on the same CUDA plan as GraphWeatherForecaster.

The reference builds three graphs per region with DynamicGraphBuilder (local numbering over the H3 cells the coordinates
touch), gathers the region's rows of a global per-cell embedding table, and runs -- per sample, in Python -- node encoder,
one bipartite GNN block (observations -> cells), `num_blocks` latent blocks, one GNN block over the REVERSED encoder edges
(cells -> observations, one edge per observation) and the node decoder, then adds the first `output_dim` input channels
(:252-291).  That is the forecaster's pipeline with other graphs, so it runs on the forecaster's kernels: the module keeps
the reference's parameter names (`node_encoder`, `encoder_gnn`, `decoder_edge_encoder`, ...; same state_dict keys and shapes)
and hands them to the plan under the names the C ABI binds (include/gw_b200.h), with the region's embedding rows as
`encoder.h3_nodes`.  A plan is sized for one region; a region with other counts gets its own plan (a handful are kept).

Training (`train_precision`, as on the other wrappers): in train mode with autograd on, a forward runs the forecaster's CUDA
training step on training plans of the region (`use_checkpointing=True`: the bounded-memory step).  `h3_embeddings.grad` is
table-shaped, as the reference's: the region's rows at their cells, zero elsewhere.  A region's plans are kept while a backward
still needs one of their tapes, so the losses of more regions than the cache holds can be summed into one `backward()`.

Optional boundary nudging (:44-130): a distance-based relaxation prior plus a learned one-hidden-layer correction, blended
with a caller-supplied global forecast.  It is a [B, N, 2F+1] -> 1 element-wise tail outside the GNN; it runs as device
tensor ops (no kernels of this library), exactly the reference's arithmetic.
"""

from __future__ import annotations

import math
from collections import OrderedDict
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import graphs, h3lite
from .dynamic_graph_builder import DynamicGraphBuilder
from .models import (MLP, GraphProcessor, Processor, _maybe_check, _new_engine, _no_host_path, _pending_tape, _switch_training_engine,
                     _TrainFn, _validate_precision, _validate_train_precision, _Wrapper, _wants_grad)  # fmt: skip


@dataclass
class RegionalForecasterConfig:
    """regional_forecast.py:16-41 (same fields and defaults) + `precision` of the CUDA path and `train_precision` of its training
    step: None (the default) leaves the model inference-only, 'fp32_simt' | 'fp32' | 'bf16' train it as GraphWeatherForecaster's
    `train_precision` does (the tensor-core values need the 256-wide trunk and output_dim <= 256)."""

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
    enable_nudging: bool = False
    nudging_hidden_dim: int = 64
    precision: str = "auto"
    train_precision: Optional[str] = None

    def build(self) -> "RegionalForecaster":
        return RegionalForecaster(self)


class BoundaryNudgingLayer(nn.Module):
    """regional_forecast.py:44-130: alpha = clamp(prior + MLP([regional, global, prior]), 0, 1); out = (1-alpha) regional + alpha global."""

    def __init__(self, feature_dim: int, hidden_dim: int = 64):
        super().__init__()
        self.blend_mlp = MLP(feature_dim * 2 + 1, 1, hidden_dim, 1, None)

    def forward(self, regional: torch.Tensor, global_context: torch.Tensor, lat_lons: list) -> torch.Tensor:
        alpha_prior = self._compute_relaxation_weights(lat_lons, regional.device)
        alpha_prior = alpha_prior.unsqueeze(0).expand(regional.shape[0], -1, -1)
        h = torch.cat([regional, global_context, alpha_prior], dim=-1)
        lin0, lin1 = self.blend_mlp.model[0], self.blend_mlp.model[2]  # Linear, ReLU, Linear (one hidden layer, no norm)
        corr = torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(h, lin0.weight, lin0.bias)), lin1.weight, lin1.bias)
        alpha = torch.clamp(alpha_prior + corr, 0.0, 1.0)
        return (1 - alpha) * regional + alpha * global_context

    @staticmethod
    def _compute_relaxation_weights(lat_lons: list, device) -> torch.Tensor:
        """[N, 1] relaxation prior (:92-130): great-circle distance of every coordinate from the centroid of the region (mean of
        the latitudes / longitudes in radians), divided by the largest one -- 0 at the centre, 1 at the farthest point, all zeros
        for a single point.  float32 throughout, like the reference."""
        ll = torch.as_tensor(np.asarray(lat_lons, dtype=np.float32).reshape(-1, 2)) * (math.pi / 180.0)
        lat, lon = ll[:, 0], ll[:, 1]
        lat_c, lon_c = lat.mean(), lon.mean()
        hav = torch.sin((lat - lat_c) / 2) ** 2 + torch.cos(lat) * torch.cos(lat_c) * torch.sin((lon - lon_c) / 2) ** 2
        dist = 2 * torch.asin(torch.sqrt(hav.clamp(0.0, 1.0)))
        far = dist.max()
        prior = dist / far if far > 0 else torch.zeros_like(dist)
        return prior.unsqueeze(-1).to(device)


class _RegionGraphs:
    """The three graphs of one region in the forms the plan takes (target-sorted int32 + float32 attributes)."""

    def __init__(self, builder: DynamicGraphBuilder, lat_lons):
        enc, _dec, lat, h3_indices = builder(lat_lons)
        n = len(lat_lons)
        self.n_obs = n
        self.h3_indices = np.asarray(h3_indices, dtype=np.int64)
        self.n_mesh = int(self.h3_indices.size)
        ei = enc.edge_index.numpy()
        self.mesh_local = (ei[1] - n).astype(np.int32)  # the cell (local index) every coordinate feeds, :40-66
        self.enc_attr = np.ascontiguousarray(enc.edge_attr.numpy(), dtype=np.float32)
        perm, _, _, ptr = graphs._finish_target_sorted(np.arange(n), self.mesh_local.astype(np.int64), self.n_mesh)
        self.enc_perm, self.enc_ptr = perm.astype(np.int32), ptr
        li = lat.edge_index.numpy()
        lperm, self.lat_src, self.lat_dst, self.lat_ptr = graphs._finish_target_sorted(li[0], li[1], self.n_mesh)
        self.lat_attr = np.ascontiguousarray(lat.edge_attr.numpy()[lperm], dtype=np.float32)
        self.n_lat_edges = int(li.shape[1])
        self.h3_idx = None  # h3_indices on the device (set with the region's embedding rows, RegionalForecaster._plan_named)
        # decoder = the encoder edges reversed (:247-249): exactly one edge per coordinate, from its own cell
        self.dec_src = self.mesh_local
        self.dec_ptr = np.arange(n + 1, dtype=np.int32)

    def upload(self, plan):
        plan.set_encoder_graph(self.mesh_local, self.enc_perm, self.enc_ptr, self.enc_attr)
        plan.set_latent_graph(self.lat_src, self.lat_dst, self.lat_ptr, self.lat_attr)
        plan.set_decoder_graph(self.dec_src, self.dec_ptr, self.enc_attr)


class RegionalForecaster(nn.Module):
    """RegionalForecaster(config)(features, lat_lons, global_context=None) -> [B, N_obs, output_dim]  (regional_forecast.py:133-298)."""

    _MAX_PLANS = 4

    def __init__(self, config: RegionalForecasterConfig):
        super().__init__()
        self.config = config
        c = config
        input_dim = c.feature_dim + c.aux_dim
        output_dim = c.output_dim if c.output_dim is not None else c.feature_dim
        self.output_dim = output_dim
        self.nudging = BoundaryNudgingLayer(output_dim, c.nudging_hidden_dim) if c.enable_nudging else None
        self.graph_builder = DynamicGraphBuilder(resolution=c.resolution)
        self.h3_embeddings = nn.Parameter(torch.zeros(h3lite.get_num_cells(c.resolution), input_dim))
        hn, he, ln, le = c.hidden_dim_processor_node, c.hidden_dim_processor_edge, c.hidden_layers_processor_node, c.hidden_layers_processor_edge

        def mlp(i, o, h, n):
            return MLP(i, o, h, n, c.norm_type, c.use_checkpointing)

        def block():  # one bipartite GNN block (encoder_gnn / decoder_gnn, :170-181, :211-222)
            return GraphProcessor(1, c.node_dim, c.edge_dim, hn, he, ln, le, c.norm_type)

        # registration order = the reference's (:158-231): it fixes the state_dict key order
        self.node_encoder = mlp(input_dim, c.node_dim, hn, ln)
        self.edge_encoder = mlp(2, c.edge_dim, he, le)
        self.encoder_gnn = block()
        self.latent_edge_encoder = mlp(2, c.edge_dim, he, le)
        self.processor = Processor(input_dim=c.node_dim, edge_dim=c.edge_dim, num_blocks=c.num_blocks, hidden_dim_processor_edge=he,
                                   hidden_layers_processor_node=ln, hidden_dim_processor_node=hn, hidden_layers_processor_edge=le,
                                   mlp_norm_type=c.norm_type, precision=c.precision)  # fmt: skip
        self.decoder_edge_encoder = mlp(2, c.edge_dim, he, le)
        self.decoder_gnn = block()
        self.node_decoder = mlp(c.node_dim, output_dim, c.hidden_dim_decoder, c.hidden_layers_decoder)  # WITH the norm (:224-231)
        self._base_dims = dict(
            in_dim=input_dim, enc_edge_attr_dim=2, out_dim=output_dim, residual_dim=output_dim, node_dim=c.node_dim, edge_dim=c.edge_dim,
            hidden_node=c.hidden_dim_processor_node, hidden_edge=c.hidden_dim_processor_edge,
            hidden_layers_node=c.hidden_layers_processor_node, hidden_layers_edge=c.hidden_layers_processor_edge,
            hidden_dec=c.hidden_dim_decoder, hidden_layers_dec=c.hidden_layers_decoder, num_blocks=c.num_blocks,
        )  # fmt: skip
        probe = dict(self._base_dims, n_in=1, n_out=1, n_mesh=1, n_lat_edges=1, n_dec_edges=1)
        _validate_precision(c.precision, probe)
        if c.train_precision is not None:
            _validate_train_precision(c.train_precision, probe)
            if c.train_precision != "fp32_simt" and output_dim > 256:
                raise ValueError(
                    f"train_precision={c.train_precision!r} with output_dim={output_dim}: the node decoder ends in a LayerNorm over "
                    "output_dim columns, and a LayerNorm'd row must stay in one tensor-core chain of at most 256 columns; use "
                    "train_precision='fp32_simt'")  # fmt: skip
        self.train_precision = c.train_precision
        self.use_checkpointing = c.use_checkpointing
        # per-region state: graphs are cached like the reference's builder caches them (same list object -> same graphs)
        self.__dict__["_regions"] = OrderedDict()  # id(lat_lons) -> (lat_lons, _RegionGraphs, engines)
        self.__dict__["_active"] = None  # (graphs, engines) of the region of the current training forward

    # ---- the plan's view of the parameters -------------------------------------------------------------------------------
    _RENAME = (
        ("node_encoder.", "encoder.node_encoder."),
        ("edge_encoder.", "encoder.edge_encoder."),
        ("encoder_gnn.", "encoder.graph_processor."),
        ("latent_edge_encoder.", "encoder.latent_edge_encoder."),
        ("processor.", "processor."),
        ("decoder_edge_encoder.", "decoder.edge_encoder."),
        ("decoder_gnn.", "decoder.graph_processor."),
        ("node_decoder.", "decoder.node_decoder."),
    )

    def _plan_named(self, region: _RegionGraphs):
        out = []
        for k, v in self.state_dict(keep_vars=True).items():
            if k == "h3_embeddings":  # the region's rows of the global table (:243); re-gathered only when the table changed
                key = (v.data_ptr(), v._version, str(v.device))
                if getattr(region, "_h3_key", None) != key:
                    region.h3_idx = torch.from_numpy(region.h3_indices).to(v.device)
                    region._h3_rows, region._h3_key = v.detach()[region.h3_idx].contiguous(), key
                out.append(("encoder.h3_nodes", region._h3_rows))
                continue
            for a, b in self._RENAME:
                if k.startswith(a):
                    out.append((b + k[len(a):], v))
                    break
        return out

    # ---- what _TrainFn asks of its wrapper, for the region of the current training forward -------------------------------
    def _named(self):
        return self._plan_named(self._active[0])

    def _out_shape(self, batch):
        return (batch, self._active[0].n_obs, self.output_dim)

    def _training_engine(self):
        """The region's training engine of precision `train_precision`: the bounded-memory step (a training-only plan) when
        use_checkpointing is set, else the taped step; switching closes the region's other training plan (see
        _Wrapper._training_engine)."""
        region, engines = self._active

        def make(bounded):
            return _new_engine(engines["infer"].dims, self.train_precision, [region.upload], train_only=bounded)

        eng = _switch_training_engine(engines, bool(self.use_checkpointing), make)
        self.__dict__["_train_engine"] = eng
        return eng

    def _processor_segments(self) -> int:
        """Processor segments of a training forward (`processor.set_checkpoint_segments`)."""
        return self.processor.checkpoint_segments

    def _grad_bindings(self):
        """The plan's parameters; `encoder.h3_nodes` (the region's rows of h3_embeddings) differentiates the table: the rows'
        gradients go to the region's cells (unique, so a copy), every other row is zero.  The nudging layer is not bound: its
        parameters are differentiated by torch."""
        named = self._named()
        table, idx = self.h3_embeddings, self._active[0].h3_idx

        def to_table(g):
            full = g.new_zeros(table.shape)
            full[idx] = g
            return full

        return [(k, v, table, to_table) if k == "encoder.h3_nodes" else (k, v, v, None) for k, v in named]

    multi_step = _Wrapper.multi_step

    def _region(self, lat_lons):
        """The region's graphs and engines ({"infer": inference, False: taped step, True: bounded step}), built on first use.
        Least recently used regions beyond _MAX_PLANS are dropped with their plans, except a region one of whose tapes a
        backward still needs: the cache then holds more regions until those tapes are consumed or dropped, and shrinks back
        at a later forward."""
        key = id(lat_lons)
        hit = self._regions.get(key)
        if hit is not None and hit[0] is lat_lons:
            self._regions.move_to_end(key)
            g, engines = hit[1], hit[2]
        else:
            g = _RegionGraphs(self.graph_builder, lat_lons)
            dims = dict(self._base_dims, n_in=g.n_obs, n_out=g.n_obs, n_mesh=g.n_mesh, n_lat_edges=g.n_lat_edges, n_dec_edges=g.n_obs)
            engines = {"infer": _new_engine(dims, self.config.precision, [g.upload])}
            self._regions[key] = (lat_lons, g, engines)
        for k in list(self._regions):
            if len(self._regions) <= self._MAX_PLANS:
                break
            if k == key or any(_pending_tape(e) for e in self._regions[k][2].values()):
                continue
            for e in self._regions.pop(k)[2].values():
                if e.plan is not None:
                    e.plan.close()
                    e.plan = None
        return g, engines

    def forward(self, features: torch.Tensor, lat_lons: list, global_context: Optional[torch.Tensor] = None) -> torch.Tensor:
        if features.device.type != "cuda":
            _no_host_path("RegionalForecaster.forward")
        B, N = features.shape[0], features.shape[1]
        if N != len(lat_lons):
            raise ValueError(f"features has {N} rows per sample but lat_lons has {len(lat_lons)} coordinates")
        if features.shape[-1] < self.output_dim:
            raise RuntimeError(f"features needs at least output_dim ({self.output_dim}) channels for the residual add (:288)")
        train = _wants_grad(self, features)
        if train and self.train_precision is None:
            # (fail instead of returning a tensor that silently carries no graph)
            raise NotImplementedError("RegionalForecaster: training needs RegionalForecasterConfig.train_precision ('fp32_simt', 'fp32' "
                                      "or 'bf16'); call under torch.no_grad() or in eval() mode for inference")
        region, engines = self._region(lat_lons)
        if train:
            self.__dict__["_active"] = (region, engines)
            try:
                bindings = self._grad_bindings()
                out = _TrainFn.apply(self, features, None, bindings, *[q for _, _, q, _ in bindings])
            finally:
                self.__dict__["_active"] = None
        else:
            plan = engines["infer"].ensure(features.device, B, self._plan_named(region))
            f = features.detach().to(torch.float32).contiguous()
            out = torch.empty((B, N, self.output_dim), dtype=torch.float32, device=f.device)
            plan.forward(f, out)  # encoder -> processor -> decoder -> + features[..., :output_dim]
            _maybe_check(plan)
        if self.nudging is not None and global_context is not None:
            out = self.nudging(out, global_context.to(out.device), lat_lons)
        return out
