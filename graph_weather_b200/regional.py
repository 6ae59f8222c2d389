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

`forward_regions(features, regions, global_context)` runs B regions in one call, as one sample whose graphs are the disjoint union
of the regions' graphs (`_RegionBatch`: each region's point, cell and edge ids offset by the regions before it, its edge order
kept, so every per-target sum adds in the order of a single-region call).  The union is padded with inert rows up to a capacity
(points, cells, latent edges; powers of two, grown when a batch does not fit and never shrunk), so one plan per step kind serves
every batch within it: a new set of regions costs its host graphs, their upload and the inference plan's per-graph constants
(gw_plan_set_h3_nodes), never a new plan, a weight upload or a weight-image repack.  Output i is `forward` on region i alone.

Training (`train_precision`, as on the other wrappers): in train mode with autograd on, a forward runs the forecaster's CUDA
training step on training plans of the region (`use_checkpointing=True`: the bounded-memory step).  `h3_embeddings.grad` is
table-shaped, as the reference's: the region's rows at their cells, zero elsewhere.  A region's plans are kept while a backward
still needs one of their tapes, so the losses of more regions than the cache holds can be summed into one `backward()`.
`forward_regions` trains the same way on its union plans; a cell two regions share gets the sum of their rows' gradients, added
in a fixed order on the device (gw_segment_sum).  The union plan holds the graphs of its last call, so a backward after a later
`forward_regions` raises, and `forward_regions` refuses to train inside `multi_step()`.

Optional boundary nudging (:44-130): a distance-based relaxation prior plus a learned one-hidden-layer correction, blended
with a caller-supplied global forecast.  It is a [B, N, 2F+1] -> 1 element-wise tail outside the GNN; it runs as device
tensor ops (no kernels of this library), exactly the reference's arithmetic.
"""

from __future__ import annotations

import math
import time
from collections import OrderedDict
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import _capi, graphs, h3lite
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


def _pow2(n: int) -> int:
    return 1 << max(0, int(n) - 1).bit_length()


def _spread(n_items: int, first: int, n_slots: int) -> np.ndarray:
    """Slots first .. first + n_slots - 1 for n_items padding rows, non-decreasing and as even as the counts allow."""
    return (first + (np.arange(n_items, dtype=np.int64) * n_slots) // max(n_items, 1)).astype(np.int32)


class _RegionBatch:
    """B regions' graphs as one graph (the disjoint union), padded to a capacity `cap` of points (n_in = n_out = n_dec_edges),
    cells (n_mesh) and latent edges (n_lat_edges).  Region i's points, cells and edges follow those of regions 0 .. i-1, in its
    own order.  The padding is inert: padding points (zero features and edge attributes) feed, and are decoded from, padding cells
    only; padding cells (zero h3_nodes rows) carry only self loops with zero attributes.  No padding edge touches a real row, every
    row stays finite, and real rows see exactly their region's edges.  There is always at least one padding cell."""

    def __init__(self, graphs: list, cap: dict):
        self.graphs = graphs
        n = [g.n_obs for g in graphs]
        m = [g.n_mesh for g in graphs]
        e = [g.n_lat_edges for g in graphs]
        self.n_real, self.m_real, self.e_real = sum(n), sum(m), sum(e)
        P, C, E = cap["n_in"], cap["n_mesh"], cap["n_lat_edges"]
        if P < self.n_real or C <= self.m_real or E < max(self.e_real, 1):
            raise ValueError(f"capacity {cap} does not hold {self.n_real} points, {self.m_real} + 1 cells and {self.e_real} latent edges")
        self.cap = dict(cap)
        po = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
        co = np.concatenate([[0], np.cumsum(m)]).astype(np.int64)
        eo = np.concatenate([[0], np.cumsum(e)]).astype(np.int64)
        self.point_offsets, self.cell_offsets, self.edge_offsets = po, co, eo
        n_pad, c_pad, e_pad = P - self.n_real, C - self.m_real, E - self.e_real
        pad_cell = _spread(n_pad, self.m_real, c_pad)
        self.mesh_local = np.concatenate([g.mesh_local + co[i] for i, g in enumerate(graphs)] + [pad_cell]).astype(np.int32)
        self.enc_perm = np.concatenate([g.enc_perm + po[i] for i, g in enumerate(graphs)]
                                       + [np.arange(self.n_real, P)]).astype(np.int32)  # fmt: skip
        self.enc_ptr = np.zeros(C + 1, dtype=np.int32)
        np.cumsum(np.bincount(self.mesh_local, minlength=C), out=self.enc_ptr[1:])
        self.enc_attr = np.concatenate([g.enc_attr for g in graphs] + [np.zeros((n_pad, 2), np.float32)]).astype(np.float32)
        pad_self = _spread(e_pad, self.m_real, c_pad)
        self.lat_src = np.concatenate([g.lat_src + co[i] for i, g in enumerate(graphs)] + [pad_self]).astype(np.int32)
        self.lat_dst = np.concatenate([g.lat_dst + co[i] for i, g in enumerate(graphs)] + [pad_self]).astype(np.int32)
        self.lat_ptr = np.zeros(C + 1, dtype=np.int32)
        np.cumsum(np.bincount(self.lat_dst, minlength=C), out=self.lat_ptr[1:])
        self.lat_attr = np.concatenate([g.lat_attr for g in graphs] + [np.zeros((e_pad, 2), np.float32)]).astype(np.float32)
        self.dec_src = self.mesh_local
        self.dec_ptr = np.arange(P + 1, dtype=np.int32)
        self.h3_indices = np.concatenate([g.h3_indices for g in graphs]).astype(np.int64)  # cell of every real union row
        # the table gradient: union rows grouped by cell (stable: region order inside a cell), CSR over the whole table
        self.by_cell = np.argsort(self.h3_indices, kind="stable").astype(np.int32)
        self.n_obs = P

    def cell_ptr(self, n_cells: int) -> np.ndarray:
        ptr = np.zeros(n_cells + 1, dtype=np.int32)
        np.cumsum(np.bincount(self.h3_indices, minlength=n_cells), out=ptr[1:])
        return ptr

    def upload(self, plan, h3_rows):
        """The union's graphs, then its h3_nodes rows (which also recompute the constants on the new graphs).  The latent graph goes
        first: it unbinds the weights, so the encoder graph's upload does not recompute constants on the previous graphs."""
        plan.set_latent_graph(self.lat_src, self.lat_dst, self.lat_ptr, self.lat_attr)
        plan.set_encoder_graph(self.mesh_local, self.enc_perm, self.enc_ptr, self.enc_attr)
        plan.set_decoder_graph(self.dec_src, self.dec_ptr, self.enc_attr)
        plan.set_h3_nodes(h3_rows)


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
        self.__dict__["_active"] = None  # (graphs, engines) of the region (or _RegionBatch) of the current training forward
        # forward_regions: one engine per step kind ({"infer", False: taped, True: bounded}) over the union's capacity
        self.__dict__["_batch_engines"] = {}
        self.__dict__["_batch_cap"] = None
        self.__dict__["_zero_rows"] = None  # the h3_nodes table the union plans' weight uploads carry (its rows come per call)
        # forward_regions: host seconds of the last call's graph build, weight upload (only after a weight change) and graph upload
        self.__dict__["last_setup_s"] = None

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

    def _plan_named(self, region):
        out = []
        for k, v in self.state_dict(keep_vars=True).items():
            if k == "h3_embeddings" and isinstance(region, _RegionBatch):  # rows uploaded per call (_RegionBatch.upload)
                out.append(("encoder.h3_nodes", self._zero_rows))
                continue
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
            uploaders = [] if isinstance(region, _RegionBatch) else [region.upload]  # (the union's: forward_regions, every call)
            return _new_engine(engines["infer"].dims, self.train_precision, uploaders, train_only=bounded)

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
        if isinstance(self._active[0], _RegionBatch):
            return [(k, v, table, self._active[0].to_table) if k == "encoder.h3_nodes" else (k, v, v, None) for k, v in named]

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

    # ---- a batch of regions in one call ------------------------------------------------------------------------------------
    def _batch(self, regions: list, device) -> tuple:
        """The union of the regions' graphs, padded to the capacity (grown to the next power of two of each count when the union does
        not fit, never shrunk), with its h3_nodes rows, its table-gradient map and its rows on the device; and the batch engines.
        Returns (_RegionBatch, engines)."""
        t0 = time.perf_counter()
        graphs = [_RegionGraphs(self.graph_builder, r) for r in regions]
        need = dict(n_in=sum(g.n_obs for g in graphs), n_mesh=sum(g.n_mesh for g in graphs) + 1,
                    n_lat_edges=max(1, sum(g.n_lat_edges for g in graphs)))  # fmt: skip
        cap = self._batch_cap or {}
        if any(need[k] > cap.get(k, 0) for k in need):
            cap = {k: max(cap.get(k, 0), _pow2(need[k])) for k in need}
            cap.update(n_out=cap["n_in"], n_dec_edges=cap["n_in"])
            self.__dict__["_batch_cap"] = cap
        batch = _RegionBatch(graphs, cap)
        t1 = time.perf_counter()
        table = self.h3_embeddings
        if self._zero_rows is None or tuple(self._zero_rows.shape) != (cap["n_mesh"], table.shape[1]) or self._zero_rows.device != device:
            self.__dict__["_zero_rows"] = torch.zeros((cap["n_mesh"], table.shape[1]), dtype=torch.float32, device=device)
        engines = self._batch_engines
        if "infer" not in engines:
            engines["infer"] = _new_engine(dict(self._base_dims, n_in=1, n_out=1, n_mesh=2, n_lat_edges=1, n_dec_edges=1),
                                           self.config.precision, [])  # fmt: skip
        batch.h3_idx = torch.from_numpy(batch.h3_indices).to(device)
        batch.by_cell_d = torch.from_numpy(batch.by_cell).to(device)
        batch.cell_ptr_d = torch.from_numpy(batch.cell_ptr(table.shape[0])).to(device)

        def to_table(g):  # h3_nodes gradient [n_mesh, in_dim] -> table gradient: per cell, the sum of its rows in region order
            out = g.new_empty(table.shape)
            _capi.segment_sum(g.contiguous(), batch.by_cell_d, batch.cell_ptr_d, out)
            return out

        batch.to_table = to_table
        rows = torch.zeros((cap["n_mesh"], table.shape[1]), dtype=torch.float32, device=device)
        rows[: batch.m_real] = table.detach()[batch.h3_idx]
        batch.h3_rows = rows
        self.__dict__["last_setup_s"] = {"build": t1 - t0}
        return batch, engines

    def _batch_plan(self, eng, batch, device):
        """`eng`'s plan at the batch's capacity with the current weights, the union's graphs and rows uploaded."""
        t0 = time.perf_counter()
        plan = eng.ensure(device, 1, self._plan_named(batch), grow=batch.cap)
        t1 = time.perf_counter()
        batch.upload(plan, batch.h3_rows)
        self.last_setup_s.update(weights=t1 - t0, upload=time.perf_counter() - t1)
        return plan

    def forward_regions(self, features, regions: list, global_context=None):
        """B regions in one call: output i is `self(features[i:i+1], regions[i], global_context[i:i+1])[0]`, nudging included.

        regions: B coordinate lists (each as forward's lat_lons).  features: [B, N, F] when every region has N points, or a list of B
        tensors [N_i, F]; global_context: the output's form, or None.  Returns [B, N, output_dim] or a list of [N_i, output_dim], in
        the form of `features`.  In train mode with autograd on (and a train_precision) it is differentiable: the gradients of a loss
        over its outputs are those of the sum of the B single-region steps, up to the order of float sums.  The regions run as one
        graph on one plan per step kind, kept from call to call (see the module docstring).  Training inside `multi_step()` raises:
        the plan holds one set of regions, so only the last call's forward can be differentiated."""
        stacked = torch.is_tensor(features)
        feats = list(features.unbind(0)) if stacked else list(features)
        if len(feats) != len(regions) or not regions:
            raise ValueError(f"{len(feats)} feature sets for {len(regions)} regions (need one per region, at least one)")
        device = feats[0].device
        if device.type != "cuda":
            _no_host_path("RegionalForecaster.forward_regions")
        for f, r in zip(feats, regions):
            if f.dim() != 2 or f.shape[0] != len(r):
                raise ValueError(f"a region's features must be [{len(r)}, F] (one row per coordinate), got {tuple(f.shape)}")
            if f.shape[1] < self.output_dim:
                raise RuntimeError(f"features needs at least output_dim ({self.output_dim}) channels for the residual add (:288)")
        F = feats[0].shape[1]
        if any(f.shape[1] != F for f in feats):
            raise ValueError("every region's features need the same number of channels")
        train = torch.is_grad_enabled() and self.training and (any(f.requires_grad for f in feats)
                                                               or any(q.requires_grad for q in self.parameters()))  # fmt: skip
        if train and self.train_precision is None:
            raise NotImplementedError("RegionalForecaster: training needs RegionalForecasterConfig.train_precision ('fp32_simt', 'fp32' "
                                      "or 'bf16'); call under torch.no_grad() or in eval() mode for inference")
        if train and self.__dict__.get("_multi_step", 0):
            raise NotImplementedError("RegionalForecaster.forward_regions inside multi_step(): the union graph a training forward runs on "
                                      "belongs to the plan, not to the forward, so several calls cannot stay differentiable at once")
        batch, engines = self._batch(regions, device)
        P = batch.n_obs
        pad = feats[0].new_zeros((P - batch.n_real, F))
        union = torch.cat([f.to(torch.float32) for f in feats] + [pad.to(torch.float32)])[None]
        if train:
            self.__dict__["_active"] = (batch, engines)
            try:
                self._batch_plan(self._training_engine(), batch, device)
                bindings = self._grad_bindings()
                out = _TrainFn.apply(self, union, None, bindings, *[q for _, _, q, _ in bindings])
            finally:
                self.__dict__["_active"] = None
        else:
            plan = self._batch_plan(engines["infer"], batch, device)
            out = torch.empty((1, P, self.output_dim), dtype=torch.float32, device=device)
            plan.forward(union.detach().contiguous(), out)
            _maybe_check(plan)
        po = batch.point_offsets
        outs = [out[0, po[i]: po[i + 1]] for i in range(len(regions))]
        if self.nudging is not None and global_context is not None:
            gcs = list(global_context.unbind(0)) if torch.is_tensor(global_context) else list(global_context)
            if len(gcs) != len(regions):
                raise ValueError(f"{len(gcs)} global contexts for {len(regions)} regions")
            outs = [self.nudging(o[None], g.to(o.device)[None], r)[0] for o, g, r in zip(outs, gcs, regions)]
        return torch.stack(outs) if stacked else outs
