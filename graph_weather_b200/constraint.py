"""PhysicalConstraintLayer (graph_weather/models/layers/constraint_layer.py:12-188) and the grid <-> graph mapping of
GraphWeatherForecaster (forecast.py:178-213) for the CUDA path.

The reference moves every tensor through Python loops over the nodes (`graph_to_grid` / `grid_to_graph`, O(N) Python per
call) and a handful of eager ops.  Here the mapping is two precomputed index vectors and the constraint itself is
`gw_constraint_apply` (csrc/gw_constraint.cu): column means + one element-wise pass on the device, no layout copies.
The backward (training, and any call on tensors that require grad) is `gw_constraint_backward`: column sums of the upstream
gradient, then one pass that sums each row's nodes through the CSR of the row index.
Only `upsampling_factor == 1` exists in the reference's forecaster (forecast.py:166) and only that is built."""

from __future__ import annotations

import ctypes

import numpy as np
import torch
from torch import nn

from . import _capi

CONSTRAINT_TYPES = {"additive": 1, "multiplicative": 2, "softmax": 3}


class GridMapping:
    """node -> (row, col) exactly as forecast.py:178-192 computes it (same float expression, same int() truncation), plus the
    two index vectors its loops amount to:
        cell[n]  flat grid cell of node n                      grid_to_graph: graph[n] = grid[cell[n]]          (:205-213)
        last[c]  the last node written to cell c, or -1       graph_to_grid: grid[c] = graph[last[c]] or 0     (:194-203)"""

    def __init__(self, lat_lons):
        ll = np.asarray([(float(a), float(b)) for a, b in lat_lons], dtype=np.float64).reshape(-1, 2)
        lats, lons = np.unique(ll[:, 0]), np.unique(ll[:, 1])
        self.grid_shape = (int(lats.size), int(lons.size))
        H, W = self.grid_shape
        with np.errstate(invalid="ignore", divide="ignore"):
            r = (ll[:, 0] - lats.min()) / (lats.max() - lats.min()) * (H - 1)
            c = (ll[:, 1] - lons.min()) / (lons.max() - lons.min()) * (W - 1)
        if not (np.isfinite(r).all() and np.isfinite(c).all()):  # a single latitude or longitude: the reference divides by zero
            raise ZeroDivisionError("float division by zero")
        row, col = r.astype(np.int64), c.astype(np.int64)  # int(): truncation toward zero
        self.node_to_grid = list(zip(row.tolist(), col.tolist()))
        self.cell = (row * W + col).astype(np.int64)
        last = np.full(H * W, -1, dtype=np.int64)
        last[self.cell] = np.arange(ll.shape[0])  # duplicate cells: numpy keeps the last assignment, like the reference's loop
        self.last = last
        self._dev = {}

    def tensors(self, device):
        key = str(device)
        if key not in self._dev:
            cell = torch.from_numpy(self.cell).to(device)
            last = torch.from_numpy(self.last).to(device)
            self._dev[key] = (cell, last)
        return self._dev[key]

    def graph_to_grid(self, graph_tensor: torch.Tensor) -> torch.Tensor:
        """[B, N, C] -> [B, C, H, W]  (forecast.py:194-203): cells no node maps to stay zero; the last node wins a shared cell."""
        B, _, C = graph_tensor.shape
        H, W = self.grid_shape
        cell, last = self.tensors(graph_tensor.device)
        rows = graph_tensor[:, last.clamp(min=0), :] * (last >= 0).to(graph_tensor.dtype)[None, :, None]
        return rows.permute(0, 2, 1).reshape(B, C, H, W).contiguous()

    def grid_to_graph(self, grid_tensor: torch.Tensor) -> torch.Tensor:
        """[B, C, H, W] -> [B, H*W, C]  (forecast.py:205-213)."""
        B, C, H, W = grid_tensor.shape
        cell, _ = self.tensors(grid_tensor.device)
        if cell.numel() != H * W:  # the reference allocates H*W rows and indexes them by node: mismatching sizes fail the same way
            raise IndexError(f"index {cell.numel() - 1} is out of bounds for dimension 1 with size {H * W}")
        return grid_tensor.reshape(B, C, H * W)[:, :, cell].permute(0, 2, 1).contiguous()


class PhysicalConstraintLayer(nn.Module):
    """Same constructor and call as the reference layer (constraint_layer.py:34-102): `forward(hr, lr)` takes graph ([B, N, C])
    or grid ([B, C, H, W]) tensors and returns the adjusted output in graph format."""

    def __init__(self, model, grid_shape, upsampling_factor, constraint_type="none", exp_factor=1.0):
        super().__init__()
        self.__dict__["model"] = model  # (not registered as a sub-module: the reference's back-reference creates a cycle)
        self.constraint_type = constraint_type
        self.grid_shape = tuple(grid_shape)
        self.exp_factor = exp_factor
        self.upsampling_factor = upsampling_factor
        if upsampling_factor != 1:
            raise NotImplementedError("upsampling_factor != 1: GraphWeatherForecaster only ever uses 1 (forecast.py:166)")

    def _prepare(self, hr: torch.Tensor, lr: torch.Tensor):
        """The float32 rows the kernels read: hr contiguous, lr with unit column stride and rows of one stride."""
        if self.constraint_type not in CONSTRAINT_TYPES:
            raise ValueError(f"Unknown constraint type: {self.constraint_type}")
        if not hr.is_cuda:
            raise RuntimeError("graph_weather_b200.PhysicalConstraintLayer runs on CUDA tensors only (no CPU fallback)")
        N = hr.shape[1]
        hr = hr.detach().to(torch.float32).contiguous()
        lr = lr.detach().to(torch.float32)
        if lr.stride(-1) != 1 or lr.stride(0) != N * lr.stride(1):
            lr = lr.contiguous()
        return hr, lr

    def apply_rows(self, hr: torch.Tensor, lr: torch.Tensor, src: torch.Tensor, lr_channels: int) -> torch.Tensor:
        """hr [B, N, C] rows, lr [B, N, >= lr_channels] rows (any row stride), src [N] int32 -> constrained rows [B, N, C].
        No autograd: `constrain_rows` is the differentiable form."""
        hr, lr = self._prepare(hr, lr)
        return self._launch_apply(hr, lr, src, lr_channels)

    def _launch_apply(self, hr, lr, src, lr_channels):
        lib = _capi.load()
        B, N, C = hr.shape
        out = torch.empty_like(hr)
        ws = torch.empty(int(lib.gw_constraint_workspace_bytes(B, C)), dtype=torch.uint8, device=hr.device)  # (per call: stream-ordered)
        with torch.cuda.device(hr.device):
            st = torch.cuda.current_stream().cuda_stream
            _capi._check(lib.gw_constraint_apply(
                CONSTRAINT_TYPES[self.constraint_type], ctypes.c_void_p(hr.data_ptr()), ctypes.c_void_p(lr.data_ptr()), int(lr.stride(1)),
                int(lr_channels), ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(out.data_ptr()), B, N, C, float(self.exp_factor),
                ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(st)))  # fmt: skip
        return out

    def _backward(self, dy, hr, lr, src, need_lr):
        """gw_constraint_backward: d loss / d out [B, N, C] -> (d_hr [B, N, C], d_lr [B, N, C] or None)."""
        lib = _capi.load()
        B, N, C = hr.shape
        dy = dy.to(torch.float32).contiguous()
        d_hr = torch.empty_like(hr)
        d_lr = torch.empty_like(hr) if need_lr else None
        ws = torch.empty(int(lib.gw_constraint_backward_workspace_bytes(B, N, C)), dtype=torch.uint8, device=hr.device)
        with torch.cuda.device(hr.device):
            st = torch.cuda.current_stream().cuda_stream
            _capi._check(lib.gw_constraint_backward(
                CONSTRAINT_TYPES[self.constraint_type], ctypes.c_void_p(dy.data_ptr()), ctypes.c_void_p(hr.data_ptr()),
                ctypes.c_void_p(lr.data_ptr()), int(lr.stride(1)), int(lr.shape[-1]), ctypes.c_void_p(src.data_ptr()),
                ctypes.c_void_p(d_hr.data_ptr()), ctypes.c_void_p(d_lr.data_ptr() if d_lr is not None else None), B, N, C,
                float(self.exp_factor), ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(st)))  # fmt: skip
        return d_hr, d_lr

    def constrain_rows(self, hr: torch.Tensor, lr: torch.Tensor, src: torch.Tensor) -> torch.Tensor:
        """apply_rows with lr_channels = lr.shape[-1], differentiable in hr and lr (gw_constraint_backward)."""
        return _ConstraintFn.apply(self, hr, lr, src)

    def forward(self, hr_graph: torch.Tensor, lr_graph: torch.Tensor) -> torch.Tensor:
        m: GridMapping = self.model._grid_mapping
        cell, last = m.tensors(hr_graph.device)
        if hr_graph.dim() == 3:
            # graph format goes through graph_to_grid first (constraint_layer.py:74-77): node n then sees the row of the last
            # node that shares its cell
            src = last[cell].to(torch.int32)
            hr, lr = hr_graph, lr_graph
        elif hr_graph.dim() == 4:
            _, _, H, W = hr_graph.shape
            if (H, W) != self.grid_shape:
                raise ValueError(f"Expected spatial dimensions {self.grid_shape}, got {(H, W)}")
            src = cell.to(torch.int32)
            hr = hr_graph.reshape(hr_graph.shape[0], hr_graph.shape[1], H * W).permute(0, 2, 1)
            lr = lr_graph.reshape(lr_graph.shape[0], lr_graph.shape[1], H * W).permute(0, 2, 1).contiguous()
        else:
            raise ValueError("Input tensor must be either 3D (graph) or 4D (grid).")
        if torch.is_grad_enabled() and (hr.requires_grad or lr.requires_grad):
            return self.constrain_rows(hr, lr, src.contiguous())
        return self.apply_rows(hr, lr, src.contiguous(), lr.shape[-1])


class _ConstraintFn(torch.autograd.Function):
    """autograd node of PhysicalConstraintLayer on rows: forward = gw_constraint_apply, backward = gw_constraint_backward (the
    gradients of hr and of lr, the latter only when lr requires it).  Reshapes and permutes around it are torch's."""

    @staticmethod
    def forward(ctx, layer, hr, lr, src):
        hr32, lr32 = layer._prepare(hr, lr)
        out = layer._launch_apply(hr32, lr32, src, lr32.shape[-1])
        ctx.layer, ctx.dtypes = layer, (hr.dtype, lr.dtype)
        ctx.save_for_backward(hr32, lr32, src)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        hr32, lr32, src = ctx.saved_tensors
        d_hr, d_lr = ctx.layer._backward(grad_out, hr32, lr32, src, ctx.needs_input_grad[2])
        return (None, d_hr.to(ctx.dtypes[0]) if ctx.needs_input_grad[1] else None,
                d_lr.to(ctx.dtypes[1]) if d_lr is not None else None, None)  # fmt: skip
