"""Loss boundary of the forward: a mirror of graph_weather/models/losses.py:9-94 (`NormalizedMSELoss`) whose reduction runs in
one HBM-bound CUDA kernel behind the C ABI (`gw_normalized_mse_loss_sum`).  Forward only (SURVEY 8(f) row 2); there is no CPU
fallback: tensors must live on a CUDA device.

Data-parallel use: every rank reduces its own batch shard to one double and the ranks all-reduce that scalar
(`forward(pred, target, group=...)`), instead of all-gathering the [B, N, F] outputs to evaluate the loss on every rank."""

from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _capi


def node_weights(lat_lons, num_nodes: int) -> np.ndarray:
    """cos(latitude) of every grid node exactly as the reference tiles it (losses.py:37-42, 78-88): the sorted unique
    latitudes, each repeated num_nodes // num_unique times in node order."""
    unique_lats = sorted(set(lat for lat, _ in lat_lons))
    w = np.array([np.cos(lat * np.pi / 180.0) for lat in unique_lats]).astype(np.float32)  # torch.tensor(..., dtype=float)
    num_unique = w.shape[0]
    num_lon = num_nodes // num_unique
    if num_unique * num_lon != num_nodes:  # the reference's reshape(1, num_nodes) fails the same way (losses.py:84)
        raise RuntimeError(f"shape '[1, {num_nodes}]' is invalid for input of size {num_unique * num_lon}")
    return np.repeat(w, num_lon)


class _LossFn(torch.autograd.Function):
    """value = sum_all_ranks(local sums) / rows;  d value / d pred = w(n) 2 (pred - target) inv_var / (F rows)  (one kernel)."""

    @staticmethod
    def forward(ctx, pred, target, crit, group, total_batch):
        s = crit.local_sum(pred, target)
        nodes = int(np.prod(pred.shape[1:-1]))
        rows = pred.shape[0] * nodes
        if group is not None or total_batch is not None:
            import torch.distributed as dist

            if total_batch is None:
                cnt = torch.tensor([float(pred.shape[0])], dtype=torch.float64, device=s.device)
                dist.all_reduce(cnt, op=dist.ReduceOp.SUM, group=group)
                total_batch = int(round(float(cnt.item())))
            s = s.clone()
            dist.all_reduce(s, op=dist.ReduceOp.SUM, group=group)
            rows = int(total_batch) * nodes
        ctx.crit, ctx.rows = crit, rows
        ctx.save_for_backward(pred.detach(), target.detach())
        return (s / rows).to(torch.float32).reshape(())

    @staticmethod
    def backward(ctx, grad_value):
        pred, target = ctx.saved_tensors
        return ctx.crit.grad_pred(pred, target, grad_value, 1.0 / ctx.rows), None, None, None, None


class NormalizedMSELoss(torch.nn.Module):
    """Variance-normalised, cos(lat)-weighted MSE (losses.py:9-94): same constructor, same `forward(pred, target)` value."""

    def __init__(self, feature_variance: list, lat_lons: list, device="cpu", normalize: bool = False):
        super().__init__()
        self.feature_variance = torch.tensor(feature_variance)
        assert not torch.isnan(self.feature_variance).any()
        self.lat_lons = [(float(a), float(b)) for a, b in lat_lons]
        unique_lats = sorted(set(lat for lat, _ in self.lat_lons))
        self.weights = torch.tensor([np.cos(lat * np.pi / 180.0) for lat in unique_lats], dtype=torch.float)
        self.normalize = normalize
        assert not torch.isnan(self.weights).any()
        self._dev = {}  # per device and shape: (inv_variance, node_weight), constant tables

    def _device_state(self, device, num_nodes, num_features):
        key = (str(device), num_nodes, num_features)
        if key not in self._dev:
            lib = _capi.load()
            inv = (1.0 / self.feature_variance.to(torch.float32)).reshape(-1).expand(num_features).to(device).contiguous()
            w = torch.from_numpy(node_weights(self.lat_lons, num_nodes)).to(device)
            self._dev[key] = (inv, w)
        return self._dev[key]

    def local_sum(self, pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """sum over the local rows of w(n) * mean_f(...): a new 1-element float64 device tensor.  The result and the kernel's
        workspace come from torch's allocator on the current stream, so calls on several streams do not share them."""
        if not (pred.is_cuda and target.is_cuda):
            raise RuntimeError("graph_weather_b200.NormalizedMSELoss runs on CUDA tensors only (no CPU fallback)")
        if pred.shape != target.shape:
            raise RuntimeError(f"pred {tuple(pred.shape)} and target {tuple(target.shape)} differ")
        lib = _capi.load()
        F = pred.shape[-1]
        B = pred.shape[0]
        num_nodes = int(np.prod(pred.shape[1:-1]))
        if self.normalize and self.feature_variance.numel() not in (1, F):  # a 1-element variance broadcasts (losses.py:70)
            raise RuntimeError("feature_variance does not match the feature dimension")
        p = pred.detach().to(torch.float32).contiguous()
        t = target.detach().to(torch.float32).contiguous()
        inv, w = self._device_state(pred.device, num_nodes, F)
        if B == 0:  # an empty batch shard (total_batch < world size) contributes nothing; the kernel is not launched
            return torch.zeros(1, dtype=torch.float64, device=pred.device)
        s = torch.empty(1, dtype=torch.float64, device=pred.device)
        ws = torch.empty(int(lib.gw_loss_workspace_bytes()), dtype=torch.uint8, device=pred.device)
        with torch.cuda.device(pred.device):
            st = torch.cuda.current_stream().cuda_stream
            _capi._check(lib.gw_normalized_mse_loss_sum(
                ctypes.c_void_p(p.data_ptr()), ctypes.c_void_p(t.data_ptr()),
                ctypes.c_void_p(inv.data_ptr()) if self.normalize else None, ctypes.c_void_p(w.data_ptr()), B, num_nodes, F,
                ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(st)))  # fmt: skip
        return s

    def grad_pred(self, pred: torch.Tensor, target: torch.Tensor, upstream: torch.Tensor, scale: float) -> torch.Tensor:
        """upstream * scale * d(local sum)/d pred as one kernel (gw_normalized_mse_loss_grad); `upstream` is a 0-d device tensor."""
        lib = _capi.load()
        B, F = pred.shape[0], pred.shape[-1]
        num_nodes = int(np.prod(pred.shape[1:-1]))
        p = pred.detach().to(torch.float32).contiguous()
        t = target.detach().to(torch.float32).contiguous()
        inv, w = self._device_state(pred.device, num_nodes, F)
        up = upstream.detach().to(device=pred.device, dtype=torch.float32).reshape(1).contiguous()
        g = torch.empty_like(p)
        if B == 0:
            return g
        with torch.cuda.device(pred.device):
            st = torch.cuda.current_stream().cuda_stream
            _capi._check(lib.gw_normalized_mse_loss_grad(
                ctypes.c_void_p(p.data_ptr()), ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(inv.data_ptr()) if self.normalize else None,
                ctypes.c_void_p(w.data_ptr()), B, num_nodes, F, ctypes.c_void_p(up.data_ptr()), float(scale), ctypes.c_void_p(g.data_ptr()),
                ctypes.c_void_p(st)))  # fmt: skip
        return g.reshape(pred.shape)

    def forward(self, pred: torch.Tensor, target: torch.Tensor, group=None, total_batch: int | None = None):
        """losses.py:46-94.  With `group` (torch.distributed), `pred` / `target` are this rank's batch shard and the result is
        the loss over the whole batch of `total_batch` samples: the ranks exchange one scalar.  Differentiable with respect
        to `pred` (training: `loss.backward()` runs gw_normalized_mse_loss_grad, then the model's CUDA backward)."""
        if torch.is_grad_enabled() and pred.requires_grad:
            return _LossFn.apply(pred, target, self, group, total_batch)
        s = self.local_sum(pred, target)
        nodes = int(np.prod(pred.shape[1:-1]))
        rows = pred.shape[0] * nodes
        if group is not None or total_batch is not None:
            import torch.distributed as dist

            if total_batch is None:  # derive the global batch from the shards: [sum, local batch] reduced together
                s = torch.cat([s, torch.tensor([float(pred.shape[0])], dtype=torch.float64, device=s.device)])
                dist.all_reduce(s, op=dist.ReduceOp.SUM, group=group)
                return (s[0] / (s[1] * nodes)).to(torch.float32).reshape(())
            s = s.clone()
            dist.all_reduce(s, op=dist.ReduceOp.SUM, group=group)
            rows = int(total_batch) * nodes
        out = (s / rows).to(torch.float32).reshape(())
        return out

    def checked(self, pred: torch.Tensor, target: torch.Tensor, **kw):
        """forward + the reference's NaN assertion on the result (losses.py:59-62,93 assert on every intermediate; a NaN in
        any of them makes the result NaN).  Synchronises; use in debugging runs."""
        out = self.forward(pred, target, **kw)
        assert not torch.isnan(out).any()
        return out
