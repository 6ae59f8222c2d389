"""The gradients of PhysicalConstraintLayer (constraint_layer.py:58-188, forecast.py:178-213): a torch restatement used as the
oracle of the CUDA backward (gw_constraint_backward; tests/test_gpu_constraint_training.py), held here to the reference's own
autograd gradients (tests/golden/constraint_grads.npz, made by tests/golden/make_constraint_grads.py).  CPU only."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.training  # autograd stays enabled


def grid_mapping(lat_lons):
    from graph_weather_b200.constraint import GridMapping

    m = GridMapping(lat_lons)
    return m.grid_shape, torch.from_numpy(m.cell), torch.from_numpy(m.last)


def restate_constraint(ctype, hr, lr, grid_shape, cell, last, exp_factor=1.0):
    """PhysicalConstraintLayer.forward with upsampling factor 1 in differentiable torch ops, in the dtype of hr / lr.
    hr, lr: graph [B, N, C] or grid [B, C, H, W]; returns graph [B, N, C].  The mapping's semantics are the reference's:
    graph_to_grid leaves empty cells 0 and the last node written to a shared cell wins (earlier writers get no gradient);
    grid_to_graph reads cell[n] for node n.  The constraint itself is constraint_layer.py:100-188, op for op."""
    H, W = grid_shape
    cells = torch.nonzero(last >= 0).flatten()
    writers = last[cells]

    def graph_to_grid(t):
        B, _, C = t.shape
        g = t.new_zeros((B, H * W, C)).index_copy(1, cells, t[:, writers, :])
        return g.permute(0, 2, 1).reshape(B, C, H, W)

    def grid_to_graph(t):
        B, C = t.shape[:2]
        return t.reshape(B, C, H * W)[:, :, cell].permute(0, 2, 1)

    if hr.dim() == 3:
        hr_grid, lr_grid = graph_to_grid(hr), graph_to_grid(lr)
    else:
        hr_grid, lr_grid = hr, lr
    if ctype == "additive":
        hg, lg = grid_to_graph(hr_grid), grid_to_graph(lr_grid)
        res = graph_to_grid(hg + (lg - hg.mean(dim=1, keepdim=True)))
    elif ctype == "multiplicative":
        hg, lg = grid_to_graph(hr_grid), grid_to_graph(lr_grid)
        res = graph_to_grid(hg * (lg.mean(dim=1, keepdim=True) / (hg.mean(dim=1, keepdim=True) + 1e-8)))
    elif ctype == "softmax":
        y = torch.exp(exp_factor * hr_grid)
        sum_y = y * 1  # AvgPool2d(1) * kernel area 1
        res = y * (lr_grid * (1 / sum_y))
    else:
        raise ValueError(ctype)
    return grid_to_graph(res)


def rows_to_grid(t, grid_shape):
    """The forecaster's rearrange(x, "b (h w) c -> b c h w") (forecast.py:236, 242)."""
    H, W = grid_shape
    return t.reshape(t.shape[0], H, W, t.shape[-1]).permute(0, 3, 1, 2)


def restate_grads(ctype, hr, lr, dy, grid_shape, cell, last, exp_factor=1.0, dtype=torch.float32, rows=False):
    """(out, d_hr, d_lr) of restate_constraint under torch.autograd in `dtype` (fp32: what the reference computes; fp64: ground
    truth).  rows=True: hr / lr are [B, H*W, C] rows that the forecaster's rearrange turns into grid tensors."""
    h = hr.detach().to(dtype).clone().requires_grad_(True)
    l_ = lr.detach().to(dtype).clone().requires_grad_(True)
    if rows:
        y = restate_constraint(ctype, rows_to_grid(h, grid_shape), rows_to_grid(l_, grid_shape), grid_shape, cell, last, exp_factor)
    else:
        y = restate_constraint(ctype, h, l_, grid_shape, cell, last, exp_factor)
    y.backward(dy.to(dtype))
    return y.detach(), h.grad, l_.grad


def load_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "constraint_grads.npz"))
    cfg = json.loads(str(z["config"]))
    return z, cfg


def fixture_inputs(z, cfg, ctype, form, grid_shape, cell, last):
    """hr, lr in the case's input form (the leaves the reference differentiated: rows for the "rows" form) and dy."""
    shift = cfg["multiplicative_shift"] if ctype == "multiplicative" else 0.0
    hr, lr = torch.from_numpy(z["hr"]) + shift, torch.from_numpy(z["lr"]) + shift
    if form == "grid":
        hr = restate_graph_to_grid(hr, grid_shape, last)
        lr = restate_graph_to_grid(lr, grid_shape, last)
    return hr, lr, torch.from_numpy(z["dy"])


def restate_graph_to_grid(t, grid_shape, last):
    H, W = grid_shape
    B, _, C = t.shape
    g = torch.zeros((B, H * W, C), dtype=t.dtype)
    ok = last >= 0
    g[:, ok] = t[:, last[ok]]
    return g.permute(0, 2, 1).reshape(B, C, H, W).contiguous()


def _case_ids(cfg):
    out = []
    for ctype, a in cfg["cases"]:
        for form in cfg["forms"]:
            out.append((ctype, a, form, f"{ctype}{'' if a == 1.0 else '_a' + str(a)}_{form}"))
    return out


def test_restatement_matches_the_reference_gradients(golden_dir):
    z, cfg = load_fixture(golden_dir)
    ll = [(a, b) for a in cfg["lats"] for b in cfg["lons"]]
    grid_shape, cell, last = grid_mapping(ll)
    assert (np.bincount(cell.numpy(), minlength=24) != 1).any()  # shared and empty cells exist
    cases = _case_ids(cfg)
    assert len(cases) == 12
    for ctype, a, form, key in cases:
        hr, lr, dy = fixture_inputs(z, cfg, ctype, form, grid_shape, cell, last)
        out, d_hr, d_lr = restate_grads(ctype, hr, lr, dy, grid_shape, cell, last, a, rows=form == "rows")
        ref_out, ref_hr, ref_lr = (torch.from_numpy(z[key + s]) for s in ("_out", "_d_hr", "_d_lr"))
        assert d_hr.shape == ref_hr.shape and d_lr.shape == ref_lr.shape, key
        # softmax: d_hr is analytically 0 (the layer returns lr up to rounding); its scale is that of d_lr
        scale_hr = float(ref_lr.abs().max()) if ctype == "softmax" else float(ref_hr.abs().max())
        for got, ref, scale, what in ((out, ref_out, float(ref_out.abs().max()), "out"), (d_hr, ref_hr, scale_hr, "d_hr"),
                                      (d_lr, ref_lr, float(ref_lr.abs().max()), "d_lr")):  # fmt: skip
            err = float((got - ref).abs().max()) / scale
            assert err <= 1e-6, (key, what, err)


def test_restatement_in_fp64_agrees(golden_dir):
    """The fp64 restatement (the ground truth of the GPU tests) is within fp32 rounding of the reference's fp32 gradients."""
    z, cfg = load_fixture(golden_dir)
    ll = [(a, b) for a in cfg["lats"] for b in cfg["lons"]]
    grid_shape, cell, last = grid_mapping(ll)
    for ctype, a, form, key in _case_ids(cfg):
        if ctype == "softmax":
            continue
        hr, lr, dy = fixture_inputs(z, cfg, ctype, form, grid_shape, cell, last)
        _, d_hr, d_lr = restate_grads(ctype, hr, lr, dy, grid_shape, cell, last, a, torch.float64, rows=form == "rows")
        for got, what in ((d_hr, "_d_hr"), (d_lr, "_d_lr")):
            ref = torch.from_numpy(z[key + what]).double()
            assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max()), (key, what)
