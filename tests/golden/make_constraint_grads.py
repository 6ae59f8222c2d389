"""Generates tests/golden/constraint_grads.npz: the gradients of the reference's OWN PhysicalConstraintLayer
(constraint_layer.py, located by oracle/ref_shims.py) under torch.autograd, on the irregular 4 x 6 grid of make_golden.py's
constraint case (unevenly spaced latitudes: grid row 0 holds two nodes per cell, grid row 2 none).  Runs only where the
reference sources are present; the fixture travels with the repository.

    python tests/golden/make_constraint_grads.py

For each case it stores the inputs hr, lr, the upstream gradient dy and the reference's d_hr, d_lr, for three input forms:
    graph    hr, lr [B, N, C] passed as graph tensors (the layer's graph_to_grid: last writer wins a shared cell)
    grid     graph_to_grid(hr), graph_to_grid(lr) [B, C, H, W] passed as grid tensors
    rows     the forecaster's own `rearrange(x, "b (h w) c -> b c h w")` of [B, N, C] rows (forecast.py:236-246)
"""

import json
import os
import sys

import numpy as np
import torch
from einops import rearrange

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_shims  # noqa: E402

LATS, LONS = [-80.0, -75.0, 10.0, 80.0], [0.0, 50.0, 130.0, 200.0, 290.0, 350.0]
CASES = [("additive", 1.0), ("multiplicative", 1.0), ("softmax", 1.0), ("softmax", 0.5)]
FORMS = ("graph", "grid", "rows")


def case_name(ctype, exp_factor, form):
    return f"{ctype}{'' if exp_factor == 1.0 else '_a' + str(exp_factor)}_{form}"


def main(name="constraint_grads"):
    R = ref_shims.load_reference()
    ll = [(a, b) for a in LATS for b in LONS]
    H, W = len(LATS), len(LONS)
    rng = np.random.Generator(np.random.PCG64(31))
    B, N, C = 2, len(ll), 3
    # multiplicative: the inputs are shifted away from zero mean (as physical fields are), so the ratio is well conditioned
    hr = rng.standard_normal((B, N, C)).astype(np.float32)
    lr = rng.standard_normal((B, N, C)).astype(np.float32)
    dy = rng.standard_normal((B, N, C)).astype(np.float32)
    out = dict(hr=hr, lr=lr, dy=dy)
    for ctype, a in CASES:
        model = R.GraphWeatherForecaster(ll, constraint_type=ctype, feature_dim=4, aux_dim=0, output_dim=4)
        layer = model.constraint
        layer.exp_factor = a
        shift = 3.0 if ctype == "multiplicative" else 0.0
        for form in FORMS:
            h0 = torch.from_numpy(hr + shift)
            l0 = torch.from_numpy(lr + shift)
            if form == "grid":
                h0, l0 = model.graph_to_grid(h0), model.graph_to_grid(l0)
            h, l = h0.clone().requires_grad_(True), l0.clone().requires_grad_(True)
            if form == "rows":
                y = layer(rearrange(h, "b (h w) c -> b c h w", h=H, w=W), rearrange(l, "b (h w) c -> b c h w", h=H, w=W))
            else:
                y = layer(h, l)
            y.backward(torch.from_numpy(dy))
            k = case_name(ctype, a, form)
            out[k + "_out"] = y.detach().numpy()
            out[k + "_d_hr"] = h.grad.numpy()
            out[k + "_d_lr"] = l.grad.numpy()
            print(k, "max|d_hr|", float(h.grad.abs().max()), "max|d_lr|", float(l.grad.abs().max()))
    cfg = dict(lats=LATS, lons=LONS, seed=31, multiplicative_shift=3.0, cases=[[c, a] for c, a in CASES], forms=list(FORMS))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), config=json.dumps(cfg), **out)


if __name__ == "__main__":
    main()
