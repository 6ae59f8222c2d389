"""Pins the CPU restatement (oracle/restate.py) to outputs of the reference's own unmodified code (tests/golden/*.npz)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate, weights


def _grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


@pytest.mark.parametrize("name", ["forecaster_10deg_b2", "forecaster_small_hidden64", "forecaster_5deg_b1", "forecaster_mixed_shapes"])
def test_restatement_matches_reference(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = json.loads(str(z["config"]))
    kw = cfg["kw"]
    ll = _grid(cfg["step"])
    g = restate.build_forecaster_graphs(ll)
    sd = weights.make_state_dict(weights.forecaster_shapes(**kw), cfg["seed"])
    fdim = kw.get("feature_dim", 78)
    x = weights.make_features(cfg["batch"], len(ll), fdim + kw.get("aux_dim", 24), cfg["seed"])
    nb = kw.get("num_blocks", 9)
    hl = dict(hl_node=kw.get("hidden_layers_processor_node", 2), hl_edge=kw.get("hidden_layers_processor_edge", 2))
    with torch.no_grad():
        enc_x, ei, ea = restate.encoder_forward(sd, g, x, **hl)
        proc_x = restate.processor_forward(sd, enc_x, ei, ea, nb, **hl)
    out = restate.forecaster_forward(sd, g, x, feature_dim=fdim, num_blocks=nb, hl_dec=kw.get("hidden_layers_decoder", 2), **hl)
    # same ops in the same order on the same machine class: expect (near) bit equality; 1e-5 is the tolerance the
    # reference's own equivalence tests use (tests/models/layers/test_efficient_batching.py:53,91)
    assert np.abs(enc_x.numpy()[::53] - z["enc_x_sub"]).max() < 1e-5
    assert np.abs(proc_x.numpy()[::53] - z["proc_x_sub"]).max() < 1e-5
    assert out.shape == z["out"].shape
    assert np.abs(out.numpy() - z["out"]).max() < 1e-5


def test_assimilator_restatement_matches_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "assimilator_readme.npz"))
    cfg = json.loads(str(z["config"]))
    g = restate.build_assimilator_graphs(_grid(cfg["step"]))
    sd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=cfg["analysis_dim"]), cfg["seed"])
    obs = torch.from_numpy(z["obs"])
    x = weights.make_features(1, obs.shape[0], 2, cfg["seed"])
    out = restate.assimilator_forward(sd, g, x, obs)
    assert np.abs(out.numpy() - z["out"]).max() < 1e-5


def test_graphcast_restatement_matches_reference(golden_dir):
    """graphcast/model.py wrapper: Decoder with hidden 256 and the full input as residual; replicated == efficient batching."""
    z = np.load(os.path.join(golden_dir, "graphcast_10deg_b2.npz"))
    cfg = json.loads(str(z["config"]))
    ll = _grid(cfg["step"])
    g = restate.build_forecaster_graphs(ll)
    sd = weights.make_state_dict(weights.forecaster_shapes(feature_dim=78, aux_dim=0, hidden_dim_decoder=256), cfg["seed"])
    x = weights.make_features(cfg["batch"], len(ll), 78, cfg["seed"])
    out = restate.forecaster_forward(sd, g, x, feature_dim=78)
    assert np.abs(out.numpy() - z["out"]).max() < 1e-5
    assert np.abs(z["out"] - z["out_efficient"]).max() < 1e-4  # the reference's own tolerance, test_efficient_batching.py:145


def _loss_case(golden_dir):
    z = np.load(os.path.join(golden_dir, "loss_5deg.npz"))
    cfg = json.loads(str(z["config"]))
    lat_lons = [(float(a), float(b)) for a in range(-90, 90, cfg["step"]) for b in range(0, 360, cfg["step"])]
    rng = np.random.Generator(np.random.PCG64(cfg["seed"]))
    shape = (cfg["batch"], len(lat_lons), cfg["features"])
    pred = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    target = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    var = rng.uniform(0.5, 2.0, cfg["features"]).astype(np.float32)
    assert np.array_equal(var, z["feature_variance"])
    return z, lat_lons, pred, target, var


def test_loss_restatement_matches_reference(golden_dir):
    """oracle.restate.normalized_mse_loss vs NormalizedMSELoss of the reference's own losses.py (fixture made by make_golden.py)."""
    z, lat_lons, pred, target, var = _loss_case(golden_dir)
    for normalize, key in ((False, "loss_plain"), (True, "loss_normalized")):
        got = float(restate.normalized_mse_loss(pred, target, var.tolist(), lat_lons, normalize))
        assert abs(got - float(z[key])) <= 1e-6 * abs(float(z[key]))


def test_loss_shard_sums_compose(golden_dir):
    """The multi-GPU form of the loss: per-shard sums of w(n) * mean_f(...) added and divided by the global row count equal the
    loss over the whole batch (what graph_weather_b200.NormalizedMSELoss.forward(group=...) exchanges is one scalar per rank)."""
    from graph_weather_b200.losses import node_weights

    z, lat_lons, pred, target, var = _loss_case(golden_dir)
    w = torch.from_numpy(node_weights(lat_lons, pred.shape[1])).double()
    per_row = (((pred - target) ** 2) / torch.from_numpy(var)).mean(-1).double() * w
    total = float(per_row[:2].sum() + per_row[2:].sum()) / (pred.shape[0] * pred.shape[1])
    assert abs(total - float(z["loss_normalized"])) <= 1e-6 * float(z["loss_normalized"])
    with pytest.raises(RuntimeError):
        node_weights(lat_lons, pred.shape[1] + 1)
