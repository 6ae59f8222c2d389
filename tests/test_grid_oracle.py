"""The chunked oracle (tests/grid_oracle.py) against the unchunked one (oracle/restate.py, tests/training_oracle.py) and the
reference's own output, on the CPU: 10 degrees, batch 2, chunks of 37 points, which cut mesh cells and decoder point groups at odd
places and give 18 chunks per stage."""
import os

import numpy as np
import pytest
import torch

import grid_oracle
from oracle import restate, weights
from training_oracle import forecaster_case, grid, rel_max

pytestmark = pytest.mark.training

CHUNK = 37
# unequal node / edge / hidden widths, 1 and 3 hidden layers (tests/test_gpu_model_shapes.py's "mixed")
MIXED = dict(node_dim=48, edge_dim=80, hidden_dim_processor_node=96, hidden_dim_processor_edge=64, hidden_layers_processor_node=1,
             hidden_layers_processor_edge=3, hidden_dim_decoder=40, hidden_layers_decoder=3, feature_dim=7, aux_dim=5, num_blocks=2)
SHAPES = {"default": {}, "mixed": MIXED}


def _oracle_kw(kw):
    return dict(feature_dim=kw.get("feature_dim", 78), num_blocks=kw.get("num_blocks", 9),
                hl_node=kw.get("hidden_layers_processor_node", 2), hl_edge=kw.get("hidden_layers_processor_edge", 2),
                hl_dec=kw.get("hidden_layers_decoder", 2))  # fmt: skip


def _chunked_step(name, dtype):
    kw = SHAPES[name]
    ll, sd, x, target, var, ref32, ref64 = forecaster_case(10, 2, 21, **kw)
    ours = grid_oracle.train_step(sd, grid_oracle.build_graphs(ll), x, target, var, ll, dtype, "cpu", CHUNK, **_oracle_kw(kw))
    return ours, ref32, ref64, len(weights.forecaster_shapes(**kw))


@pytest.mark.parametrize("name", list(SHAPES))
def test_fp64_step_equals_the_unchunked_oracle(name):
    (out, loss, gx, grads), _, ref64, n_params = _chunked_step(name, torch.float64)
    assert len(grads) == n_params and grads.keys() == ref64[3].keys()
    errs = {"out": rel_max(out, ref64[0]), "loss": abs(loss - ref64[1]) / abs(ref64[1]), "features": rel_max(gx, ref64[2])}
    errs.update({k: rel_max(g, ref64[3][k]) for k, g in grads.items()})
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"{name} fp64: worst max-relative difference to the unchunked oracle {worst[1]:.2e} ({worst[0]})")
    assert worst[1] < 1e-12, worst


@pytest.mark.parametrize("name", list(SHAPES))
def test_fp32_step_is_as_accurate_as_the_unchunked_oracle(name):
    """In fp32 the chunks reorder the sums over the encoder's points and over the samples of the edge encoders, so the two fp32
    oracles differ by rounding: each of their results is held to its error against fp64, which must stay within 2x the unchunked
    fp32 oracle's + 1e-6 (measured on the CPU: no error more than 1.7e-7 above the unchunked oracle's); the output and the loss
    to 1e-6 of the unchunked fp32 oracle's (measured: the output bit for bit, the loss 1.1e-7)."""
    (out, loss, gx, grads), ref32, ref64, _ = _chunked_step(name, torch.float32)
    d_out, d_loss = float((out - ref32[0]).abs().max()), abs(loss - ref32[1]) / abs(ref32[1])
    print(f"{name} fp32: output {d_out:.2e} max-abs, loss {d_loss:.2e} relative to the unchunked fp32 oracle")
    assert d_out < 1e-6 and d_loss < 1e-6
    pairs = [("features", gx, ref32[2], ref64[2])] + [(k, g, ref32[3][k], ref64[3][k]) for k, g in grads.items()]
    fails, worst = [], (0.0, "")
    for k, ours, theirs, truth in pairs:
        e, e_ref = rel_max(ours, truth), rel_max(theirs, truth)
        worst = max(worst, (e - e_ref, k))
        if not e < 2 * e_ref + 1e-6:
            fails.append((k, e, e_ref))
    print(f"{name} fp32: largest excess over the unchunked oracle's error against fp64: {worst[0]:.2e} ({worst[1]})")
    assert not fails, fails


def test_fp32_forward_matches_the_reference_fixture(golden_dir):
    """The reference's own output (tests/golden/forecaster_10deg_b2.npz) at test_oracle.py's tolerance."""
    import json

    z = np.load(os.path.join(golden_dir, "forecaster_10deg_b2.npz"))
    cfg = json.loads(str(z["config"]))
    assert not cfg["kw"]
    ll = grid(cfg["step"])
    sd = weights.make_state_dict(weights.forecaster_shapes(), cfg["seed"])
    x = weights.make_features(cfg["batch"], len(ll), 102, cfg["seed"])
    out = grid_oracle.forward(sd, grid_oracle.build_graphs(ll), x, torch.float32, "cpu", CHUNK)
    err = float(np.abs(out.numpy() - z["out"]).max())
    print(f"chunked fp32 forward: max|oracle - reference| = {err:.2e}")
    assert err < 1e-5


@pytest.mark.parametrize("name", list(SHAPES))
def test_forward_equals_the_unchunked_forward(name):
    """forward() in fp64 against restate.forecaster_forward in fp64 (1e-12 relative), and in fp32 against it in fp32."""
    kw = SHAPES[name]
    ll, sd, x = forecaster_case(10, 2, 21, **kw)[:3]
    okw = _oracle_kw(kw)
    g = restate.build_forecaster_graphs(ll)
    gg = grid_oracle.build_graphs(ll)
    for dtype, bar in ((torch.float64, 1e-12), (torch.float32, 1e-6)):
        sd_t = {k: v.to(dtype) for k, v in sd.items()}
        g_t = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in g.items()}
        ref = restate.forecaster_forward(sd_t, g_t, x.to(dtype), okw["feature_dim"], okw["num_blocks"], okw["hl_node"], okw["hl_edge"],
                                         okw["hl_dec"])  # fmt: skip
        out = grid_oracle.forward(sd, gg, x, dtype, "cpu", CHUNK, **okw)
        err = rel_max(out, ref)
        print(f"{name} {dtype}: forward max-relative difference {err:.2e}")
        assert out.dtype == dtype and err < bar


def test_tf32_setting_is_restored():
    before = (torch.backends.cuda.matmul.allow_tf32, torch.get_float32_matmul_precision())
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        with grid_oracle.exact_fp32():
            assert not torch.backends.cuda.matmul.allow_tf32 and torch.get_float32_matmul_precision() == "highest"
        assert torch.backends.cuda.matmul.allow_tf32
    finally:
        torch.set_float32_matmul_precision(before[1])
        torch.backends.cuda.matmul.allow_tf32 = before[0]
