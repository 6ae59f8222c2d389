"""-m gpu: GraphCast trains.  `model(features)` in train mode with autograd on, a loss and `loss.backward()` run the CUDA training
step (the forecaster's, with the full input as the residual); the checkpoint strategies of GraphCastConfig choose between the taped
step and the bounded-memory one.

  * one step (10 degrees, batch 2) against torch.autograd on the CPU oracle (encoder -> processor -> decoder + x), in fp32 and in
    fp64, with the bars of tests/test_gpu_training.py (fp32_simt) and tests/test_gpu_lean_training.py (fp32, bf16);
  * every GraphCastConfig strategy, with efficient_batching off and on, against the taped step: the same forward bit for bit and
    gradients within 1e-5 norm-relative, with many small chunks;
  * the reference's own two training tests (tests/models/test_gradient_checkpointing.py), restated on the GPU;
  * an SGD step lowers the loss, inference is untouched by training, switching strategy between a forward and its backward raises."""
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import check_bf16_bars, check_fp32_bars, forecaster_case, grid, rel_norm, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]

STRATEGIES = ["no_checkpointing", "full_checkpointing", "balanced_checkpointing", "processor_only_checkpointing",
              "fine_grained_checkpointing"]  # fmt: skip
BOUNDED = {"full_checkpointing", "balanced_checkpointing"}


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture(scope="module")
def case10():
    """GraphCast's default model (78 -> 78, hidden 256, 9 blocks) on the 10-degree grid, batch 2, and its oracle step (fp32 and
    fp64): GraphCast is the forecaster's network with no auxiliary features and a 256-wide decoder.  Seed 21, as in
    tests/test_gpu_training.py.  The fp32_simt bar admits no ReLU-mask flip between this step and the fp32 oracle: with seed 31
    one hidden unit of the last processor block sits at the edge of its mask, and the forecaster of the same shapes misses the
    bar on the same unit as GraphCast does (block 8's node-MLP layer 0, 5e-4 against 2e-7)."""
    return forecaster_case(10, 2, 21, feature_dim=78, aux_dim=0, hidden_dim_decoder=256)


def _model(ll, sd, tp="fp32_simt", strategy=None, **kw):
    from graph_weather_b200 import GraphCast, GraphCastConfig

    model = GraphCast(ll, train_precision=tp, **kw).cuda().train()
    model.load_state_dict(sd)
    if strategy is not None:
        getattr(GraphCastConfig, strategy)(model)
    return model


def _step(model, ll, x, target, var, feat_grad=True):
    from graph_weather_b200 import NormalizedMSELoss

    return train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target, feat_grad=feat_grad)


@pytest.mark.parametrize("strategy", ["no_checkpointing", "balanced_checkpointing"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_gradients_match_the_oracle(case10, monkeypatch, tp, strategy):
    ll, sd, x, target, var, ref32, ref64 = case10
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")  # (the bounded step: 18 decoder chunks)
    model = _model(ll, sd, tp, strategy)
    ours = _step(model, ll, x, target, var)
    assert model._train_engine.plan.train_only == (strategy in BOUNDED)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=0.99, total_cos=None,
                        tag=strategy)  # fmt: skip
        return
    # fp32 mode: a floor for a ReLU unit within ~1e-6 of zero that switches between the two fp32 implementations (the case
    # tests/test_gpu_train_precision.py describes, whose 2e-3 covers the forecaster's switched units).  Here one unit of the decoder
    # block's node MLP switches and leaves 6.1e-3 / 5.9e-3 on its model.2 weight / bias (fp32 oracle 3.7e-7 / 1.5e-7), measured on an H100, in the
    # taped and the bounded step alike; every other parameter is within 10x the fp32 oracle's error or below 2e-3.  The features'
    # gradient is that of the full input, residual path included (decoder.py:93 adds all 78 input channels).
    check_fp32_bars(ours, ref32, ref64, n_params=215, floor=1e-2 if tp == "fp32" else 0.0, feat_floor=False, median=False,
                    ill=None, skip_zero=False, norm_bar=None, tag=f"{tp} {strategy}")  # fmt: skip


@pytest.mark.parametrize("efficient", [False, True])
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_strategies_match_the_taped_step(case10, monkeypatch, tp, efficient):
    """Each strategy's forward equals the taped step's bit for bit, and its gradients are within 1e-5 of the taped step's (the
    bounded step sums the same rows in chunks: 1-point chunks on the 648-point grid)."""
    ll, sd, x, target, var = case10[:5]
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "1")
    out_t, loss_t, gx_t, g_t = _step(_model(ll, sd, tp), ll, x, target, var)
    for strategy in STRATEGIES:
        model = _model(ll, sd, tp, strategy, efficient_batching=efficient)
        out, loss, gx, grads = _step(model, ll, x, target, var)
        assert model._train_engine.plan.train_only == (strategy in BOUNDED), strategy
        assert torch.equal(out, out_t) and loss == loss_t, strategy
        worst = max((rel_norm(grads[k], g), k) for k, g in g_t.items() if float(g.norm()) > 0)
        print(f"{tp} {strategy} efficient_batching={efficient}: worst gradient difference to the taped step {worst}; "
              f"features {rel_norm(gx, gx_t):.2e}")
        assert worst[0] <= 1e-5 and rel_norm(gx, gx_t) <= 1e-5, (strategy, worst)


def _reference_grid():
    """create_lat_lon_grid(resolution_deg=10.0) of the reference's checkpointing tests: 18 x 36 points."""
    return [(float(lat), float(lon)) for lat in np.arange(-90.0, 90.0, 10.0) for lon in np.arange(0.0, 360.0, 10.0)]


def test_reference_backward_with_checkpointing():
    """tests/models/test_gradient_checkpointing.py::test_backward_pass_with_checkpointing on the GPU: use_checkpointing=True,
    efficient batching, balanced_checkpointing; every gradient exists and is finite."""
    from graph_weather_b200 import GraphCast, GraphCastConfig

    lat_lons = _reference_grid()
    model = GraphCast(lat_lons, use_checkpointing=True, efficient_batching=True).cuda()
    GraphCastConfig.balanced_checkpointing(model)
    model.train()
    torch.manual_seed(42)
    features = torch.randn((1, len(lat_lons), 78), device="cuda")
    target = torch.randn((1, len(lat_lons), 78), device="cuda")
    output = model(features)
    torch.nn.functional.mse_loss(output, target).backward()
    assert model._train_engine.plan.train_only
    assert all(q.grad is not None for q in model.parameters())
    for q in model.parameters():
        assert not torch.isnan(q.grad).any() and not torch.isinf(q.grad).any()


def test_reference_gradient_equivalence():
    """tests/models/test_gradient_checkpointing.py::test_gradient_equivalence on the GPU: gradients without checkpointing (the
    taped step) and with balanced_checkpointing (the bounded step) agree to atol 1e-5."""
    from graph_weather_b200 import GraphCast, GraphCastConfig

    lat_lons = _reference_grid()
    torch.manual_seed(42)
    features = torch.randn((1, len(lat_lons), 78)).cuda()
    target = torch.randn((1, len(lat_lons), 78)).cuda()
    model_no_cp = GraphCast(lat_lons, use_checkpointing=False, efficient_batching=True).cuda()
    GraphCastConfig.no_checkpointing(model_no_cp)
    model_no_cp.train()
    torch.nn.functional.mse_loss(model_no_cp(features), target).backward()
    grads_no_cp = [q.grad.clone() for q in model_no_cp.parameters() if q.grad is not None]
    model_with_cp = GraphCast(lat_lons, use_checkpointing=False, efficient_batching=True).cuda()
    model_with_cp.load_state_dict(model_no_cp.state_dict())
    GraphCastConfig.balanced_checkpointing(model_with_cp)
    model_with_cp.train()
    torch.nn.functional.mse_loss(model_with_cp(features), target).backward()
    grads_with_cp = [q.grad.clone() for q in model_with_cp.parameters() if q.grad is not None]
    assert not model_no_cp._train_engine.plan.train_only and model_with_cp._train_engine.plan.train_only
    assert len(grads_no_cp) == len(grads_with_cp) == 215
    for g1, g2 in zip(grads_no_cp, grads_with_cp):
        assert torch.allclose(g1, g2, atol=1e-5), float((g1 - g2).abs().max())


@pytest.mark.parametrize("strategy", ["no_checkpointing", "balanced_checkpointing"])
def test_sgd_lowers_the_loss_and_inference_is_untouched(case10, strategy):
    ll, sd, x, target, var = case10[:5]
    model = _model(ll, sd, "fp32_simt", strategy)
    xc = x.cuda()
    model.eval()
    with torch.no_grad():
        before = model(xc).clone()
    model.train()
    _, loss0, _, _ = _step(model, ll, x, target, var, feat_grad=False)
    model.eval()
    with torch.no_grad():
        after = model(xc)
    assert not after.requires_grad
    assert torch.equal(after, before)  # the training step runs on its own plan
    model.train()
    opt = torch.optim.SGD(model.parameters(), lr=1e-2)
    opt.step()
    opt.zero_grad()
    _, loss1, _, grads = _step(model, ll, x, target, var, feat_grad=False)
    assert loss1 < loss0
    assert all(torch.isfinite(g).all() for g in grads.values())


def test_strategy_switch_between_forward_and_backward_raises(case10):
    """Only one training plan is held: a forward under one strategy, a forward under another, then the first one's backward."""
    from graph_weather_b200 import GraphCastConfig

    ll, sd, x = case10[:3]
    model = _model(ll, sd)
    a = model(x.cuda())
    GraphCastConfig.balanced_checkpointing(model)
    b = model(x.cuda())
    assert model._train_engines[False].plan is None  # the taped step's plan was closed
    b.square().mean().backward()
    with pytest.raises(RuntimeError, match="one backward per forward"):
        a.square().mean().backward()


def test_tensor_core_precision_needs_two_hidden_layers():
    from graph_weather_b200 import GraphCast

    with pytest.raises(ValueError, match="train_precision"):
        GraphCast(grid(10), hidden_layers=3, train_precision="bf16")
