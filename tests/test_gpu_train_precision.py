"""-m gpu: the training step on tensor cores (`train_precision="fp32"` / `"bf16"`, gw_train.cu + gw_wgrad_tc.cu) against the
CPU autograd oracle (fp32 and the fp64 ground truth), against the exact-fp32 training path, and its side conditions:
convergence, repeatable weight gradients, raw input magnitudes and an untouched inference path.  The 1-degree grid is held to the
fp64 oracle in tests/test_gpu_full_grid.py."""
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import ILL_CONDITIONED, check_bf16_bars, check_fp32_bars, forecaster_case, grid, rel_norm, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture(scope="module")
def case10():
    """The seeded 10-degree, batch-2 step of tests/test_gpu_training.py and its oracle results (fp32 and fp64)."""
    return forecaster_case(10, 2, 21)


def _step(tp, ll, sd, x, target, var, feat_grad=True):
    """One training step of a fresh forecaster: (model, out, loss, d features, {name: grad})."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    model = GraphWeatherForecaster(ll, train_precision=tp).cuda().train()
    model.load_state_dict(sd)
    return (model, *train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target, feat_grad=feat_grad))


def _norm_bar(k, tol):
    return 5 * tol if k.startswith(ILL_CONDITIONED) else tol


def test_fp32_matches_the_oracle(case10):
    ll, sd, x, target, var, ref32, ref64 = case10
    model, *ours = _step("fp32", ll, sd, x, target, var)
    assert model._train_engine.resolved_precision == "fp32"
    # (measured: every parameter within 10x the fp32 oracle's error except three at 1.0e-3 .. 1.1e-3 max-relative error where the
    # oracle is at 1.8e-7 .. 6e-5: isolated ReLU units within ~1e-6 of zero switch between the two fp32 implementations -- the fp32
    # oracle itself is at 1.07e-3 on processor block 4 for the same reason.  A 2e-3 floor covers a switched unit.)
    check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3, feat_floor=False, median=False, ill=None, skip_zero=False,
                    norm_bar=None)  # fmt: skip


def test_bf16_matches_the_oracle(case10):
    ll, sd, x, target, var, ref32, ref64 = case10
    model, *ours = _step("bf16", ll, sd, x, target, var)
    assert model._train_engine.resolved_precision == "bf16"
    # (measured: 0.9858 for h3_nodes and 0.9895 for node_encoder.model.0.weight, >= 0.998 for every other parameter)
    check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999)


def test_convergence_against_the_exact_path(case10):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = case10[:5]
    xc, tc = x.cuda(), target.cuda()
    final = {}
    for tp in ("fp32_simt", "fp32", "bf16"):
        torch.manual_seed(0)
        model = GraphWeatherForecaster(ll, train_precision=tp).cuda().train()
        model.load_state_dict(sd)
        crit = NormalizedMSELoss(var, ll, normalize=True)
        opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
        losses = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            loss = crit(model(xc), tc)
            loss.backward()
            opt.step()
            losses.append(float(loss))
        model._train_engine.plan.status()
        assert all(np.isfinite(losses)), (tp, losses)
        final[tp] = losses
    print({k: (v[0], v[-1]) for k, v in final.items()})
    ref = final["fp32_simt"][-1]
    assert abs(final["fp32"][-1] - ref) <= 0.01 * abs(ref)
    assert abs(final["bf16"][-1] - ref) <= 0.05 * abs(ref)
    assert final["bf16"][-1] < final["bf16"][0]


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_weight_gradients_are_repeatable(case10, tp):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = case10[:5]
    model = GraphWeatherForecaster(ll, train_precision=tp).cuda().train()
    model.load_state_dict(sd)
    crit = NormalizedMSELoss(var, ll, normalize=True)
    runs = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        crit(model(x.cuda()), target.cuda()).backward()
        runs.append({k: q.grad.clone() for k, q in model.named_parameters() if k.startswith("processor.")})
    model._train_engine.plan.status()
    # the Linear layers (model.0 / .2 / .4; model.5 is the LayerNorm, whose parameter gradients are CUDA-core atomics)
    linear = [k for k in runs[0] if any(f".model.{i}." in k for i in (0, 2, 4))]
    assert len(linear) > 100
    for k in linear:
        assert torch.equal(runs[0][k], runs[1][k]), k


@pytest.mark.parametrize("scale", [1e5, 3e-4])
def test_raw_magnitudes(case10, scale):
    ll, sd, x, target, var = case10[:5]
    xs = x * scale
    ts = target * scale
    _, _, _, _, g_simt = _step("fp32_simt", ll, sd, xs, ts, var, feat_grad=False)
    model, _, loss, _, g_tc = _step("fp32", ll, sd, xs, ts, var, feat_grad=False)
    assert np.isfinite(loss)
    errs = []
    for k in g_tc:
        assert torch.isfinite(g_tc[k]).all(), k
        if float(g_simt[k].norm()) == 0.0:
            continue
        errs.append((rel_norm(g_tc[k], g_simt[k]), k))
    errs.sort(reverse=True)
    print(f"scale {scale:g}: worst |g_tc - g_simt| / |g_simt|: {errs[:4]}")
    # (x1e5 drives the first layers 5 decades above the data they were scaled for: measured up to 1.4e-3 on processor weights, so
    # that case is held to 2e-3; x3e-4 keeps 1e-3)
    tol = 2e-3 if scale > 1 else 1e-3
    for e, k in errs:
        assert e < _norm_bar(k, tol), (k, e)


def test_inference_is_untouched_by_bf16_training(case10):
    from graph_weather_b200 import GraphWeatherForecaster

    ll, sd, x, target, var = case10[:5]
    model, _, _, _, _ = _step("bf16", ll, sd, x, target, var)
    fresh = GraphWeatherForecaster(ll).cuda().eval()
    fresh.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        a = model(x.cuda())
        b = fresh(x.cuda())
    assert torch.equal(a, b)
    model.train()
    with torch.no_grad():  # no_grad in train mode is inference as well
        c = model(x.cuda())
    assert torch.equal(c, b)


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_one_backward_per_forward(tp):
    from graph_weather_b200 import GraphWeatherForecaster

    ll = grid(30)
    model = GraphWeatherForecaster(ll, num_blocks=2, train_precision=tp).cuda().train()
    x = torch.randn(1, len(ll), 102, device="cuda")
    a = model(x)
    b = model(x)  # replaces the tape of `a`
    b.sum().backward()
    with pytest.raises(RuntimeError, match="one backward per forward"):
        a.sum().backward()
