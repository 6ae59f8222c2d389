"""-m gpu: the training step (SURVEY 8(f) row 2: backward).  `model(features)` in train mode with autograd on, the CUDA
NormalizedMSELoss and `loss.backward()` against torch.autograd on the CPU oracle (the reference's own ops, oracle/restate.py):
the loss value, the gradient of the features and the gradient of every one of the 215 parameters."""
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import check_fp32_bars, forecaster_case, grid, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def test_training_step_matches_autograd_on_the_oracle():
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var, ref32, ref64 = forecaster_case(10, 2, 21)
    model = GraphWeatherForecaster(ll).cuda().train()
    model.load_state_dict(sd)
    crit = NormalizedMSELoss(var, ll, normalize=True)
    ours = train_step(model, crit, x, target)
    # Tolerance.  ReLU masks and LayerNorm statistics sit downstream of ~60 fp32 GEMM layers, so two fp32 implementations of the
    # same step differ by far more than a summation-order ulp (a unit within 1e-6 of zero flips its mask).  The yardstick is
    # therefore the fp64 ground truth: this implementation must be as close to it as the reference's own fp32 arithmetic is
    # (within a factor, plus a floor for gradients that are numerically zero).
    check_fp32_bars(ours, ref32, ref64, n_params=215, floor=0.0, feat_floor=False, median=True, ill=None, skip_zero=False,
                    norm_bar=None)  # fmt: skip
    loss = ours[1]
    # a second step after an optimiser update: weights are re-uploaded, the tape is fresh
    opt = torch.optim.SGD(model.parameters(), lr=1e-2)
    opt.step()
    opt.zero_grad()
    loss2 = crit(model(x.cuda()), target.cuda())
    loss2.backward()
    assert float(loss2) < loss  # one SGD step on a fixed batch lowers the loss
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in model.parameters())
    # inference is unchanged by all this: eval + no_grad is the tensor-core path
    model.eval()
    with torch.no_grad():
        y = model(x.cuda())
    assert not y.requires_grad
    assert model._engine.resolved_precision in ("fp32", "fp32_simt")


def test_one_backward_per_forward():
    from graph_weather_b200 import GraphWeatherForecaster

    ll = grid(30)
    model = GraphWeatherForecaster(ll, num_blocks=2).cuda().train()
    x = torch.randn(1, len(ll), 102, device="cuda")
    a = model(x)
    b = model(x)  # replaces the tape of `a`
    b.sum().backward()
    with pytest.raises(RuntimeError, match="one backward per forward"):
        a.sum().backward()
