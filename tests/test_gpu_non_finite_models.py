"""-m gpu: NaN and +-inf inputs through whole models, inference and training, against the CPU oracle (the reference arithmetic).

The cases (tests/test_non_finite_oracle.py, which also checks on the CPU that each is informative) poison one feature of one point
of sample 1 of the seeded 10-degree, batch-2 forecaster case, in a residual column (5) or an auxiliary one (90), with NaN, +inf or
-inf; GraphCast and the assimilator get one NaN case each.  The contract (README, "Non-finite inputs"):
  * fp32_simt propagates non-finite values as torch does: the NaN / +inf / -inf pattern of the output, the loss and the feature
    gradient is the oracle's, a parameter gradient contains a NaN exactly when the oracle's does, the clean sample is untouched
    bit for bit, and finite entries are within TOL of the oracle;
  * the tensor-core precisions (fp32, bf16) refuse non-finite features or weights, in inference and in both training steps:
    the call raises the RuntimeError of status bit 3, and the same model then computes on clean data exactly what a fresh one
    does."""
import math

import pytest
import torch

import __graft_entry__ as ge
from test_non_finite_oracle import (ASSIM_DIM, FORECASTER_CASES, assimilator_base, assimilator_oracle, assimilator_poisoned, forecaster_base,
                                    forecaster_oracle, poisoned)  # fmt: skip
from training_oracle import rel_norm, train_step

pytestmark = pytest.mark.gpu

TOL = 1e-4
BIT3 = "a magnitude bound is not finite"  # _capi.Plan.status' text for status bit 3
POISONED_WEIGHT = "processor.graph_processor.blocks.3.edge_model.edge_mlp.model.2.weight"  # read in full by every path


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


CASES = [pytest.param(v, c, id=f"{v}-col{c}") for v, c in FORECASTER_CASES]


def _forecaster(prec="fp32_simt", tp="fp32_simt", bounded=False, model="forecaster", sd=None):
    from graph_weather_b200 import GraphCast, GraphWeatherForecaster

    ll, base_sd = forecaster_base(model)[:2]
    cls = GraphCast if model == "graphcast" else GraphWeatherForecaster
    m = cls(ll, precision=prec, train_precision=tp, use_checkpointing=bounded).cuda()
    m.load_state_dict(base_sd if sd is None else sd)
    return m


def _mask_fails(got, want, tag):
    """NaN, +inf and -inf exactly where want has them; finite entries within TOL."""
    got, want = got.double().cpu(), want.double().cpu()
    fails = [f"{tag}: {f.__name__[2:]} pattern differs at {int((f(got) != f(want)).sum())} of {got.numel()} entries"
             for f in (torch.isnan, torch.isposinf, torch.isneginf) if not torch.equal(f(got), f(want))]  # fmt: skip
    fin = torch.isfinite(got) & torch.isfinite(want)
    err = float((got[fin] - want[fin]).abs().max()) if bool(fin.any()) else 0.0
    if not err < TOL:
        fails.append(f"{tag}: finite entries differ by {err:.2e}")
    return fails


def _grad_nan_fails(grads, ref, tag):
    """Each parameter gradient contains a NaN exactly when the oracle's does."""
    assert set(grads) == set(ref)
    return [f"{tag}: {k} has NaN {bool(torch.isnan(g).any())}, oracle {bool(torch.isnan(ref[k]).any())}"
            for k, g in grads.items() if bool(torch.isnan(g).any()) != bool(torch.isnan(ref[k]).any())]  # fmt: skip


# ---- inference --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value,col", CASES)
def test_simt_inference_propagates_as_torch(value, col):
    x = forecaster_base()[2]
    model = _forecaster().eval()
    clean = model(x.cuda()).cpu()
    out = model(poisoned(x, value, col).cuda()).cpu()
    fails = _mask_fails(out, forecaster_oracle("forecaster", value, col)[0], "forecast")
    if not torch.equal(out[0].view(torch.int32), clean[0].view(torch.int32)):
        fails.append("the clean sample's forecast changed")
    assert not fails, fails


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("value,col", CASES)
def test_tensor_core_inference_refuses(value, col, prec):
    x = forecaster_base()[2].cuda()
    model = _forecaster(prec).eval()
    with pytest.raises(RuntimeError, match=BIT3):
        model(poisoned(x.cpu(), value, col).cuda())
    again = model(x)
    fresh = _forecaster(prec).eval()(x)
    assert torch.equal(again.view(torch.int32), fresh.view(torch.int32)), "the model computes differently after a refused call"


def _poisoned_sd(value="nan"):
    sd = {k: v.clone() for k, v in forecaster_base()[1].items()}
    sd[POISONED_WEIGHT][7, 11] = float(value)
    return sd


@pytest.mark.parametrize("prec", ["fp32_simt", "fp32", "bf16"])
def test_non_finite_weight(prec):
    """One NaN in a processor edge-MLP weight: fp32_simt gives the oracle's pattern (the whole forecast, as in torch), the
    tensor-core precisions raise; after reloading clean weights the model computes what a fresh one does."""
    from oracle import restate

    ll, sd, x = forecaster_base()[:3]
    bad = _poisoned_sd()
    model = _forecaster(prec, sd=bad).eval()
    if prec == "fp32_simt":
        want = restate.forecaster_forward(bad, restate.build_forecaster_graphs(ll), x)
        fails = _mask_fails(model(x.cuda()).cpu(), want, "forecast")
        assert not fails, fails
    else:
        with pytest.raises(RuntimeError, match=BIT3):
            model(x.cuda())
    model.load_state_dict(sd)
    again = model(x.cuda())
    fresh = _forecaster(prec).eval()(x.cuda())
    assert torch.equal(again.view(torch.int32), fresh.view(torch.int32))


# ---- training -----------------------------------------------------------------------------------------------------------------------
def _loss_fn(model="forecaster"):
    from graph_weather_b200 import NormalizedMSELoss

    ll, _, _, _, var = forecaster_base(model)
    return NormalizedMSELoss(var, ll, normalize=True)


@pytest.mark.training
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("value,col", CASES)
def test_simt_training_propagates_as_torch(value, col, bounded, monkeypatch):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")  # (the bounded step: many chunks)
    x, target = forecaster_base()[2], forecaster_base()[3]
    model = _forecaster(bounded=bounded).train()
    out, loss, gx, grads = train_step(model, _loss_fn(), poisoned(x, value, col), target)
    r_out, r_loss, r_gx, r_grads = forecaster_oracle("forecaster", value, col)
    fails = _mask_fails(out, r_out, "out") + _mask_fails(gx, r_gx, "d features") + _grad_nan_fails(grads, r_grads, "grad")
    if math.isnan(loss) != math.isnan(r_loss) or (math.isinf(r_loss) and loss != r_loss):
        fails.append(f"loss {loss}, oracle {r_loss}")
    assert not fails, fails


def _same_step(a, b):
    """Two clean training steps agree: output and loss bit for bit, the processor's Linear weight gradients (tensor-core weight
    gradients, repeatable: tests/test_gpu_train_precision.py) bit for bit, everything else within 1e-5 (float atomics)."""
    out, loss, gx, grads = a
    out_f, loss_f, gx_f, grads_f = b
    fails = [] if torch.equal(out, out_f) and loss == loss_f else ["output or loss differ"]
    for k, g in grads.items():
        if k.startswith("processor.") and any(f".model.{i}." in k for i in (0, 2, 4)):
            same = torch.equal(g, grads_f[k])
        else:
            same = rel_norm(g, grads_f[k]) <= 1e-5
        if not same:
            fails.append(k)
    if not rel_norm(gx, gx_f) <= 1e-5:
        fails.append("d features")
    return fails


@pytest.mark.training
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
@pytest.mark.parametrize("value,col", CASES)
def test_tensor_core_training_refuses(value, col, tp, bounded, monkeypatch):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    x, target = forecaster_base()[2], forecaster_base()[3]
    model = _forecaster(tp=tp, bounded=bounded).train()
    with pytest.raises(RuntimeError, match=BIT3):
        model(poisoned(x, value, col).cuda().requires_grad_(True))
    fails = _same_step(train_step(model, _loss_fn(), x, target), train_step(_forecaster(tp=tp, bounded=bounded).train(), _loss_fn(), x, target))
    assert not fails, fails


@pytest.mark.training
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_training_refuses_a_non_finite_weight(tp):
    x, target = forecaster_base()[2], forecaster_base()[3]
    model = _forecaster(tp=tp, sd=_poisoned_sd()).train()
    with pytest.raises(RuntimeError, match=BIT3):
        model(x.cuda().requires_grad_(True))
    model.load_state_dict(forecaster_base()[1])
    fails = _same_step(train_step(model, _loss_fn(), x, target), train_step(_forecaster(tp=tp).train(), _loss_fn(), x, target))
    assert not fails, fails


# ---- GraphCast and the assimilator --------------------------------------------------------------------------------------------------
def test_graphcast_simt_inference_propagates_as_torch():
    x = forecaster_base("graphcast")[2]
    model = _forecaster(model="graphcast").eval()
    out = model(poisoned(x, "nan", 5).cuda()).cpu()
    fails = _mask_fails(out, forecaster_oracle("graphcast", "nan", 5)[0], "GraphCast forecast")
    assert not fails, fails


@pytest.mark.training
def test_graphcast_bf16_training_refuses():
    x = forecaster_base("graphcast")[2]
    model = _forecaster(tp="bf16", model="graphcast").train()
    with pytest.raises(RuntimeError, match=BIT3):
        model(poisoned(x, "nan", 5).cuda().requires_grad_(True))


def _assimilator(prec="fp32_simt", tp="fp32_simt"):
    from graph_weather_b200 import GraphWeatherAssimilator

    out_ll, sd = assimilator_base()[:2]
    model = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=ASSIM_DIM, precision=prec, train_precision=tp).cuda()
    model.load_state_dict(sd)
    return model


def test_assimilator_simt_inference_propagates_as_torch():
    obs = assimilator_base()[4]
    out = _assimilator().eval()(assimilator_poisoned().cuda(), obs.cuda()).cpu()
    fails = _mask_fails(out, assimilator_oracle()[0], "analysis")
    assert not fails, fails


@pytest.mark.training
def test_assimilator_bf16_training_refuses():
    obs = assimilator_base()[4]
    model = _assimilator(tp="bf16").train()
    with pytest.raises(RuntimeError, match=BIT3):
        model(assimilator_poisoned().cuda().requires_grad_(True), obs.cuda())
