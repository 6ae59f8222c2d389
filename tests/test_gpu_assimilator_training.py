"""-m gpu: GraphWeatherAssimilator trains.  `model(features, obs_lat_lon_heights)` in train mode with autograd on builds the
observation graph on the device for the call, and `loss.backward()` runs the CUDA training step on it.

The model is the reference README's (5-degree output grid, analysis_dim 24, 2 values per observation), on a few hundred random
observations.  The oracle is torch.autograd through the restatement of analysis.py's forward (oracle/restate.py's pieces, composed
as restate.assimilator_forward composes them), in fp32 and in fp64, at batch 1 (the README's; the reference replicates the input
graph with an offset that is only a per-sample block at batch 1).
  * every parameter's gradient and the observation values' gradient against fp64, in every train precision, taped and bounded
    (in fp32 / bf16 this runs the K = 2 node-encoder layer and the N = 2 feature gradient on tensor cores);
  * two steps on different observation sets, the second larger (the plan regrows), each against the oracle on its own set;
  * the bounded step's chunk tables follow the observation graph: set A then set B at the same batch equals a fresh model on B;
  * a forward on other observations between a forward and its backward makes that backward raise;
  * a NaN observation raises as in inference (status bit 16), and the next call with finite observations trains."""
import re

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import assimilator_oracle_step, check_bf16_bars, check_fp32_bars, rel_norm, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]

ANALYSIS_DIM = 24


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _out_grid():
    return [(float(lat), float(lon)) for lat in range(-90, 90, 5) for lon in range(0, 360, 5)]


def _obs(n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return torch.from_numpy(np.stack([rng.uniform(-90, 90, n), rng.uniform(0, 360, n), rng.uniform(0, 1, n)], 1).astype(np.float32))


@pytest.fixture(scope="module")
def setup():
    from oracle import restate, weights

    out_ll = _out_grid()
    sd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=ANALYSIS_DIM), 41)
    return out_ll, sd, restate.build_assimilator_graphs(out_ll)


def _case(setup, n, seed, batch=1):
    from oracle import weights

    out_ll = setup[0]
    x = weights.make_features(batch, n, 2, seed)
    target = torch.randn(batch, len(out_ll), ANALYSIS_DIM, generator=torch.Generator().manual_seed(seed))
    return x, _obs(n, seed), target


def _oracle(sd, g_static, x, obs, target):
    """The oracle step in fp32 and in fp64."""
    return [assimilator_oracle_step(sd, g_static, x, obs, target, dt) for dt in (torch.float32, torch.float64)]


def _model(setup, tp="fp32_simt", lean=False):
    from graph_weather_b200 import GraphWeatherAssimilator

    model = GraphWeatherAssimilator(output_lat_lons=setup[0], analysis_dim=ANALYSIS_DIM, train_precision=tp, use_checkpointing=lean)
    model = model.cuda().train()
    model.load_state_dict(setup[1])
    return model


def _step(model, x, obs, target):
    return train_step(model, torch.nn.functional.mse_loss, x, target, obs=obs)


def _check(tp, res, ref32, ref64, tag=""):
    """The bars of tests/test_gpu_training.py (fp32_simt) and tests/test_gpu_lean_training.py (fp32, bf16), with the floor on the
    observation values' gradient too; 214 parameters (the reference keeps the encoder's h3_nodes a plain tensor)."""
    if tp == "bf16":
        check_bf16_bars(res, ref32, ref64, n_params=214, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=0.98, total_cos=None, tag=tag)
    else:
        check_fp32_bars(res, ref32, ref64, n_params=214, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=True, median=False,
                        ill=None, skip_zero=False, norm_bar=None, tag=f"{tag} {tp}")  # fmt: skip


@pytest.fixture(scope="module")
def case300(setup):
    x, obs, target = _case(setup, 300, 51)
    sd, g = setup[1], setup[2]
    return (x, obs, target, *_oracle(sd, g, x, obs, target))


@pytest.mark.parametrize("lean", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_gradients_match_the_oracle(setup, case300, monkeypatch, tp, lean):
    x, obs, target, ref32, ref64 = case300
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "23")
    model = _model(setup, tp, lean)
    res = _step(model, x, obs, target)
    assert model._train_engine.plan.train_only == lean
    assert model._train_engine.resolved_precision == tp
    _check(tp, res, ref32, ref64, "300 obs")


@pytest.mark.parametrize("lean", [False, True], ids=["taped", "bounded"])
def test_a_larger_observation_set_regrows_the_plan(setup, case300, monkeypatch, lean):
    """Step 1 on 300 observations, step 2 on 450 others: the training plan is rebuilt for 450, and each step's gradients meet the
    bars against the oracle on its own set."""
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "23")
    model = _model(setup, "fp32_simt", lean)
    x, obs, target, ref32, ref64 = case300
    _check("fp32_simt", _step(model, x, obs, target), ref32, ref64, "step 1")
    gen = model._train_engine.generation
    x2, obs2, target2 = _case(setup, 450, 52)
    res = _step(model, x2, obs2, target2)
    assert model._train_engine.generation == gen + 1 and model._train_engine.dims["n_in"] == 450
    sd, g = setup[1], setup[2]
    _check("fp32_simt", res, *_oracle(sd, g, x2, obs2, target2), "step 2")


@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_bounded_step_follows_the_observation_graph(setup, monkeypatch, tp):
    """Many small chunks, batch 2: a step on set A, then a step on set B of the same size (same plan, same batch), equals a fresh
    model's step on B.  Chunk tables kept from A's graph would cover the wrong observations."""
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "7")
    xa, obs_a, ta = _case(setup, 400, 61, batch=2)
    xb, obs_b, tb = _case(setup, 400, 62, batch=2)
    model = _model(setup, tp, True)
    _step(model, xa, obs_a, ta)
    gen = model._train_engine.generation
    out, loss, gx, grads = _step(model, xb, obs_b, tb)
    assert model._train_engine.generation == gen  # no new plan: the same plan took the second graph
    out_f, loss_f, gx_f, grads_f = _step(_model(setup, tp, True), xb, obs_b, tb)
    assert torch.equal(out, out_f) and loss == loss_f
    worst = max((rel_norm(grads[k], g), k) for k, g in grads_f.items() if float(g.norm()) > 0)
    print(f"{tp}: set A then B vs fresh on B: worst gradient difference {worst}; features {rel_norm(gx, gx_f):.2e}")
    assert worst[0] <= 1e-6 and rel_norm(gx, gx_f) <= 1e-6


@pytest.mark.parametrize("lean", [False, True], ids=["taped", "bounded"])
def test_forward_on_other_observations_before_the_backward_raises(setup, lean):
    model = _model(setup, "fp32_simt", lean)
    xa, obs_a, _ = _case(setup, 300, 71)
    xb, obs_b, _ = _case(setup, 350, 72)
    a = model(xa.cuda(), obs_a.cuda())
    b = model(xb.cuda(), obs_b.cuda())  # replaces the tape (and the observation graph) of `a`
    b.square().mean().backward()
    with pytest.raises(RuntimeError, match="one backward per forward"):
        a.square().mean().backward()


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32"])
def test_non_finite_observation_raises_and_the_next_step_trains(setup, monkeypatch, tp):
    """As in inference (tests/test_gpu_graph_kernels.py::test_assimilator_refuses_non_finite_observation): status bit 16."""
    monkeypatch.setenv("GW_B200_CHECK", "1")  # synchronise and read the status word after every forward
    model = _model(setup, tp)
    x, obs, target = _case(setup, 300, 81)
    bad = obs.clone()
    bad[77, 0] = float("nan")
    with pytest.raises(RuntimeError) as e:
        model(x.cuda().requires_grad_(True), bad.cuda())
    m = re.search(r"device status (\d+)", str(e.value))
    assert m and int(m.group(1)) & 16, str(e.value)
    out, loss, gx, grads = _step(model, x, obs, target)
    assert np.isfinite(loss) and torch.isfinite(gx).all() and all(torch.isfinite(g).all() for g in grads.values())
