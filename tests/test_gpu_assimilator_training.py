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
from test_gpu_train_precision import ILL_CONDITIONED  # (tests/ is on sys.path: pytest imports its modules by basename)

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


def _oracle(sd, g_static, x, obs, target, dtype=torch.float32):
    """torch.autograd through analysis.py's forward (assimilator_encoder.py:118-168 + processor + assimilator decoder) and
    MSELoss: (out, loss, d features, {name: grad})."""
    from oracle import restate

    sd_g = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    g = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in g_static.items()}
    xg = x.to(dtype).clone().requires_grad_(True)
    B, nobs = x.shape[0], obs.shape[0]
    in_ei, in_ea = restate.assimilator_input_graph(obs, g["base_h3_grid"])
    h3_nodes = torch.zeros((g["num_h3"], x.shape[-1]), dtype=dtype)
    feats = torch.cat([xg, h3_nodes.unsqueeze(0).expand(B, -1, -1)], dim=1).reshape(-1, x.shape[-1])
    h = restate.mlp(sd_g, "encoder.node_encoder", feats)
    ea = restate.mlp(sd_g, "encoder.edge_encoder", in_ea.to(dtype)).repeat(B, 1)
    h, _ = restate.graph_processor(sd_g, "encoder.graph_processor", h, restate._replicate(in_ei, B), ea, 1)
    h = h.reshape(B, -1, h.shape[-1])[:, nobs:, :].reshape(-1, h.shape[-1])
    lat_ea = restate.mlp(sd_g, "encoder.latent_edge_encoder", g["lat_edge_attr"].repeat(B, 1))
    h = restate.processor_forward(sd_g, h, restate._replicate(g["lat_edge_index"], B), lat_ea, 9)
    out = restate.assimilator_decoder_forward(sd_g, g, h, B)
    loss = torch.nn.functional.mse_loss(out, target.to(dtype))
    loss.backward()
    return out.detach(), float(loss.detach()), xg.grad, {k: v.grad for k, v in sd_g.items()}


def _model(setup, tp="fp32_simt", lean=False):
    from graph_weather_b200 import GraphWeatherAssimilator

    model = GraphWeatherAssimilator(output_lat_lons=setup[0], analysis_dim=ANALYSIS_DIM, train_precision=tp, use_checkpointing=lean)
    model = model.cuda().train()
    model.load_state_dict(setup[1])
    return model


def _step(model, x, obs, target):
    xc = x.cuda().requires_grad_(True)
    out = model(xc, obs.cuda())
    assert out.requires_grad
    loss = torch.nn.functional.mse_loss(out, target.cuda())
    loss.backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    return out.detach().cpu(), float(loss), xc.grad.cpu(), grads


def _rel_max(a, b):
    return float((a.double() - b.double()).abs().max()) / (float(b.double().abs().max()) + 1e-30)


def _rel_norm(a, b):
    return float((a.double() - b.double()).norm()) / (float(b.double().norm()) + 1e-30)


def _check(tp, res, ref32, ref64, tag=""):
    """The bars of tests/test_gpu_training.py (fp32_simt) and tests/test_gpu_lean_training.py (fp32, bf16)."""
    out, loss, gx, grads = res
    out32, loss32, gx32, g32 = ref32
    _, _, gx64, g64 = ref64
    assert set(grads) == set(g64) and len(grads) == 214
    if tp == "bf16":
        assert float((out - out32).abs().max()) < 2e-2 and abs(loss - loss32) <= 1e-2 * abs(loss32)
        big = max(float(g.abs().max()) for g in g64.values())
        for k, g in grads.items():
            ref = g64[k].double().flatten()
            if float(ref.abs().max()) <= 1e-6 * big:
                continue
            cos = float(torch.nn.functional.cosine_similarity(g.double().flatten(), ref, dim=0))
            assert cos >= (0.98 if k.startswith(ILL_CONDITIONED) else 0.99), (tag, k, cos)
        cos = float(torch.nn.functional.cosine_similarity(gx.double().flatten(), gx64.double().flatten(), dim=0))
        assert cos >= 0.98, (tag, cos)
        return
    assert float((out - out32).abs().max()) < 1e-4 and abs(loss - loss32) <= 1e-5 * abs(loss32), tag
    floor = 2e-3 if tp == "fp32" else 0.0
    e_ours, e_ref = _rel_max(gx, gx64), _rel_max(gx32, gx64)
    print(f"{tag} {tp}: d observation values rel err vs fp64 {e_ours:.2e} (fp32 oracle {e_ref:.2e})")
    assert e_ours < max(10 * e_ref + 2e-5, floor), (tag, e_ours, e_ref)
    errs = sorted(((_rel_max(grads[k], g64[k]), _rel_max(g32[k], g64[k]), k) for k in grads), reverse=True)
    print(f"{tag} {tp}: worst rel err vs fp64 {errs[:4]}")
    for eo, er, k in errs:
        assert eo < max(10 * er + 2e-5, floor), (tag, k, eo, er)


@pytest.fixture(scope="module")
def case300(setup):
    x, obs, target = _case(setup, 300, 51)
    sd, g = setup[1], setup[2]
    return x, obs, target, _oracle(sd, g, x, obs, target), _oracle(sd, g, x, obs, target, torch.float64)


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
    _check("fp32_simt", res, _oracle(sd, g, x2, obs2, target2), _oracle(sd, g, x2, obs2, target2, torch.float64), "step 2")


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
    worst = max((_rel_norm(grads[k], g), k) for k, g in grads_f.items() if float(g.norm()) > 0)
    print(f"{tp}: set A then B vs fresh on B: worst gradient difference {worst}; features {_rel_norm(gx, gx_f):.2e}")
    assert worst[0] <= 1e-6 and _rel_norm(gx, gx_f) <= 1e-6


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
