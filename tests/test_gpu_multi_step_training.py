"""-m gpu: multi-step (autoregressive rollout) training.  Inside `model.multi_step()` every training forward keeps a tape of its own,
so a loss summed over K chained forecasts back-propagates with one `backward()`:

  * a 3-step rollout of the forecaster (10 degrees, batch 2, seed 21; fresh auxiliary features every step; the sum of three
    NormalizedMSELoss values) against torch.autograd on the CPU oracle chained three times, in fp32 and fp64, in every train
    precision on the taped and the bounded step; GraphCast and the forecaster with the additive constraint layer over 2 steps;
  * composition: K = 1 in the window is the plain step, and independent forwards back-propagated in either order are each the
    forward done alone (also with two batch sizes on the bounded step, whose chunk tables are keyed on the batch);
  * lifetime: tape bytes per forward, nothing left after the backward or after a dropped graph, and the backward that must raise
    (a second one, after the plan was replaced, after the weights were re-uploaded); outside the window a forward still replaces
    the previous one's tape;
  * per-weight work (transposes, weight images) is done once per weight upload, not once per forward;
  * a refused non-finite forward leaves no tape; a 1-degree bf16 bounded smoke run."""
import gc
import weakref

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import check_bf16_bars, check_fp32_bars, forecaster_case, grid, rel_norm

pytestmark = [pytest.mark.gpu, pytest.mark.training]

BIT3 = "a magnitude bound is not finite"  # _capi.Plan.status' text for status bit 3


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


# ---- the rollout and its oracle ---------------------------------------------------------------------------------------------------
def rollout_inputs(case, steps, aux_dim):
    """Step 0's input is the case's features; steps 1.. get auxiliary features from a seeded tensor, and every step a seeded target."""
    x, target = case[2], case[3]
    B, N = x.shape[:2]
    F = target.shape[-1]
    rng = np.random.Generator(np.random.PCG64(22))
    auxs = [None] + [torch.from_numpy(rng.standard_normal((B, N, aux_dim)).astype(np.float32)) for _ in range(1, steps)]
    targets = [target] + [torch.from_numpy(rng.standard_normal((B, N, F)).astype(np.float32)) for _ in range(1, steps)]
    return auxs, targets


def rollout_oracle(case, steps, aux_dim, dtype, num_blocks=9, constraint=None):
    """torch.autograd through `steps` chained oracle forwards (oracle/restate.py; each step's input is the previous forecast, after
    the restated constraint layer if any, followed by that step's auxiliary features) and the summed NormalizedMSELoss.
    Returns (stacked outputs, loss, d x0, {name: grad})."""
    from oracle import restate

    ll, sd, x, _, var = case[:5]
    F = case[3].shape[-1]
    auxs, targets = rollout_inputs(case, steps, aux_dim)
    sd_g = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    xg = x.to(dtype).clone().requires_grad_(True)
    g = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in restate.build_forecaster_graphs(ll).items()}
    inp, loss, outs = xg, 0.0, []
    for t in range(steps):
        ex, ei, ea = restate.encoder_forward(sd_g, g, inp)
        px = restate.processor_forward(sd_g, ex, ei, ea, num_blocks)
        out = restate.assimilator_decoder_forward(sd_g, g, px, x.shape[0]) + inp[..., :F]
        if constraint is not None:
            from test_constraint_grads import grid_mapping, restate_constraint, rows_to_grid

            grid_shape, cell, last = grid_mapping(ll)
            out = restate_constraint(constraint, rows_to_grid(out, grid_shape), rows_to_grid(inp[..., :F], grid_shape), grid_shape, cell, last)
        loss = loss + restate.normalized_mse_loss(out, targets[t].to(dtype), var, ll, True)
        outs.append(out)
        if t + 1 < steps:
            inp = torch.cat([out, auxs[t + 1].to(dtype)], -1) if aux_dim else out
    loss.backward()
    return torch.stack([o.detach() for o in outs]), float(loss.detach()), xg.grad, {k: v.grad for k, v in sd_g.items()}


_ORACLES = {}


def oracle_pair(case_key, case, steps, aux_dim, constraint=None):
    key = (case_key, steps)
    if key not in _ORACLES:
        _ORACLES[key] = tuple(rollout_oracle(case, steps, aux_dim, dt, constraint=constraint) for dt in (torch.float32, torch.float64))
    return _ORACLES[key]


def rollout_step(model, case, steps, aux_dim, feat_grad=True):
    """The same rollout on the GPU inside model.multi_step(), from cleared gradients: (stacked outputs, loss, d x0, {name: grad})."""
    from graph_weather_b200 import NormalizedMSELoss

    ll, _, x, _, var = case[:5]
    crit = NormalizedMSELoss(var, ll, normalize=True)
    auxs, targets = rollout_inputs(case, steps, aux_dim)
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(feat_grad)
    inp, loss, outs = xc, 0.0, []
    with model.multi_step():
        for t in range(steps):
            y = model(inp)
            outs.append(y)
            loss = loss + crit(y, targets[t].cuda())
            if t + 1 < steps:
                inp = torch.cat([y, auxs[t + 1].cuda()], -1) if aux_dim else y
    loss.backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters()}
    return torch.stack([o.detach() for o in outs]).cpu(), float(loss.detach()), (xc.grad.cpu() if feat_grad else None), grads


def _forecaster(ll, sd, tp, bounded=False, **kw):
    from graph_weather_b200 import GraphWeatherForecaster

    model = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=bounded, **kw).cuda().train()
    model.load_state_dict(sd)
    return model


@pytest.fixture(scope="module")
def case10():
    return forecaster_case(10, 2, 21)


# ---- 1. the forecaster's 3-step rollout against the oracle ------------------------------------------------------------------------
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_forecaster_rollout_matches_the_oracle(case10, monkeypatch, tp, bounded):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")  # (the bounded step: many chunks on the 648-point grid)
    ll, sd = case10[:2]
    ref32, ref64 = oracle_pair("forecaster", case10, 3, 24)
    model = _forecaster(ll, sd, tp, bounded)
    ours = rollout_step(model, case10, 3, 24)
    assert model._train_engine.plan.train_only == bounded
    tag = f"{tp} {'bounded' if bounded else 'taped'} 3 steps"
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999, tag=tag)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=0.0 if tp == "fp32_simt" else 2e-3, feat_floor=False,
                        median=tp == "fp32_simt", ill=None, skip_zero=False, norm_bar=None, tag=tag)  # fmt: skip


# ---- 2. GraphCast and the constraint layer, 2 steps ------------------------------------------------------------------------------
@pytest.mark.parametrize("strategy", ["no_checkpointing", "balanced_checkpointing"])
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_graphcast_rollout_matches_the_oracle(monkeypatch, tp, strategy):
    from graph_weather_b200 import GraphCast, GraphCastConfig

    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    case = forecaster_case(10, 2, 21, feature_dim=78, aux_dim=0, hidden_dim_decoder=256)
    ll, sd = case[:2]
    ref32, ref64 = oracle_pair("graphcast", case, 2, 0)
    model = GraphCast(ll, train_precision=tp).cuda().train()
    model.load_state_dict(sd)
    getattr(GraphCastConfig, strategy)(model)
    ours = rollout_step(model, case, 2, 0)
    tag = f"graphcast {tp} {strategy} 2 steps"
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=0.99, total_cos=None, tag=tag)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=0.0, feat_floor=False, median=False, ill=None, skip_zero=False,
                        norm_bar=None, tag=tag)  # fmt: skip


@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_additive_constraint_rollout_matches_the_oracle(tp):
    case = forecaster_case(10, 2, 21, constraint="additive")
    ll, sd = case[:2]
    ref32, ref64 = oracle_pair("additive", case, 2, 24, constraint="additive")
    ours = rollout_step(_forecaster(ll, sd, tp, constraint_type="additive"), case, 2, 24)
    tag = f"additive {tp} 2 steps"
    # the bars of tests/test_gpu_constraint_training.py for the one-step additive case (its comment gives the measurements)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.9, ill_cos_bar=0.9, feat_cos=0.99, total_cos=None, tag=tag)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3, feat_floor=True, median=False, ill="max", skip_zero=True,
                        norm_bar=None, tag=tag)  # fmt: skip


# ---- 3. composition ----------------------------------------------------------------------------------------------------------------
def _loss_fn(case):
    from graph_weather_b200 import NormalizedMSELoss

    return NormalizedMSELoss(case[4], case[0], normalize=True)


def _one(model, x, target, crit, window):
    """One forward + loss + backward, inside a window or not: (out, d x, {name: grad})."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    if window:
        with model.multi_step():
            y = model(xc)
    else:
        y = model(xc)
    crit(y, target.cuda()).backward()
    model._train_engine.plan.status()
    return y.detach().cpu(), xc.grad.cpu(), {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters()}


def _same(a, b, tag):
    """Outputs bit for bit; feature and parameter gradients within 1e-6 norm-relative (fp32_simt's weight gradients use atomics)."""
    assert torch.equal(a[0], b[0]), f"{tag}: outputs differ"
    worst = max([(rel_norm(a[2][k], g), k) for k, g in b[2].items() if float(g.norm()) > 0] + [(rel_norm(a[1], b[1]), "features")])
    assert worst[0] <= 1e-6, (tag, worst)


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_one_step_in_the_window_is_the_plain_step(case10, monkeypatch, tp, bounded):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    ll, sd, x, target = case10[:4]
    model, crit = _forecaster(ll, sd, tp, bounded), _loss_fn(case10)
    plain = _one(model, x, target, crit, False)
    _same(_one(model, x, target, crit, True), plain, f"{tp} window")
    _same(_one(model, x, target, crit, False), plain, f"{tp} plain again")


@pytest.mark.parametrize("order", ["AB", "BA"])
@pytest.mark.parametrize("tp,bounded", [("fp32_simt", False), ("bf16", False), ("bf16", True)])
def test_independent_forwards_back_propagate_in_either_order(case10, monkeypatch, tp, bounded, order):
    """Two forwards A and B of one window (on the bounded step B has batch 1 and A batch 2, so the backward of A needs chunk
    tables of another batch than the last forward built), back-propagated A then B or B then A: each is the forward done alone."""
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    ll, sd, x, target = case10[:4]
    xa, ta = x, target
    xb, tb = (x[:1].flip(1), target[:1]) if bounded else (x.flip(1), target.flip(0))
    model, crit = _forecaster(ll, sd, tp, bounded), _loss_fn(case10)
    alone = {"A": _one(model, xa, ta, crit, False), "B": _one(model, xb, tb, crit, False)}
    ins = {"A": (xa.cuda().requires_grad_(True), ta.cuda()), "B": (xb.cuda().requires_grad_(True), tb.cuda())}
    with model.multi_step():
        ys = {k: model(v[0]) for k, v in ins.items()}
    for k in order:
        model.zero_grad(set_to_none=True)
        crit(ys[k], ins[k][1]).backward()
        model._train_engine.plan.status()
        got = (ys[k].detach().cpu(), ins[k][0].grad.cpu(), {n: q.grad.detach().cpu().clone() for n, q in model.named_parameters()})
        _same(got, alone[k], f"{tp} {order} {k}")


# ---- 4. lifetime ---------------------------------------------------------------------------------------------------------------------
def _small(tp="fp32_simt", bounded=False):
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(0)
    return GraphWeatherForecaster(grid(30), num_blocks=2, train_precision=tp, use_checkpointing=bounded).cuda().train()


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
def test_tape_bytes_and_release(bounded):
    model = _small("bf16", bounded)
    x = torch.randn(2, len(grid(30)), 102, device="cuda")
    with model.multi_step():
        y = model(x)
        single = y.grad_fn.tape.bytes()
        del y
        gc.collect()
        plan = model._train_engine.plan
        assert single > 0 and plan.live_tapes() == []  # the dropped graph's tape is gone
        ys = [model(x) for _ in range(3)]
    assert [y.grad_fn.tape.bytes() for y in ys] == [single] * 3
    assert plan.train_peak_bytes() >= 3 * single
    ref = weakref.ref(ys[1].grad_fn.tape)
    sum(y.square().mean() for y in ys).backward()
    assert plan.live_tapes() == [] and ref() is None
    # the C tape itself: consumed by its backward, 0 bytes after it
    tape = plan.tape()
    out = torch.empty(2, len(grid(30)), 78, device="cuda")
    tape.forward(x, out)
    assert tape.bytes() == single
    named = [(k, torch.empty_like(q)) for k, q in model.named_parameters()]
    tape.backward(torch.ones_like(out), None, named)
    assert tape.bytes() == 0
    with pytest.raises(RuntimeError, match="one backward per forward"):
        tape.backward(torch.ones_like(out), None, named)
    tape.close()


def test_second_backward_raises():
    model = _small()
    x = torch.randn(1, len(grid(30)), 102, device="cuda")
    with model.multi_step():
        loss = model(x).square().mean()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="one backward per forward"):
        loss.backward()


def test_backward_after_the_plan_was_replaced_raises():
    model = _small()
    x = torch.randn(1, len(grid(30)), 102, device="cuda")
    with model.multi_step():
        a = model(x)
        tape = a.grad_fn.tape
        model.use_checkpointing = True  # the bounded step: the taped step's plan is closed, its tapes die with it
        b = model(x)
    assert model._train_engines[False].plan is None and not tape.plan.handle.value
    assert tape.bytes() == 0  # its memory went with the plan
    b.square().mean().backward()
    with pytest.raises(RuntimeError, match="plan was replaced"):
        a.square().mean().backward()
    with pytest.raises(RuntimeError, match="dead"):  # the tape refuses on its own as well
        tape.backward(torch.ones(1, len(grid(30)), 78, device="cuda"), None, [])


def test_backward_after_the_weights_were_reuploaded_raises():
    model = _small("bf16")
    x = torch.randn(1, len(grid(30)), 102, device="cuda")
    opt = torch.optim.SGD(model.parameters(), lr=1e-2)
    with model.multi_step():
        a = model(x)
        b = model(x)
        b.square().mean().backward()
        opt.step()  # changes the weights in place; the next forward uploads them
        c = model(x)
    with pytest.raises(RuntimeError, match="weights were replaced"):
        a.square().mean().backward()
    c.square().mean().backward()


def test_outside_the_window_a_forward_still_replaces_the_tape():
    model = _small()
    x = torch.randn(1, len(grid(30)), 102, device="cuda")
    with model.multi_step():
        w = model(x)
    a = model(x)
    b = model(x)  # replaces the tape of `a`, not the window's
    b.sum().backward()
    with pytest.raises(RuntimeError, match="one backward per forward"):
        a.sum().backward()
    w.sum().backward()
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in model.parameters())


# ---- 5. per-weight work ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_per_weight_work_runs_once_per_upload(tp):
    model = _small(tp)
    x = torch.randn(1, len(grid(30)), 102, device="cuda")
    with model.multi_step():
        ys = [model(x)]
        plan = model._train_engine.plan
        plan.timing_enable(True)
        ys.append(model(x))
        second = plan.timing_read()
        with torch.no_grad():
            next(model.parameters()).add_(1e-3)
        ys.append(model(x))  # new weights: transposes (and images) again
        third = plan.timing_read()
        plan.timing_enable(False)
    assert second["train_weights"][0] == 0, second
    assert third["train_weights"][0] > 0, third
    del ys


# ---- 6. a refused non-finite forward --------------------------------------------------------------------------------------------
def test_non_finite_second_step_leaves_no_tape():
    model = _small("bf16")
    N = len(grid(30))
    x = torch.randn(1, N, 102, device="cuda", requires_grad=True)
    with model.multi_step():
        y1 = model(x)
        x1 = torch.cat([y1, torch.randn(1, N, 24, device="cuda")], -1)
        x1 = x1 + torch.where(torch.arange(102, device="cuda") == 5, float("nan"), 0.0)
        with pytest.raises(RuntimeError, match=BIT3):
            model(x1)
    gc.collect()
    plan = model._train_engine.plan
    assert plan.live_tapes() == [y1.grad_fn.tape]
    y1.square().mean().backward()
    assert all(torch.isfinite(q.grad).all() for q in model.parameters()) and torch.isfinite(x.grad).all()


# ---- 8. 1-degree smoke ---------------------------------------------------------------------------------------------------------
def test_one_degree_bf16_bounded_two_steps():
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll = grid(1)
    torch.manual_seed(0)
    model = GraphWeatherForecaster(ll, train_precision="bf16", use_checkpointing=True).cuda().train()
    crit = NormalizedMSELoss([1.0] * 78, ll, normalize=True)
    g = torch.Generator(device="cuda").manual_seed(3)
    x0 = torch.randn(1, len(ll), 102, device="cuda", generator=g)
    aux1 = torch.randn(1, len(ll), 24, device="cuda", generator=g)
    t1, t2 = (torch.randn(1, len(ll), 78, device="cuda", generator=g) for _ in range(2))
    opt = torch.optim.SGD(model.parameters(), lr=1e-2)

    def two_steps():
        with model.multi_step():
            y1 = model(x0)
            y2 = model(torch.cat([y1, aux1], -1))
        return crit(y1, t1) + crit(y2, t2)

    opt.zero_grad(set_to_none=True)
    loss0 = two_steps()
    loss0.backward()
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in model.parameters())
    opt.step()
    loss1 = two_steps()
    model._train_engine.plan.status()
    print(f"1 deg bf16 bounded, 2 steps: loss {float(loss0):.6f} -> {float(loss1):.6f}")
    assert float(loss1) < float(loss0)
