"""-m gpu: processor segments (`processor.set_checkpoint_segments(N)`, `GraphCast.set_checkpoint_processor(N)`).  A training forward
with segments keeps only the first node and edge rows of every segment of N blocks (-1: one segment) and the processor's output;
its backward recomputes each segment with the forward's own ops before differentiating it.  Only memory and time change:

  * bit-identity: output, the features' gradient and every parameter's gradient equal the step without segments (S = 0) on the
    same weights and inputs, in every train precision, on the taped and the bounded step; the forecaster with 9 blocks (N = 2
    leaves a short last segment), the assimilator, GraphCast under every GraphCastConfig strategy and RegionalForecaster.  The
    gradients the step reduces with float atomics are the exception: LayerNorm weights and biases, Linear layers with at most 16
    inputs (the edge encoders', the assimilator's node encoder's) and, in fp32_simt, every weight gradient -- the S = 0 step does
    not repeat those bit for bit either, so they are held to 1e-6 norm-relative;
  * multi-step: a 3-forward window back-propagates to the same bits, also when S changes between its forwards or between a
    forward and its backward (each tape follows the S its forward ran with);
  * memory: the tape bytes S = 1 and S = -1 save are exactly the processor tensors they drop, computed from the shapes here, and a
    3-tape window's peak is lower with S = 1;
  * failures: a non-finite feature still raises and leaves no tape; a second backward still raises."""
import gc

import numpy as np
import pytest
import torch
from torch import nn

import __graft_entry__ as ge

pytestmark = [pytest.mark.gpu, pytest.mark.training]

PRECISIONS = ["fp32_simt", "fp32", "bf16"]
BIT3 = "a magnitude bound is not finite"  # _capi.Plan.status' text for status bit 3
ATOMIC_BAR = 1e-6


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


def _randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _atomic(model, tp):
    """Names of the parameters whose gradients the step sums with float atomics (not repeatable bit for bit at any S)."""
    if tp == "fp32_simt":
        return {k for k, _ in model.named_parameters()}
    names = set()
    for mname, m in model.named_modules():
        if isinstance(m, nn.LayerNorm) or (isinstance(m, nn.Linear) and m.in_features <= 16):
            names |= {f"{mname}.{k}" for k, _ in m.named_parameters(recurse=False)}
    return names


def _step(model, x, *args):
    """One training forward + a seeded linear loss + backward from cleared gradients: (out, d features, {name: grad}) on the host."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    out = model(xc, *args)
    (out * _randn(out.shape, 5).cuda()).sum().backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters() if q.grad is not None}
    return out.detach().cpu(), xc.grad.cpu(), grads


def _rel(a, b):
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))


def _assert_same(res, ref, atomic, tag):
    out, gx, grads = res
    assert torch.equal(out, ref[0]), f"{tag}: output"
    assert torch.equal(gx, ref[1]), f"{tag}: features' gradient"
    assert grads.keys() == ref[2].keys(), tag
    bad = [k for k in grads if k not in atomic and not torch.equal(grads[k], ref[2][k])]
    assert not bad, f"{tag}: gradients differ: {bad[:5]}"
    worst = max([(_rel(grads[k], ref[2][k]), k) for k in atomic if k in grads and float(ref[2][k].norm()) > 0] or [(0.0, "")])
    assert worst[0] <= ATOMIC_BAR, f"{tag}: {worst}"


def _forecaster(tp, bounded, num_blocks=9):
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(0)
    return GraphWeatherForecaster(_grid(30), num_blocks=num_blocks, train_precision=tp, use_checkpointing=bounded).cuda().train()


# ---- bit-identity -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_forecaster_segments_are_bit_identical(monkeypatch, tp, bounded):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")  # (the bounded step: several chunks on the 72-point grid)
    model = _forecaster(tp, bounded)
    x = _randn((2, len(_grid(30)), 102), 1)
    ref = _step(model, x)
    assert model._train_engine.plan.train_only == bounded
    for s in (-1, 1, 2, 3, 9):
        model.processor.set_checkpoint_segments(s)
        _assert_same(_step(model, x), ref, _atomic(model, tp), f"{tp} bounded={bounded} S={s}")


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_assimilator_segments_are_bit_identical(tp, bounded):
    from graph_weather_b200 import GraphWeatherAssimilator

    torch.manual_seed(0)
    model = GraphWeatherAssimilator(output_lat_lons=_grid(20), analysis_dim=24, num_blocks=4, train_precision=tp,
                                    use_checkpointing=bounded).cuda().train()  # fmt: skip
    rng = np.random.Generator(np.random.PCG64(3))
    n = 200
    obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, n), rng.uniform(0, 360, n), rng.uniform(0, 1, n)], 1).astype(np.float32)).cuda()
    x = _randn((1, n, 2), 2)
    ref = _step(model, x, obs)
    for s in (-1, 1, 3):
        model.processor.set_checkpoint_segments(s)
        _assert_same(_step(model, x, obs), ref, _atomic(model, tp), f"assimilator {tp} bounded={bounded} S={s}")


STRATEGIES = ["no_checkpointing", "full_checkpointing", "balanced_checkpointing", "processor_only_checkpointing",
              "fine_grained_checkpointing"]  # fmt: skip


@pytest.mark.parametrize("tp", PRECISIONS)
def test_graphcast_strategies_are_bit_identical(tp):
    """Each strategy against itself without processor segments (set_checkpoint_processor(0) after it: the step it selects stays),
    and set_checkpoint_processor(2) on the taped step."""
    from graph_weather_b200 import GraphCast, GraphCastConfig

    torch.manual_seed(0)
    model = GraphCast(_grid(30), train_precision=tp).cuda().train()
    x = _randn((2, len(_grid(30)), 78), 4)
    atomic = _atomic(model, tp)
    for strategy in STRATEGIES:
        getattr(GraphCastConfig, strategy)(model)
        segments = model._checkpoint_processor_segments
        bounded = model._bounded_step()
        model.set_checkpoint_processor(0)
        ref = _step(model, x)
        model.set_checkpoint_processor(segments)
        assert model._bounded_step() == bounded
        _assert_same(_step(model, x), ref, atomic, f"GraphCast {tp} {strategy}")
        if strategy in ("balanced_checkpointing", "processor_only_checkpointing"):
            assert segments == -1
    GraphCastConfig.no_checkpointing(model)
    ref = _step(model, x)
    model.set_checkpoint_processor(2)
    _assert_same(_step(model, x), ref, atomic, f"GraphCast {tp} set_checkpoint_processor(2)")
    model.set_checkpoint_processor(0)
    model.processor.set_checkpoint_segments(1)  # the processor's own setting applies when GraphCast's is 0
    assert model._processor_segments() == 1
    _assert_same(_step(model, x), ref, atomic, f"GraphCast {tp} processor.set_checkpoint_segments(1)")


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_regional_segments_are_bit_identical(tp, bounded):
    from graph_weather_b200.regional import RegionalForecasterConfig

    torch.manual_seed(0)
    model = RegionalForecasterConfig(num_blocks=3, train_precision=tp, use_checkpointing=bounded).build().cuda().train()
    ll = [(float(lat), float(lon)) for lat in range(36, 70, 3) for lon in range(-10, 30, 3)]
    x = _randn((2, len(ll), 102), 6)
    ref = _step(model, x, ll)
    for s in (-1, 1, 2):
        model.processor.set_checkpoint_segments(s)
        _assert_same(_step(model, x, ll), ref, _atomic(model, tp), f"regional {tp} bounded={bounded} S={s}")


# ---- multi-step ---------------------------------------------------------------------------------------------------------------------
def _window(model, x, auxs, segments, after=None):
    """Three chained forwards in multi_step(), forward j with processor segments segments[j]; `after` is set before the backward."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    inp, outs = xc, []
    with model.multi_step():
        for j, s in enumerate(segments):
            model.processor.set_checkpoint_segments(s)
            outs.append(model(inp))
            if j + 1 < len(segments):
                inp = torch.cat([outs[-1], auxs[j].cuda()], -1)
    if after is not None:
        model.processor.set_checkpoint_segments(after)
    sum((o * _randn(o.shape, 7 + j).cuda()).sum() for j, o in enumerate(outs)).backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters()}
    return torch.stack([o.detach().cpu() for o in outs]), xc.grad.cpu(), grads


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_multi_step_window(tp, bounded):
    model = _forecaster(tp, bounded, num_blocks=4)
    N = len(_grid(30))
    x = _randn((2, N, 102), 8)
    auxs = [_randn((2, N, 24), 9 + j) for j in range(2)]
    atomic = _atomic(model, tp)
    ref = _window(model, x, auxs, [0, 0, 0])
    _assert_same(_window(model, x, auxs, [1, 1, 1]), ref, atomic, f"{tp} bounded={bounded} S=1")
    _assert_same(_window(model, x, auxs, [1, 0, -1]), ref, atomic, f"{tp} bounded={bounded} S=1,0,-1")
    _assert_same(_window(model, x, auxs, [2, 2, 0], after=1), ref, atomic, f"{tp} bounded={bounded} S changed before the backward")
    _assert_same(_window(model, x, auxs, [0, 0, 0], after=-1), ref, atomic, f"{tp} bounded={bounded} S=0, -1 before the backward")


# ---- memory -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
def test_tape_bytes_follow_the_shapes(bounded):
    """S = 1 drops every block's MLP tapes and per-node sums, the factored layer 1's node terms P and e[nb], and keeps x[1..nb] and
    e[1..nb-1]; S = -1 keeps none of those either.  fp32 bytes, exactly."""
    nb, B = 5, 2
    model = _forecaster("bf16", bounded, num_blocks=nb)
    x = _randn((B, len(_grid(30)), 102), 10).cuda()
    tape_bytes = {}
    for s in (0, 1, -1):
        model.processor.set_checkpoint_segments(s)
        with model.multi_step():
            y = model(x)
        tape_bytes[s] = y.grad_fn.tape.bytes()
        del y
        gc.collect()
    d = model._train_engine.plan.dims
    H, El, Dn, De, Hn, He = d.n_mesh, d.n_lat_edges, d.node_dim, d.edge_dim, d.hidden_node, d.hidden_edge
    per_block = B * El * (2 * He + De) + B * H * De + B * H * (2 * Hn + Dn)  # edge MLP tape, agg, node MLP tape
    assert tape_bytes[0] - tape_bytes[1] == 4 * (B * H * 2 * He + B * El * De + nb * per_block)
    assert tape_bytes[1] - tape_bytes[-1] == 4 * (nb - 1) * (B * H * Dn + B * El * De)
    print(f"bounded={bounded}: tape bytes S=0 {tape_bytes[0]}, S=1 {tape_bytes[1]}, S=-1 {tape_bytes[-1]}")


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
def test_window_peak_is_lower(bounded):
    model = _forecaster("bf16", bounded, num_blocks=4)
    x = _randn((2, len(_grid(30)), 102), 11).cuda()
    peak = {}
    for s in (0, 1):
        model.processor.set_checkpoint_segments(s)
        with model.multi_step():
            ys = [model(x) for _ in range(3)]
        sum(y.square().mean() for y in ys).backward()
        peak[s] = model._train_engine.plan.train_peak_bytes()
        del ys
        gc.collect()
    assert 0 < peak[1] < peak[0], peak


# ---- failures -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_non_finite_feature_raises_and_leaves_no_tape(tp, bounded):
    model = _forecaster(tp, bounded, num_blocks=3)
    model.processor.set_checkpoint_segments(1)
    x = _randn((1, len(_grid(30)), 102), 12)
    x[0, 7, 3] = float("nan")
    with pytest.raises(RuntimeError, match=BIT3):
        model(x.cuda())
    gc.collect()
    assert model._train_engine.plan.live_tapes() == []
    x[0, 7, 3] = 0.0
    out, gx, grads = _step(model, x)  # the next step trains
    assert torch.isfinite(gx).all() and all(torch.isfinite(g).all() for g in grads.values())


def test_second_backward_raises():
    model = _forecaster("bf16", False, num_blocks=3)
    model.processor.set_checkpoint_segments(1)
    x = _randn((1, len(_grid(30)), 102), 13).cuda()
    loss = model(x).square().mean()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="one backward per forward"):
        loss.backward()
    # the C tape itself, consumed by its backward
    plan = model._train_engine.plan
    tape = plan.tape()
    out = torch.empty(1, len(_grid(30)), 78, device="cuda")
    tape.forward(x, out)
    named = [(k, torch.empty_like(q)) for k, q in model.named_parameters()]
    tape.backward(torch.ones_like(out), None, named)
    assert tape.bytes() == 0
    with pytest.raises(RuntimeError, match="one backward per forward"):
        tape.backward(torch.ones_like(out), None, named)
    tape.close()
