"""-m gpu: RegionalForecaster.forward_regions, B regions in one call on one union plan reused from call to call.

  * inference: every output against `forward` on its region alone (fp32_simt bit for bit; fp32 / bf16 against the fp64 oracle),
    stacked and list inputs, nudging on, off and without a context;
  * training, taped and bounded, in every train_precision: outputs, loss and gradients against the per-region steps, overlapping
    regions (the table rows of shared cells are sums), bit-repeatable under torch.use_deterministic_algorithms, SGD on moving boxes;
  * plan reuse: the same plans for a new batch within capacity, no weight-image or weight launches, one growth for a larger batch;
  * safety: a backward after a later call, multi_step(), non-finite features, a non-default stream."""
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from regional_training_oracle import regional_oracle_step
from training_oracle import rel_max

pytestmark = [pytest.mark.gpu, pytest.mark.training]  # (autograd on: the inference tests turn it off themselves)

_TRUNK = dict(feature_dim=9, aux_dim=0, num_blocks=2)  # the 256-wide trunk the tensor-core precisions run, RegionalDataset's 9 channels


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _box(lat0, lon0, k, step=0.5):
    return [(lat0 + step * a, lon0 + step * b) for a in range(k) for b in range(k)]


def _regions(equal):
    """Three boxes: the first two overlap (they share cells); unequal sizes unless `equal`."""
    ks = (9, 9, 9) if equal else (9, 7, 12)
    return [_box(45.0, 0.0, ks[0]), _box(46.5, 1.5, ks[1]), _box(-20.0, 130.0, ks[2])]


def _model(seed=5, **kw):
    from oracle import weights

    from graph_weather_b200.regional import RegionalForecasterConfig

    cfg = dict(_TRUNK, **kw)
    shapes = {k: tuple(v.shape) for k, v in RegionalForecasterConfig(**dict(cfg, precision="fp32_simt")).build().state_dict().items()}
    sd = weights.make_state_dict(shapes, seed)
    m = RegionalForecasterConfig(**cfg).build().cuda()
    m.load_state_dict(sd)
    return m, sd


def _data(regions, F, seed):
    from oracle import weights

    return [weights.make_features(1, len(r), F, seed + i)[0] for i, r in enumerate(regions)]


# ---- inference -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctx", ["off", "nudged", "no_context"])
@pytest.mark.parametrize("equal", [True, False], ids=["stacked", "list"])
@pytest.mark.parametrize("precision", ["fp32_simt", "fp32", "bf16"])
def test_inference_matches_forward_per_region(precision, equal, ctx):
    model, sd = _model(precision=precision, enable_nudging=ctx != "off")
    model.eval()
    regions = _regions(equal)
    xs = [x.cuda() for x in _data(regions, 9, 10)]
    gcs = [g.cuda() for g in _data(regions, 9, 20)] if ctx == "nudged" else None
    with torch.no_grad():
        outs = model.forward_regions(torch.stack(xs) if equal else xs, regions,
                                     (torch.stack(gcs) if equal else gcs) if gcs is not None else None)  # fmt: skip
        if equal:
            assert torch.is_tensor(outs) and outs.shape == (3, len(regions[0]), 9)
        else:
            assert isinstance(outs, list) and [tuple(o.shape) for o in outs] == [(len(r), 9) for r in regions]
        for i, r in enumerate(regions):
            one = model(xs[i][None], r, None if gcs is None else gcs[i][None])[0]
            if precision == "fp32_simt":
                assert torch.equal(outs[i], one), (i, float((outs[i] - one).abs().max()))
                continue
            # fp32: test_regional.py's bar of the CUDA path against the oracle; bf16: the bar of the bf16 tests of this
            # LayerNorm'd output (tests/test_gpu_regional_training.py)
            with torch.enable_grad():
                ref = regional_oracle_step(sd, r, xs[i][None].cpu(), torch.zeros(1, len(r), 9), torch.float64, output_dim=9, num_blocks=2,
                                           global_context=None if gcs is None else gcs[i][None].cpu())[0][0]  # fmt: skip
            bar = 1e-4 if precision == "fp32" else 5e-2
            err, err_one = float((outs[i].double().cpu() - ref).abs().max()), float((one.double().cpu() - ref).abs().max())
            assert err < bar, (i, err, err_one)


# ---- training ------------------------------------------------------------------------------------------------------------------
def _per_region_steps(model, xs, regions, targets):
    """The reference semantics: B single-region training steps, their gradients summed."""
    model.zero_grad(set_to_none=True)
    outs, gxs, loss = [], [], 0.0
    for x, r, t in zip(xs, regions, targets):
        xc = x[None].clone().requires_grad_(True)
        o = model(xc, r)
        li = torch.nn.functional.mse_loss(o, t[None], reduction="sum")
        li.backward()
        outs.append(o.detach()[0]), gxs.append(xc.grad[0])
        loss = loss + float(li)
    grads = {k: q.grad.detach().clone() for k, q in model.named_parameters() if q.grad is not None}
    return outs, loss, gxs, grads


def _batch_step(model, xs, regions, targets):
    model.zero_grad(set_to_none=True)
    xcs = [x.clone().requires_grad_(True) for x in xs]
    outs = model.forward_regions(xcs, regions)
    loss = sum(torch.nn.functional.mse_loss(o, t, reduction="sum") for o, t in zip(outs, targets))
    loss.backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().clone() for k, q in model.named_parameters() if q.grad is not None}
    return [o.detach() for o in outs], float(loss), [x.grad for x in xcs], grads


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_training_matches_the_sum_of_per_region_steps(tp, bounded):
    """The step checked is the second on the union plan: a first step on other, larger regions sets up the plan, so every table the
    step keeps per graph (source-sorted edges, chunk tables) must follow the new regions' graphs."""
    model, sd = _model(train_precision=tp, use_checkpointing=bounded)
    model.train()
    first = [_box(10.0, 10.0, 12), _box(-30.0, -60.0, 12), _box(60.0, 30.0, 12)]
    _batch_step(model, [x.cuda() for x in _data(first, 9, 25)], first, [t.cuda() for t in _data(first, 9, 35)])
    plan, cap = model._train_engine.plan, dict(model._batch_cap)
    regions = _regions(False)
    xs = [x.cuda() for x in _data(regions, 9, 30)]
    ts = [t.cuda() for t in _data(regions, 9, 40)]
    b_out, b_loss, b_gx, b_g = _batch_step(model, xs, regions, ts)
    assert model._train_engine.plan is plan and model._batch_cap == cap  # (the same plan, now on other graphs)
    assert model._train_engine.plan.train_only == bounded
    r_out, r_loss, r_gx, r_g = _per_region_steps(model, xs, regions, ts)
    assert set(b_g) == set(r_g)
    if tp == "fp32_simt":
        for i in range(3):
            assert torch.equal(b_out[i], r_out[i]) and torch.equal(b_gx[i], r_gx[i]), i
        assert b_loss == pytest.approx(r_loss, rel=1e-6)
        bar, out_bar = 1e-4, 0.0
    else:
        # the per-region steps and the union run the same tensor-core arithmetic on other operand bounds (they span all regions):
        # the bars of tests/test_gpu_regional_training.py (fp32: the 1e-2 floor; bf16: the output bar 5e-2, gradients by cosine)
        out_bar = 1e-4 if tp == "fp32" else 5e-2
        bar = 1e-2
        for i in range(3):
            assert float((b_out[i] - r_out[i]).abs().max()) < out_bar, i
        assert b_loss == pytest.approx(r_loss, rel=1e-3 if tp == "fp32" else 5e-2)
    fails = []
    for k in r_g:
        if tp == "bf16":
            c = float(torch.nn.functional.cosine_similarity(b_g[k].double().flatten(), r_g[k].double().flatten(), dim=0))
            if not c > 0.99 and float(r_g[k].abs().max()) > 1e-6:
                fails.append((k, c))
        elif not rel_max(b_g[k], r_g[k]) < bar:
            fails.append((k, rel_max(b_g[k], r_g[k])))
    if tp != "bf16":
        fails += [(f"features {i}", rel_max(b_gx[i], r_gx[i])) for i in range(3) if not rel_max(b_gx[i], r_gx[i]) < bar]
    assert not fails, fails
    # the first two boxes share cells: their table rows are the sums of both regions' rows, and nonzero
    from graph_weather_b200.regional import _RegionGraphs

    cells = [set(_RegionGraphs(model.graph_builder, r).h3_indices.tolist()) for r in regions[:2]]
    shared = sorted(cells[0] & cells[1])
    assert shared and b_g["h3_embeddings"][shared].abs().sum() > 0


def test_fp32_simt_table_gradient_against_the_oracle():
    """Overlapping regions in fp32_simt: the table gradient (rows of shared cells summed) and every other gradient against the sum
    of the fp64 oracle's per-region steps."""
    model, sd = _model(train_precision="fp32_simt")
    model.train()
    regions = _regions(False)
    xs = [x.cuda() for x in _data(regions, 9, 50)]
    ts = [t.cuda() for t in _data(regions, 9, 60)]
    _, _, _, g = _batch_step(model, xs, regions, ts)
    want = {}
    for r, x, t in zip(regions, xs, ts):
        n = x.shape[0] * 9  # (mse_loss's mean over one region -> its sum)
        for k, v in regional_oracle_step(sd, r, x[None].cpu(), t[None].cpu(), torch.float64, output_dim=9, num_blocks=2)[3].items():
            if v is not None:
                want[k] = want.get(k, 0) + v * n
    fails = [(k, rel_max(g[k], want[k])) for k in want if k in g and not rel_max(g[k], want[k]) < 2e-3]
    assert not fails, fails


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_deterministic_steps_repeat_bit_for_bit(tp, bounded):
    model, _ = _model(train_precision=tp, use_checkpointing=bounded)
    model.train()
    regions = _regions(False)
    xs = [x.cuda() for x in _data(regions, 9, 70)]
    ts = [t.cuda() for t in _data(regions, 9, 80)]
    torch.use_deterministic_algorithms(True)
    try:
        a = _batch_step(model, xs, regions, ts)
        b = _batch_step(model, xs, regions, ts)
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(p, q) for p, q in zip(a[0], b[0])) and a[1] == b[1]
    assert all(torch.equal(p, q) for p, q in zip(a[2], b[2]))
    assert all(torch.equal(a[3][k], b[3][k]) for k in a[3]), [k for k in a[3] if not torch.equal(a[3][k], b[3][k])]


@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_sgd_on_moving_boxes_lowers_the_loss(tp):
    model, _ = _model(train_precision=tp)
    model.train()
    opt = torch.optim.SGD(model.parameters(), lr=2e-3)
    rng = np.random.default_rng(0)
    target = lambda x: torch.roll(x, 1, dims=-1)  # noqa: E731  (a fixed map the model can learn)
    losses = []
    for step in range(6):
        regions = [_box(float(rng.uniform(-40, 40)), float(rng.uniform(-150, 150)), int(rng.integers(5, 9))) for _ in range(4)]
        xs = [x.cuda() for x in _data(regions, 9, 100)]  # the same features each step: only the boxes move
        opt.zero_grad(set_to_none=True)
        outs = model.forward_regions(xs, regions)
        loss = sum(torch.nn.functional.mse_loss(o, target(x)) for o, x in zip(outs, xs)) / 4
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses


# ---- plan reuse ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_new_regions_within_capacity_keep_the_plan(precision):
    model, _ = _model(precision=precision)
    model.eval()
    first = _regions(False)
    xs = [x.cuda() for x in _data(first, 9, 110)]
    with torch.no_grad():
        model.forward_regions(xs, first)
        eng = model._batch_engines["infer"]
        plan, cap = eng.plan, dict(model._batch_cap)
        plan.timing_enable(True)
        plan.timing_read()
        uploads = []
        set_weights = plan.set_weights
        plan.set_weights = lambda named: (uploads.append(1), set_weights(named))[1]
        second = [_box(10.0, 10.0, 7), _box(-30.0, -60.0, 7)]
        xs2 = [x.cuda() for x in _data(second, 9, 120)]
        outs = model.forward_regions(xs2, second)
        t = plan.timing_read()
        assert eng.plan is plan and model._batch_cap == cap
        assert not uploads  # no weight upload, so no weight-image repack
        assert t["const"][0] > 0, t  # the per-graph constants ran (the weight images are packed by set_weights only, counted above)
        plan.timing_enable(False)
        assert all(torch.isfinite(o).all() for o in outs)
        # a larger batch grows the capacity once; the batch after it reuses the grown plan
        big = [_box(-50.0 + 10 * i, 5.0 * i, 10) for i in range(8)]
        model.forward_regions([x.cuda() for x in _data(big, 9, 130)], big)
        grown, cap2 = eng.plan, dict(model._batch_cap)
        assert grown is not plan and all(cap2[k] >= cap[k] for k in cap) and cap2 != cap
        model.forward_regions([x.cuda() for x in _data(big[::-1], 9, 140)], big[::-1])
        assert eng.plan is grown and model._batch_cap == cap2


def test_training_plan_is_reused_and_weights_are_not_repacked():
    model, _ = _model(train_precision="bf16")
    model.train()
    first = _regions(False)
    xs = [x.cuda() for x in _data(first, 9, 150)]
    sum(o.sum() for o in model.forward_regions(xs, first)).backward()
    plan = model._train_engine.plan
    plan.timing_enable(True)
    plan.timing_read()
    second = [_box(12.0, 40.0, 7), _box(-35.0, 20.0, 6)]
    sum(o.sum() for o in model.forward_regions([x.cuda() for x in _data(second, 9, 160)], second)).backward()
    t = plan.timing_read()
    plan.timing_enable(False)
    assert model._train_engine.plan is plan
    assert t["train_weights"][0] == 0, t  # (weight transposes and images; "train_pack" is the per-step operand bounds)


# ---- safety --------------------------------------------------------------------------------------------------------------------
def test_backward_after_a_later_call_raises():
    model, _ = _model(train_precision="fp32_simt")
    model.train()
    a, b = _regions(False), [_box(0.0, 0.0, 6)]
    out_a = model.forward_regions([x.cuda() for x in _data(a, 9, 170)], a)
    out_b = model.forward_regions([x.cuda() for x in _data(b, 9, 180)], b)
    with pytest.raises(RuntimeError, match="replaced|consumed"):
        sum(o.sum() for o in out_a).backward()
    sum(o.sum() for o in out_b).backward()  # the last call's backward runs


def test_the_graph_generation_check_in_the_library():
    """The library itself refuses a backward whose tape's union graphs were replaced (the wrapper's own bookkeeping bypassed: a tape
    made directly on the union plan, then another batch uploaded within capacity, with the same weights)."""
    model, _ = _model(train_precision="fp32_simt")
    model.train()
    a, b = _regions(False), [_box(0.0, 0.0, 6)]
    dev = torch.device("cuda", torch.cuda.current_device())
    batch, engines = model._batch(a, dev)
    model.__dict__["_active"] = (batch, engines)
    eng = model._training_engine()
    model.__dict__["_active"] = None
    plan = model._batch_plan(eng, batch, dev)
    tape = plan.tape()
    f = torch.zeros(1, batch.n_obs, 9, device="cuda")
    out = torch.empty(1, batch.n_obs, 9, device="cuda")
    tape.forward(f, out)
    batch2, _ = model._batch(b, dev)
    model._batch_plan(eng, batch2, dev)
    named = [(k, torch.empty_like(v)) for k, v in model._plan_named(batch2) if not k.startswith("nudging")]
    with pytest.raises(RuntimeError, match="graphs or h3_nodes rows were replaced"):
        tape.backward(torch.ones_like(out), None, named)
    tape.close()


def test_multi_step_refuses_training_calls():
    model, _ = _model(train_precision="fp32_simt")
    model.train()
    r = _regions(False)
    xs = [x.cuda() for x in _data(r, 9, 190)]
    with model.multi_step():
        with pytest.raises(NotImplementedError, match="multi_step"):
            model.forward_regions(xs, r)
        with torch.no_grad():
            assert len(model.forward_regions(xs, r)) == 3  # inference is unaffected


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_non_finite_features_raise_and_the_next_call_is_clean(precision, monkeypatch):
    monkeypatch.setenv("GW_B200_CHECK", "1")
    model, sd = _model(precision=precision)
    model.eval()
    r = _regions(False)
    xs = [x.cuda() for x in _data(r, 9, 200)]
    bad = [x.clone() for x in xs]
    bad[1][3, 2] = float("nan")
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="not finite"):
            model.forward_regions(bad, r)
        outs = model.forward_regions(xs, r)
        fresh, _ = _model(precision=precision)
        fresh.eval()
        want = fresh.forward_regions(xs, r)
    assert all(torch.equal(o, w) for o, w in zip(outs, want))


def test_a_call_on_a_non_default_stream():
    model, _ = _model(precision="fp32_simt")
    model.eval()
    r = _regions(False)
    xs = [x.cuda() for x in _data(r, 9, 210)]
    with torch.no_grad():
        want = model.forward_regions(xs, r)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            got = model.forward_regions(xs, r)
        torch.cuda.current_stream().wait_stream(s)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_training_without_train_precision_raises():
    model, _ = _model()
    model.train()
    r = _regions(False)
    with pytest.raises(NotImplementedError, match="train_precision"):
        model.forward_regions([x.cuda().requires_grad_(True) for x in _data(r, 9, 220)], r)
