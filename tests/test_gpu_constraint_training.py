"""-m gpu: training through PhysicalConstraintLayer.  The layer's CUDA backward (gw_constraint_backward) against the reference's
own gradients (tests/golden/constraint_grads.npz) and the torch restatement in fp32 / fp64 (tests/test_constraint_grads.py), and
GraphWeatherForecaster(constraint_type=...) training steps in every train_precision against torch.autograd on the CPU oracle
with the restated layer appended."""
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from test_constraint_grads import _case_ids, fixture_inputs, grid_mapping, load_fixture, restate_grads, rows_to_grid
from training_oracle import check_bf16_bars, check_fp32_bars, forecaster_case, grid, rel_max, rel_norm, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _layer(ll, ctype, exp_factor=1.0):
    from graph_weather_b200 import GraphWeatherForecaster

    m = GraphWeatherForecaster(ll, constraint_type=ctype, feature_dim=4, aux_dim=0, output_dim=4, num_blocks=1).cuda()
    m.constraint.exp_factor = exp_factor
    return m.constraint


def _gpu_grads(layer, hr, lr, dy, form, grid_shape):
    """(out, d_hr, d_lr) of the CUDA layer under autograd, for inputs in the fixture's forms."""
    h = hr.detach().cuda().clone().requires_grad_(True)
    l_ = lr.detach().cuda().clone().requires_grad_(True)
    y = layer(rows_to_grid(h, grid_shape), rows_to_grid(l_, grid_shape)) if form == "rows" else layer(h, l_)
    assert y.grad_fn is not None
    y.backward(dy.cuda())
    return y.detach().cpu(), h.grad.cpu(), l_.grad.cpu()


def _check_against_oracle(ctype, a, hr, lr, dy, got, grid_shape, cell, last, rows, what=""):
    _, d_hr32, d_lr32 = restate_grads(ctype, hr, lr, dy, grid_shape, cell, last, a, torch.float32, rows=rows)
    _, d_hr64, d_lr64 = restate_grads(ctype, hr, lr, dy, grid_shape, cell, last, a, torch.float64, rows=rows)
    _, g_hr, g_lr = got
    e_lr, r_lr = rel_max(g_lr, d_lr64), rel_max(d_lr32, d_lr64)
    assert e_lr <= max(10 * r_lr, 2e-6), (what, "d_lr", e_lr, r_lr)
    if ctype == "softmax":
        # d_hr is analytically 0: both are rounding noise, ours within a few times the reference's own noise
        noise = 4 * float(d_hr32.abs().max()) + 1e-7 * float(dy.abs().max() * lr.abs().max() * a)
        assert float(g_hr.abs().max()) <= noise, (what, float(g_hr.abs().max()), noise)
    else:
        e_hr, r_hr = rel_max(g_hr, d_hr64), rel_max(d_hr32, d_hr64)
        assert e_hr <= max(10 * r_hr, 2e-6), (what, "d_hr", e_hr, r_hr)
    return d_hr32, d_lr32


@pytest.fixture(scope="module")
def fixture_case(golden_dir):
    z, cfg = load_fixture(golden_dir)
    ll = [(a, b) for a in cfg["lats"] for b in cfg["lons"]]
    return z, cfg, ll, grid_mapping(ll)


@pytest.mark.parametrize("case", range(12))
def test_layer_gradients_match_the_reference(fixture_case, case):
    """Graph (3D), grid (4D) and the forecaster's rearranged (4D) inputs on the irregular grid (shared and empty cells)."""
    z, cfg, ll, (grid_shape, cell, last) = fixture_case
    ctype, a, form, key = _case_ids(cfg)[case]
    hr, lr, dy = fixture_inputs(z, cfg, ctype, form, grid_shape, cell, last)
    got = _gpu_grads(_layer(ll, ctype, a), hr, lr, dy, form, grid_shape)
    assert got[1].shape == hr.shape and got[2].shape == lr.shape
    assert float((got[0] - torch.from_numpy(z[key + "_out"])).abs().max()) <= 1e-5 * max(1.0, float(np.abs(z[key + "_out"]).max()))
    _check_against_oracle(ctype, a, hr, lr, dy, got, grid_shape, cell, last, form == "rows", key)
    # the reference's own gradients, at the same bars relative to their scale
    for g, what in ((got[1], "_d_hr"), (got[2], "_d_lr")):
        ref = torch.from_numpy(z[key + what])
        scale = float(torch.from_numpy(z[key + "_d_lr"]).abs().max()) if ctype == "softmax" else float(ref.abs().max())
        assert float((g - ref).abs().max()) <= 1e-5 * scale, (key, what)
    # rows (or grid cells) no node reads get exactly 0
    H, W = grid_shape
    if form == "graph":
        unread = torch.ones(hr.shape[1], dtype=torch.bool)
        unread[last[cell]] = False
        assert unread.any()
        assert torch.all(got[1][:, unread] == 0) and torch.all(got[2][:, unread] == 0)
    else:
        unread = torch.ones(H * W, dtype=torch.bool)
        unread[cell] = False
        assert unread.any()
        flat = (lambda t: t.reshape(t.shape[0], -1, H * W).transpose(1, 2)) if form == "grid" else (lambda t: t)
        assert torch.all(flat(got[1])[:, unread] == 0) and torch.all(flat(got[2])[:, unread] == 0)


def _regular(step_lat=20, step_lon=22.5):
    lats = [-70.0 + step_lat * i for i in range(8)]
    lons = [step_lon * j for j in range(16)]
    return [(a, b) for a in lats for b in lons]


@pytest.mark.parametrize("ctype,a", [("additive", 1.0), ("multiplicative", 1.0), ("softmax", 1.0), ("softmax", 0.5)])
def test_layer_on_the_10_degree_grid(ctype, a):
    """B = 2, C = 78 rows as the forecaster passes them (lr = the first 78 of 102 feature columns, a strided view)."""
    ll = grid(10)
    grid_shape, cell, last = grid_mapping(ll)
    g = torch.Generator().manual_seed(5)
    hr = torch.randn(2, len(ll), 78, generator=g)
    feats = torch.randn(2, len(ll), 102, generator=g)
    if ctype == "multiplicative":
        hr, feats = hr + 3, feats + 3
    dy = torch.randn(2, len(ll), 78, generator=g)
    layer = _layer(ll, ctype, a)
    h = hr.cuda().requires_grad_(True)
    f = feats.cuda().requires_grad_(True)
    y = layer.constrain_rows(h, f[..., :78], cell.to(torch.int32).cuda())
    y.backward(dy.cuda())
    assert torch.all(f.grad[..., 78:] == 0)
    got = (y.detach().cpu(), h.grad.cpu(), f.grad[..., :78].cpu())
    _check_against_oracle(ctype, a, hr, feats[..., :78], dy, got, grid_shape, cell, last, True, ctype)


def test_additive_exact_integers_bit_for_bit():
    """Exact-integer dy and N = 128 (a power of two): every term is exact, so the fp64 result rounds to the same bits."""
    ll = _regular()
    grid_shape, cell, last = grid_mapping(ll)
    g = torch.Generator().manual_seed(3)
    hr = torch.randn(2, len(ll), 5, generator=g)
    lr = torch.randn(2, len(ll), 5, generator=g)
    dy = torch.randint(-8, 9, (2, len(ll), 5), generator=g).float()
    got = _gpu_grads(_layer(ll, "additive"), hr, lr, dy, "rows", grid_shape)
    _, d_hr64, d_lr64 = restate_grads("additive", hr, lr, dy, grid_shape, cell, last, 1.0, torch.float64, rows=True)
    assert torch.equal(got[1], d_hr64.float()) and torch.equal(got[2], d_lr64.float())


def test_additive_gradient_sums_to_zero():
    """y = hr + lr - mean(hr): shifting hr by a constant leaves y unchanged, so sum_r d_hr = 0 per sample and channel."""
    ll = grid(10)
    grid_shape, _, _ = grid_mapping(ll)
    g = torch.Generator().manual_seed(4)
    hr, lr, dy = (torch.randn(2, len(ll), 78, generator=g) for _ in range(3))
    _, d_hr, _ = _gpu_grads(_layer(ll, "additive"), hr, lr, dy, "rows", grid_shape)
    s = d_hr.double().sum(dim=1)
    assert float(s.abs().max()) <= 1e-5 * float(dy.abs().sum(dim=1).max())


def _crowded():
    """Eight of nine latitudes truncate to grid row 0 (forecast.py:182-186): its cells are read by 8 or 16 nodes, rows 1-7 by none."""
    lats = [-80.0 + 0.5 * i for i in range(8)] + [80.0]
    return [(a, b) for a in lats for b in (0.0, 50.0, 130.0, 200.0, 290.0, 350.0)]


@pytest.mark.parametrize("ctype", ["additive", "multiplicative", "softmax"])
def test_backward_is_repeatable(ctype):
    """Repeated backward calls give identical bits where many nodes share a row (an unordered sum would not)."""
    ll = _crowded()
    grid_shape, cell, _ = grid_mapping(ll)
    assert int(np.bincount(cell.numpy()).max()) >= 8
    g = torch.Generator().manual_seed(8)
    hr, lr, dy = (torch.randn(8, len(ll), 96, generator=g) * 10 ** torch.randint(-3, 4, (8, len(ll), 96), generator=g) for _ in range(3))
    if ctype == "multiplicative":
        hr, lr = hr.abs() + 3, lr.abs() + 3
    if ctype == "softmax":
        hr = hr.clamp(-20, 20)
    layer = _layer(ll, ctype)
    for form in ("rows", "graph"):
        runs = [_gpu_grads(layer, hr, lr, dy, form, grid_shape) for _ in range(3)]
        for r in runs[1:]:
            assert torch.equal(runs[0][1], r[1]) and torch.equal(runs[0][2], r[2]), form


def test_softmax_non_finite_where_the_oracle_has_them(fixture_case):
    """exp overflows (inf * 0 = nan downstream) and underflows (1 / 0 = inf): in every row some node reads, the same entries are
    non-finite as in fp32 autograd.  Rows no node reads get exactly 0 even where exp overflowed there: the reference's autograd
    gives 0 * inf = nan for such a row (its upstream gradient is 0), which is not a gradient anyone could use."""
    z, cfg, ll, (grid_shape, cell, last) = fixture_case
    g = torch.Generator().manual_seed(9)
    hr, lr, dy = (torch.randn(2, len(ll), 4, generator=g) for _ in range(3))
    # node 3's row is read by no node in either form (grid column 3 is empty; in graph form node 9 overwrites node 3's cell)
    hr[0, 3, 1], hr[1, 7, 0], hr[1, 0, 2], hr[0, 1, 3], hr[1, 8, 1] = 200.0, 150.0, -300.0, 120.0, 95.0
    for form in ("rows", "graph"):
        src = cell if form == "rows" else last[cell]
        read = torch.zeros(len(ll), dtype=torch.bool)
        read[src] = True
        assert not read[3]
        got = _gpu_grads(_layer(ll, "softmax"), hr, lr, dy, form, grid_shape)
        _, r_hr, r_lr = restate_grads("softmax", hr, lr, dy, grid_shape, cell, last, 1.0, torch.float32, rows=form == "rows")
        assert not torch.isfinite(r_hr[:, read]).all()
        assert torch.equal(torch.isfinite(got[1][:, read]), torch.isfinite(r_hr[:, read])), form
        assert torch.equal(torch.isfinite(got[2][:, read]), torch.isfinite(r_lr[:, read])), form
        assert torch.all(got[1][:, ~read] == 0) and torch.all(got[2][:, ~read] == 0), form


def test_no_grad_path_is_unchanged(fixture_case):
    """Inputs that do not require grad take the inference path (no autograd node), as before."""
    z, cfg, ll, (grid_shape, cell, last) = fixture_case
    layer = _layer(ll, "additive")
    hr, lr = torch.from_numpy(z["hr"]).cuda(), torch.from_numpy(z["lr"]).cuda()
    y = layer(hr, lr)
    assert y.grad_fn is None
    y2 = layer(hr.clone().requires_grad_(True), lr)
    assert y2.grad_fn is not None and torch.equal(y, y2.detach())


# ---- the forecaster ---------------------------------------------------------------------------------------------------------------
SHIFT = {"additive": 0.0, "multiplicative": 3.0, "softmax": 0.0}


def _case(ctype):
    """The seeded 10-degree, batch-2 case of tests/test_gpu_train_precision.py (the first 78 input channels shifted by SHIFT[ctype])
    and its oracle steps, with the restated layer appended, in fp32 and fp64."""
    return forecaster_case(10, 2, 21, constraint=ctype, shift=SHIFT[ctype])


def _step(ctype, tp, ll, sd, x, target, var):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    model = GraphWeatherForecaster(ll, constraint_type=ctype, train_precision=tp).cuda().train()
    model.load_state_dict(sd)
    return train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target)


# Additive on tensor cores.  y = hr + lr - mean(hr) centres the gradient entering the network (sum_r d_hr = 0 per sample and channel,
# so the last decoder bias gets an analytically zero gradient, skipped below like any numerically zero one).  A gradient summed over
# all rows of a centred dY cancels its large common part: the fp32 oracle keeps ~1e-6 there, but the operands the tensor-core
# training path rounds (fp16 hi/lo split, bf16) leave an error of the common part's size.  Measured on an H100 (10-degree case):
# fp32 mode worst max-relative 1.3e-2 (decoder block-0 edge MLP, the fp32 oracle at 2.9e-6), norm-relative 3.3e-3; bf16 worst
# per-parameter cosine 0.945 (decoder block 0).  Those errors belong to the network's backward, not to the layer: the same
# gradients come out of the unconstrained network's backward fed the layer's d_hr (test_constrained_step_is_the_network_backward_
# of_the_layer_gradient).  So on tensor cores the additive case holds each parameter to bars about twice the measured error:
# norm-relative 1e-2 in fp32, cosine 0.9 in bf16.
ADDITIVE_TC_NORM, ADDITIVE_TC_COS = 1e-2, 0.9


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
@pytest.mark.parametrize("ctype", ["additive", "multiplicative", "softmax"])
def test_constrained_training_step_matches_the_oracle(ctype, tp):
    ll, sd, x, target, var, ref32, ref64 = _case(ctype)
    out, loss, gx, grads = _step(ctype, tp, ll, sd, x, target, var)
    assert len(grads) == 215
    tag = f"{ctype} {tp}"
    # features.grad: the network's paths plus the layer's lr path.  Softmax: the layer returns lr up to rounding, so d out / d hr
    # is 0 and every parameter gradient is rounding noise: those are measured against the unconstrained step below instead (not
    # against the additive step, whose last decoder bias has a zero gradient of its own).
    ours = (out, loss, gx, None if ctype == "softmax" else grads)
    if tp == "bf16":
        cos_bar, ill_cos_bar = (ADDITIVE_TC_COS, ADDITIVE_TC_COS) if ctype == "additive" else (0.99, 0.98)
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=cos_bar, ill_cos_bar=ill_cos_bar, feat_cos=0.99, total_cos=None,
                        tag=tag)  # fmt: skip
    else:
        # numerically zero gradients (additive: the last decoder bias) are left out: their direction is noise
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3, feat_floor=True, median=False, ill="max", skip_zero=True,
                        norm_bar=ADDITIVE_TC_NORM if (ctype, tp) == ("additive", "fp32") else None, tag=tag)  # fmt: skip
    if ctype == "softmax":
        _, _, _, g_plain = _step("none", tp, ll, sd, x, target, var)
        worst = 0.0
        for k, gr in grads.items():
            assert torch.isfinite(gr).all(), k
            ratio = float(gr.abs().max()) / (float(g_plain[k].abs().max()) + 1e-30)
            worst = max(worst, ratio)
            assert ratio <= 1e-4, (k, ratio)
        print(f"softmax {tp}: worst max|grad| / unconstrained {worst:.2e}")


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
@pytest.mark.parametrize("ctype", ["additive", "multiplicative"])
def test_constrained_step_is_the_network_backward_of_the_layer_gradient(ctype, tp):
    """The parameter gradients of a constrained step are those of the unconstrained network's backward fed the layer's d_hr: bit for
    bit where the tensor-core weight gradients reduce in a fixed order (the processor's Linear layers), to atomics' rounding elsewhere."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = _case(ctype)[:5]
    xc = x.cuda()
    model = GraphWeatherForecaster(ll, constraint_type=ctype, train_precision=tp).cuda().train()
    model.load_state_dict(sd)
    out = model(xc)
    out.retain_grad()
    NormalizedMSELoss(var, ll, normalize=True)(out, target.cuda()).backward()
    model._train_engine.plan.status()
    plain = GraphWeatherForecaster(ll, train_precision=tp).cuda().train()
    plain.load_state_dict(sd)
    hr = plain(xc)
    layer = model.constraint
    hr32, lr32 = layer._prepare(hr, xc[..., :78])
    d_hr, d_lr = layer._backward(out.grad, hr32, lr32, model._constraint_cell(hr32), False)
    assert d_lr is None
    hr.backward(d_hr)
    plain._train_engine.plan.status()
    pg = dict(plain.named_parameters())
    linear = 0
    for k, q in model.named_parameters():
        a, b = q.grad, pg[k].grad
        if k.startswith("processor.") and any(f".model.{i}." in k for i in (0, 2, 4)):
            assert torch.equal(a, b), k
            linear += 1
        else:
            assert rel_norm(a, b) <= 1e-5, (k, rel_norm(a, b))
    assert linear > 100


@pytest.mark.parametrize("ctype", ["additive", "multiplicative", "softmax"])
def test_constrained_train_output_is_the_layer_on_the_plain_output(ctype):
    """Bit for bit: the constrained train-mode output is apply_rows (no grad) on the unconstrained train-mode output."""
    from graph_weather_b200 import GraphWeatherForecaster

    ll, sd, x = _case(ctype)[:3]
    outs = {}
    for c in (ctype, "none"):
        model = GraphWeatherForecaster(ll, constraint_type=c, train_precision="fp32").cuda().train()
        model.load_state_dict(sd)
        outs[c] = (model, model(x.cuda().requires_grad_(True)))
    model, y = outs[ctype]
    assert y.grad_fn is not None
    cell = model._grid_mapping.tensors(y.device)[0].to(torch.int32)
    with torch.no_grad():
        ref = model.constraint.apply_rows(outs["none"][1].detach(), x.cuda(), cell, 78)
    assert torch.equal(y.detach(), ref)


def test_loss_falls_at_one_degree():
    """1-degree grid, additive constraint, bf16: four AdamW steps on a fixed batch lower the loss (seeded weights, as the
    1-degree step of tests/test_gpu_train_precision.py)."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss
    from oracle import weights

    ll = grid(1)
    model = GraphWeatherForecaster(ll, constraint_type="additive", train_precision="bf16").cuda().train()
    model.load_state_dict(weights.make_state_dict(weights.forecaster_shapes(), 5))
    crit = NormalizedMSELoss([1.0] * 78, ll, normalize=True)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    x = weights.make_features(1, len(ll), 102, 5).cuda()
    rng = np.random.Generator(np.random.PCG64(5))
    y = torch.from_numpy(rng.standard_normal((1, len(ll), 78)).astype(np.float32)).cuda()
    losses = []
    for _ in range(4):
        opt.zero_grad(set_to_none=True)
        loss = crit(model(x), y)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    model._train_engine.plan.status()
    print("1 deg additive bf16 losses", losses)
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
