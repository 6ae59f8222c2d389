"""-m gpu: RegionalForecaster trains (RegionalForecasterConfig.train_precision).  In train mode with autograd on, a forward runs the
forecaster's CUDA training step on training plans of the region; the boundary nudging layer is differentiated by torch.

  * the one-layer training row op with a LayerNorm over N real columns of a padded chain (the node decoder's output layer:
    N = output_dim), with a residual that is the first N columns of a wider row, in every precision and on both chain paths;
  * the reference suite's small config against one training step of the reference's own code (regional_small_grads.npz);
  * the default 256-wide trunk with output_dim 78 and 9 against the fp32 / fp64 oracle, in every train_precision, taped and bounded,
    with and without a global context;
  * the losses of more regions than the plan cache holds, summed into one backward; a two-step rollout in multi_step();
  * an SGD step lowers the loss, and inference after training equals a fresh model's."""
import json
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import test_gpu_kernels as tk
from test_gpu_kernels import BARS, EXACT, FLOAT, PREC_NAME, RUNS, Data, RowOp, _eps, bcast, gpu, stream
from regional_training_oracle import check_bf16_bars_ln_out, plan_names, regional_oracle_step
from training_oracle import check_fp32_bars, rel_max

pytestmark = [pytest.mark.gpu, pytest.mark.training]

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    """The kernel harness RowOp runs through (tests/test_gpu_kernels.py)."""
    tk.HK = tk._compile_harness(tmp_path_factory.mktemp("gw_regional_harness"))
    return tk.HK


# ---- the kernel: a LayerNorm over n_valid < N columns in the one-layer training chain ---------------------------------------
LN_N = [9, 12, 78, 250, 256]  # (256: no padding, the control)


def _ln_op(d, N, res_kind, rows=300, batch=2):
    """The node decoder's output layer: K = 128 hidden columns -> N outputs, LayerNorm, + the first N columns of a wider feature row
    (stream: per sample; bcast: shared).  out and save_pre rows are 5 columns wider than N: those columns must stay untouched."""
    R = rows * batch
    wide = N + 24
    res = stream(d.addend(R, wide), rows, width=N) if res_kind == "stream" else bcast(d.addend(rows, wide), width=N)
    g = torch.rand(N, generator=d.g, device="cuda") + 0.5
    b = torch.randn(N, generator=d.g, device="cuda") * 0.1
    return RowOp(rows, batch, [stream(d.operand(R, 128), rows)], d.weight(N, 128), 128, N, bias=d.addend(N), ln=(g, b), residual=res,
                 save_pre=True, ldo=N + 5)  # fmt: skip


def _untouched(t, N):
    return bool(torch.isnan(t[:, N:]).all())  # (RowOp.run fills out and save_pre with NaN first)


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("res_kind", ["stream", "bcast"])
@pytest.mark.parametrize("N", LN_N)
def test_layernorm_row_op_exact(N, res_kind, data):
    """Exact-integer data: the taped pre-LayerNorm value bit for bit, the normalised output within 1e-5 (eps_F), columns beyond N
    untouched, in every precision and with and without GW_TC3_NOFAST."""
    d = Data(3000 + N + (7 if res_kind == "bcast" else 0), **data)
    op = _ln_op(d, N, res_kind)
    y64, pre64, _ = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, pre, _ = op.run(prec, nofast)
        tag = f"N={N} {res_kind} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
        if not torch.equal(pre[:, :N].double(), pre64):
            fails.append(f"{tag}: pre-LayerNorm values differ")
        ef = float((out[:, :N].double() - y64).norm() / y64.norm())
        if not ef < 1e-5:
            fails.append(f"{tag}: LayerNorm output eps_F {ef:.2e}")
        if not (_untouched(out, N) and _untouched(pre, N)):
            fails.append(f"{tag}: columns beyond N were written")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("res_kind", ["stream", "bcast"])
@pytest.mark.parametrize("N", LN_N)
def test_layernorm_row_op_float(N, res_kind, data):
    """Random floats under the bars of test_gpu_kernels.test_row_op_float: the pre-LayerNorm value under both bars, the normalised
    output under the eps_F bar; columns beyond N untouched."""
    d = Data(4000 + N + (7 if res_kind == "bcast" else 0), **data)
    op = _ln_op(d, N, res_kind)
    y64, pre64, c = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, pre, _ = op.run(prec, nofast)
        bf, bel = BARS[prec]
        tag = f"N={N} {res_kind} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
        ef, eel = _eps(pre[:, :N], pre64, c)
        efo = float((out[:, :N].double() - y64).norm() / y64.norm())
        print(f"{tag}: eps_F {ef:.2e} eps_el {eel:.2e}; LayerNorm output eps_F {efo:.2e}")
        if not (ef < bf and eel < bel and efo < bf):
            fails.append(f"{tag}: eps_F {ef:.2e} eps_el {eel:.2e} output eps_F {efo:.2e}")
        if not (_untouched(out, N) and _untouched(pre, N)):
            fails.append(f"{tag}: columns beyond N were written")
    assert not fails, fails


# ---- models ------------------------------------------------------------------------------------------------------------------
def _build(sd, **kw):
    from graph_weather_b200.regional import RegionalForecasterConfig

    model = RegionalForecasterConfig(**kw).build().cuda().train()
    model.load_state_dict(sd)
    return model


def _step(model, x, lat_lons, target, gc=None):
    """One training forward + MSE + backward on the GPU from cleared gradients: (out, loss, d features, {name: grad}) on the host,
    parameters torch leaves without a gradient (the nudging layer without a context) left out."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    out = model(xc, lat_lons, global_context=None if gc is None else gc.cuda())
    assert out.requires_grad
    loss = torch.nn.functional.mse_loss(out, target.cuda())
    loss.backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters() if q.grad is not None}
    return out.detach().cpu(), float(loss.detach()), xc.grad.cpu(), grads


def _present(ref):
    out, loss, gx, g = ref
    return out, loss, gx, {k: v for k, v in g.items() if v is not None}


_SMALL = dict(feature_dim=12, aux_dim=4, node_dim=32, edge_dim=32, num_blocks=2, hidden_dim_processor_node=32, hidden_dim_processor_edge=32,
              hidden_dim_decoder=32)  # fmt: skip


@pytest.fixture(scope="module")
def small_fixture():
    """regional_small_grads.npz: the reference's own training step of the small config with nudging (UK region, batch 2)."""
    z = np.load(os.path.join(HERE, "golden", "regional_small_grads.npz"))
    cfg = json.loads(str(z["config"]))
    idx = torch.from_numpy(z["h3_indices"])
    sd = {}
    for k, shape in zip(cfg["keys"], cfg["shapes"]):
        w = torch.from_numpy(z["w." + k])
        sd[k] = torch.zeros(shape).index_copy_(0, idx, w) if k == "h3_embeddings" else w
    x, gc, target = (torch.from_numpy(z[k]) for k in ("x", "global_context", "target"))
    ll = [tuple(p) for p in cfg["lat_lons"]]
    ref64 = regional_oracle_step(sd, ll, x, target, torch.float64, output_dim=12, num_blocks=2, global_context=gc)
    return z, idx, sd, ll, x, gc, target, ref64


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
def test_small_config_matches_the_reference_training_step(small_fixture, bounded):
    """fp32_simt against the reference's own step: output and loss within 1e-5, every gradient within 10x the reference's own fp32
    error against fp64 (+ 1e-5).  Then the reference suite's test_backward_pass / test_nudging_backward_pass assertions."""
    z, idx, sd, ll, x, gc, target, ref64 = small_fixture
    model = _build(sd, **_SMALL, enable_nudging=True, train_precision="fp32_simt", use_checkpointing=bounded)
    out, loss, gx, grads = _step(model, x, ll, target, gc)
    assert model._train_engine.plan.train_only == bounded
    assert float((out - torch.from_numpy(z["out"])).abs().max()) < 1e-5
    assert abs(loss - float(z["loss"])) < 1e-5
    _, _, gx64, g64 = ref64
    pairs = [("features", gx, gx64, torch.from_numpy(z["grad_x"]))]
    off = torch.ones(grads["h3_embeddings"].shape[0], dtype=torch.bool)
    off[idx] = False
    assert not grads["h3_embeddings"][off].any()  # zero off the region
    for k, g in grads.items():
        if k == "h3_embeddings":
            pairs.append((k, g[idx], g64[k][idx], torch.from_numpy(z["g." + k])))
        else:
            pairs.append((k, g, g64[k], torch.from_numpy(z["g." + k])))
    assert len(grads) == len(g64)
    fails = []
    for k, ours, exact, fix in pairs:
        e_ours, e_fix = rel_max(ours, fix), rel_max(fix, exact)
        if not e_ours < 10 * e_fix + 1e-5:
            fails.append((k, e_ours, e_fix))
    assert not fails, fails
    # the reference suite's assertions (tests/test_regional_forecast.py:87-99, :187-198), on the real values
    assert model.h3_embeddings.grad is not None and model.h3_embeddings.grad[idx].abs().sum() > 0
    assert any(q.grad is not None and q.grad.abs().sum() > 0 for q in model.node_encoder.parameters())
    assert any(q.grad is not None and q.grad.abs().sum() > 0 for q in model.nudging.parameters())


def _europe():
    z = np.load(os.path.join(HERE, "golden", "regional_europe_b2.npz"))
    return [(float(a), float(b)) for a, b in z["lat_lons"]]


_CASES = {}


def trunk_case(out_dim, with_gc):
    """The default 256-wide trunk with 2 processor blocks on the Europe region (2445 points, batch 2): output_dim 78 (78 + 24
    features) or 9 (9 + 0, the shape of RegionalDataset's samples); nudging on when a global context is given.  (lat_lons,
    state_dict, model kwargs, features, global context, target, oracle step in fp32, in fp64)."""
    key = (out_dim, with_gc)
    if key not in _CASES:
        from oracle import weights

        from graph_weather_b200.regional import RegionalForecasterConfig

        ll = _europe()
        kw = dict(num_blocks=2, enable_nudging=with_gc, **(dict(feature_dim=9, aux_dim=0) if out_dim == 9 else {}))
        shapes = {k: tuple(v.shape) for k, v in RegionalForecasterConfig(**kw).build().state_dict().items()}
        seed = 40 + out_dim + with_gc
        sd = weights.make_state_dict(shapes, seed)
        F = out_dim + (24 if out_dim == 78 else 0)
        x = weights.make_features(2, len(ll), F, seed)
        gc = weights.make_features(2, len(ll), out_dim, seed + 1) if with_gc else None
        target = weights.make_features(2, len(ll), out_dim, seed + 2)
        refs = [regional_oracle_step(sd, ll, x, target, dt, output_dim=out_dim, num_blocks=2, global_context=gc)
                for dt in (torch.float32, torch.float64)]  # fmt: skip
        _CASES[key] = (ll, sd, kw, x, gc, target, *[_present(r) for r in refs])
    return _CASES[key]


@pytest.mark.parametrize("with_gc", [False, True], ids=["plain", "nudged"])
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
@pytest.mark.parametrize("out_dim", [78, 9])
def test_default_trunk_matches_the_oracle(out_dim, tp, bounded, with_gc):
    ll, sd, kw, x, gc, target, ref32, ref64 = trunk_case(out_dim, with_gc)
    model = _build(sd, **kw, train_precision=tp, use_checkpointing=bounded)
    ours = _step(model, x, ll, target, gc)
    assert model._train_engine.plan.train_only == bounded and model._train_engine.resolved_precision == tp
    g = ours[3]["h3_embeddings"]
    region = torch.zeros(g.shape[0], dtype=torch.bool)
    region[torch.tensor(model._regions[id(ll)][1].h3_indices)] = True
    assert not g[~region].any()  # exactly zero off the region
    n = len(ref64[3])
    tag = f"out_dim={out_dim} {tp} {'bounded' if bounded else 'taped'} {'nudged' if with_gc else 'plain'}"
    if tp == "bf16":
        # The gradient bars of the forecaster's bf16 tests (tests/test_gpu_lean_training.py); measured on an H100 worst cosines
        # 0.9933 (h3_embeddings), 0.9948 (node_encoder.model.0.weight), above 0.9989 elsewhere, features 0.9986.  The output bar is
        # 5e-2 instead of 2e-2: this model's output is LayerNorm'd (values up to ~4 on unit scale), which scales the bf16 error of
        # the value it normalises by 1 / std; measured worst 3.3e-2 max-abs over the 381k outputs of out_dim 78, 2.8e-2 for 9.
        check_bf16_bars_ln_out(plan_names(ours), plan_names(ref32), plan_names(ref64), out_bar=5e-2, cos_bar=0.99, ill_cos_bar=0.98,
                               feat_cos=0.99, tag=tag)  # fmt: skip
        return
    # fp32 mode: the 1e-2 floor of GraphCast's and the forecaster's tensor-core tests, for ReLU units within ~1e-6 of zero that
    # switch between two fp32 implementations; fp32_simt: the 2e-3 floor of tests/test_gpu_dense_cell_training.py.  Measured on an
    # H100: fp32 worst 1.1e-3 (decoder_gnn edge MLP), h3_embeddings 8.3e-3 against its 5x bar of 1.7e-2; fp32_simt worst 1.1e-3
    # (edge_encoder.model.0.weight, output_dim 9), h3_embeddings 4.0e-3 against its 5x bar.  (Under the plan's names the
    # ill-conditioned parameters are training_oracle.ILL_CONDITIONED's.)
    check_fp32_bars(plan_names(ours), plan_names(ref32), plan_names(ref64), n_params=n, floor=1e-2 if tp == "fp32" else 2e-3, feat_floor=False, median=False, ill="max",
                    skip_zero=True, norm_bar=None, tag=tag)  # fmt: skip


def _boxes(k, n=6):
    """n small regions of k x k points at 1-degree spacing, each its own list (and graphs)."""
    return [[(40.0 + 3 * i + 0.5 * a, -10.0 + 4 * i + 0.5 * b) for a in range(k) for b in range(k)] for i in range(n)]


def test_many_regions_one_backward():
    """The losses of 6 regions (more than the 4 the cache keeps) summed into one backward: every gradient equals the sum of the six
    oracle steps' (fp64), no 'plan was replaced', and the cache shrinks back to 4 regions at the next forward."""
    from oracle import weights

    from graph_weather_b200.regional import RegionalForecaster, RegionalForecasterConfig

    regions = _boxes(5)
    shapes = {k: tuple(v.shape) for k, v in RegionalForecasterConfig(**_SMALL).build().state_dict().items()}
    sd = weights.make_state_dict(shapes, 61)
    model = _build(sd, **_SMALL, train_precision="fp32_simt")
    xs = [weights.make_features(1, len(r), 16, 62 + i) for i, r in enumerate(regions)]
    ts = [weights.make_features(1, len(r), 12, 70 + i) for i, r in enumerate(regions)]
    loss = 0.0
    for r, x, t in zip(regions, xs, ts):
        loss = loss + torch.nn.functional.mse_loss(model(x.cuda(), r), t.cuda())
    assert len(model._regions) == 6 > RegionalForecaster._MAX_PLANS
    loss.backward()
    want = {}
    for r, x, t in zip(regions, xs, ts):
        for k, g in regional_oracle_step(sd, r, x, t, torch.float64, output_dim=12, num_blocks=2)[3].items():
            want[k] = want.get(k, 0) + g
    fails = [(k, rel_max(q.grad, want[k])) for k, q in model.named_parameters() if not rel_max(q.grad, want[k]) < 1e-4]
    assert not fails, fails
    with torch.no_grad():
        model(xs[0].cuda(), regions[0])
    assert len(model._regions) == RegionalForecaster._MAX_PLANS


def test_two_step_rollout():
    """Two forwards on one region inside multi_step(), the second fed the first's output and the auxiliary columns, one backward:
    the gradients of the unrolled loss (fp64 oracle), in fp32_simt within 1e-4 max-relative."""
    from oracle import weights

    from graph_weather_b200.regional import RegionalForecasterConfig

    r = _boxes(6, 1)[0]
    shapes = {k: tuple(v.shape) for k, v in RegionalForecasterConfig(**_SMALL).build().state_dict().items()}
    sd = weights.make_state_dict(shapes, 81)
    model = _build(sd, **_SMALL, train_precision="fp32_simt")
    x = weights.make_features(2, len(r), 16, 82)
    t = torch.stack([weights.make_features(2, len(r), 12, 83 + i) for i in range(2)])
    xc = x.cuda().requires_grad_(True)
    with model.multi_step():
        y1 = model(xc, r)
        y2 = model(torch.cat([y1, xc[..., 12:]], -1), r)
    loss = torch.nn.functional.mse_loss(y1, t[0].cuda()) + torch.nn.functional.mse_loss(y2, t[1].cuda())
    loss.backward()
    out64, loss64, gx64, g64 = regional_oracle_step(sd, r, x, t, torch.float64, output_dim=12, num_blocks=2, rollout=2)
    assert abs(float(loss) - loss64) < 1e-5 * loss64
    fails = [(k, rel_max(q.grad, g64[k])) for k, q in model.named_parameters() if not rel_max(q.grad, g64[k]) < 1e-4]
    fails += [("features", rel_max(xc.grad, gx64))] if not rel_max(xc.grad, gx64) < 1e-4 else []
    assert not fails, fails


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_sgd_lowers_the_loss_and_inference_is_untouched(tp):
    """One SGD step lowers the loss; an inference forward after training equals, bit for bit, a fresh model's inference with the
    trained weights."""
    ll, sd, kw, x, gc, target = trunk_case(78, False)[:6]
    model = _build(sd, **kw, train_precision=tp)
    _, loss0, _, _ = _step(model, x, ll, target)
    opt = torch.optim.SGD(model.parameters(), lr=1e-2)
    opt.step()
    _, loss1, _, grads = _step(model, x, ll, target)
    assert loss1 < loss0, (loss0, loss1)
    assert all(torch.isfinite(g).all() for g in grads.values())
    model.eval()
    with torch.no_grad():
        after = model(x.cuda(), ll)
        fresh = _build(model.state_dict(), **kw).eval()
        assert torch.equal(after, fresh(x.cuda(), ll))
