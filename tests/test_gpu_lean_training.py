"""-m gpu: the bounded-memory training step (GraphWeatherForecaster(use_checkpointing=True): a training-only plan whose step keeps
only the mesh-sized activations and recomputes the encoder's lat/lon side and the decoder chunk by chunk in the backward).
Its forward against the taped step's (bit for bit where the per-row arithmetic does not depend on the chunk), its gradients
against the fp64 autograd oracle and against the taped step, repeatability, memory that does not grow with the grid, and one
step on the 0.25-degree grid."""
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


def _step(tp, ll, sd, x, target, var, lean, feat_grad=True, **kw):
    """One training step of a fresh forecaster: (model, out, loss, d features, {name: grad})."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    model = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=lean, **kw).cuda().train()
    model.load_state_dict(sd)
    res = train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target, feat_grad=feat_grad)
    assert model._train_engine.plan.train_only == lean
    return (model, *res)


# chunk sizes of the 10-degree grid: one point (every encoder chunk is one mesh slot, every decoder chunk one point), a
# non-divisor of the 648 points, and one chunk for everything
CHUNKS = ["1", "37", "100000"]


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_forward_equals_the_taped_step(case10, monkeypatch, tp, chunk):
    ll, sd, x, target, var = case10[:5]
    _, out_t, loss_t, gx_t, g_t = _step(tp, ll, sd, x, target, var, False)
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", chunk)
    _, out_l, loss_l, gx_l, g_l = _step(tp, ll, sd, x, target, var, True)
    assert torch.equal(out_l, out_t)
    assert loss_l == loss_t
    worst = max((rel_norm(g_l[k], g), k) for k, g in g_t.items() if float(g.norm()) > 0)
    print(f"{tp} chunk {chunk}: worst norm-relative gradient difference to the taped step {worst}; features {rel_norm(gx_l, gx_t):.2e}")
    assert worst[0] <= 1e-5 and rel_norm(gx_l, gx_t) <= 1e-5


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_gradients_match_the_oracle(case10, monkeypatch, tp):
    """10 degrees, batch 2, 18 decoder chunks: the bars test_gpu_training.py / test_gpu_train_precision.py hold the taped step to."""
    ll, sd, x, target, var, ref32, ref64 = case10
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    _, *ours = _step(tp, ll, sd, x, target, var, True)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=None)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=False, median=False,
                        ill=None, skip_zero=False, norm_bar=None)  # fmt: skip


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_weight_gradients_are_repeatable(case10, monkeypatch, tp):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = case10[:5]
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    model = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=True).cuda().train()
    model.load_state_dict(sd)
    crit = NormalizedMSELoss(var, ll, normalize=True)
    runs = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        crit(model(x.cuda()), target.cuda()).backward()
        runs.append({k: q.grad.clone() for k, q in model.named_parameters()})
    model._train_engine.plan.status()
    # Linear layers with K > 16 inputs (model.0 / .2 / .4 weights, except the edge encoders' 2-wide first layers): fixed-order sums
    linear = [k for k, q in model.named_parameters() if k.endswith("weight") and q.dim() == 2 and q.shape[1] > 16]
    assert len(linear) == 78
    for k in linear:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_wide_model(monkeypatch):
    """train/run_fulll.py's 597 + 24 features (6 blocks here 2), fp32_simt, 10 degrees, batch 2, many chunks vs the taped step."""
    from oracle import weights

    ll = grid(10)
    kw = dict(feature_dim=597, aux_dim=24, num_blocks=2)
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(3)
    sd = {k: v.detach().clone() for k, v in GraphWeatherForecaster(ll, **kw).state_dict().items()}
    x = weights.make_features(2, len(ll), 621, 3)
    target = torch.randn(2, len(ll), 597, generator=torch.Generator().manual_seed(3))
    var = [1.0] * 597
    _, out_t, loss_t, gx_t, g_t = _step("fp32_simt", ll, sd, x, target, var, False, **kw)
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    _, out_l, loss_l, gx_l, g_l = _step("fp32_simt", ll, sd, x, target, var, True, **kw)
    assert torch.equal(out_l, out_t) and loss_l == loss_t
    worst = max((rel_norm(g_l[k], g), k) for k, g in g_t.items() if float(g.norm()) > 0)
    assert worst[0] <= 1e-5 and rel_norm(gx_l, gx_t) <= 1e-5, worst


@pytest.mark.parametrize("ctype", ["additive", "softmax"])
def test_constrained_step(case10, monkeypatch, ctype):
    ll, sd, x, target, var = case10[:5]
    _, out_t, loss_t, gx_t, g_t = _step("fp32_simt", ll, sd, x, target, var, False, constraint_type=ctype)
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    _, out_l, loss_l, gx_l, g_l = _step("fp32_simt", ll, sd, x, target, var, True, constraint_type=ctype)
    assert torch.equal(out_l, out_t) and loss_l == loss_t
    # (under the additive constraint the last decoder bias has an analytically zero gradient, sum_r d_hr = 0: its computed value
    # is rounding noise in both steps, so numerically zero gradients are left out)
    big = max(float(g.norm()) for g in g_t.values())
    worst = max((rel_norm(g_l[k], g), k) for k, g in g_t.items() if float(g.norm()) > 1e-6 * big)
    assert worst[0] <= 1e-5 and rel_norm(gx_l, gx_t) <= 1e-5, worst


def _one_degree():
    from oracle import weights

    ll = grid(1)
    sd = weights.make_state_dict(weights.forecaster_shapes(), 5)
    x = weights.make_features(1, len(ll), 102, 5)
    rng = np.random.Generator(np.random.PCG64(5))
    target = torch.from_numpy(rng.standard_normal((1, len(ll), 78)).astype(np.float32))
    return ll, sd, x, target, [1.0] * 78


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_one_degree_against_the_taped_step(tp):
    """1 degree, batch 1, the automatic chunks: per parameter, norm-relative <= 1e-5 to the taped step."""
    ll, sd, x, target, var = _one_degree()
    m, out_t, loss_t, _, g_t = _step(tp, ll, sd, x, target, var, False, feat_grad=False)
    peak_t = m._train_engine.plan.train_peak_bytes()
    del m
    torch.cuda.empty_cache()
    m, out_l, loss_l, _, g_l = _step(tp, ll, sd, x, target, var, True, feat_grad=False)
    peak_l = m._train_engine.plan.train_peak_bytes()
    if tp == "fp32":  # (each chunk's operands are scaled from the chunk's own magnitudes)
        assert float((out_l - out_t).abs().max()) < 1e-4
    else:
        assert torch.equal(out_l, out_t)
    errs = sorted(((rel_norm(g_l[k], g), k) for k, g in g_t.items() if float(g.norm()) > 0), reverse=True)
    print(f"1 deg {tp}: loss {loss_l:.7f} vs {loss_t:.7f}; peak {peak_l / 2**30:.2f} GiB vs taped {peak_t / 2**30:.2f} GiB; "
          f"above 1e-5: {[(f'{e:.1e}', k) for e, k in errs if e > 1e-5]}")
    # Bars.  fp32_simt: only the summation order of dPd and of the weight gradients differs (measured <= 1.3e-6).  fp32: each chunk's
    # operands are scaled from the chunk's magnitudes, so activations differ in their last bits too (measured 1.5e-5).  bf16: the
    # forward is identical, but a last-bit difference of dPd flips the bf16 rounding of single operands of every data gradient
    # upstream; the tensors summed over the whole graph (ILL_CONDITIONED, tests/training_oracle.py) magnify it (measured 1.7e-3
    # for h3_nodes, 5.6e-4 for node_encoder.model.0.weight, at most 4.9e-5 for every other parameter).
    for e, k in errs:
        bar = {"fp32_simt": 1e-5, "fp32": 5e-5, "bf16": 5e-3 if k.startswith(ILL_CONDITIONED) else 2e-4}[tp]
        assert e <= bar, (k, e)
    assert peak_l < peak_t


def test_memory_does_not_grow_with_the_grid(monkeypatch):
    from graph_weather_b200 import GraphWeatherForecaster

    def peak(step, lean):
        ll = grid(step)
        model = GraphWeatherForecaster(ll, train_precision="bf16", use_checkpointing=lean).cuda().train()
        x = torch.randn(1, len(ll), 102, device="cuda")
        model(x).square().mean().backward()
        plan = model._train_engine.plan
        plan.status()
        d = model._train_engine.dims
        # graphs (int32 / fp32 arrays over points, mesh nodes and edges), the weights and small constants
        small = 4 * (4 * d["n_in"] + 5 * d["n_lat_edges"] + 4 * d["n_dec_edges"] + d["n_out"] + d["n_mesh"] * (3 + d["in_dim"])
                     + sum(q.numel() + 64 for q in model.parameters())) + (1 << 20)
        r = (plan.train_peak_bytes(), plan.device_bytes(), small)
        del model, plan
        torch.cuda.empty_cache()
        return r

    taped1, taped_plan1, _ = peak(1, False)
    taped2, _, _ = peak(2, False)
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "2048")
    lean1, lean_plan1, small1 = peak(1, True)
    lean2, _, _ = peak(2, True)
    print(f"peak: taped 1 deg {taped1 / 2**30:.2f} GiB, 2 deg {taped2 / 2**30:.2f} GiB; chunked 1 deg {lean1 / 2**30:.3f} GiB, "
          f"2 deg {lean2 / 2**30:.3f} GiB; plan bytes taped {taped_plan1 / 2**20:.0f} MiB, training-only {lean_plan1 / 2**20:.1f} MiB "
          f"(graphs + weights {small1 / 2**20:.1f} MiB)")
    assert lean1 - lean2 < 0.05 * taped1
    assert lean_plan1 <= small1
    assert lean_plan1 < 0.1 * taped_plan1


def test_quarter_degree_trains():
    """0.25 degrees (721 x 1440, the grid bench.py uses), batch 1, bf16, the default 102 -> 78 model."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    lat = np.linspace(-90.0, 90.0, 721)
    lon = np.arange(0.0, 360.0, 0.25)
    ll = [(float(a), float(b)) for a in lat for b in lon]
    torch.manual_seed(0)
    model = GraphWeatherForecaster(ll, train_precision="bf16", use_checkpointing=True).cuda().train()
    crit = NormalizedMSELoss([1.0] * 78, ll, normalize=True)
    opt = torch.optim.SGD(model.parameters(), lr=1e-2)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(1, len(ll), 102, device="cuda", generator=g)
    y = torch.randn(1, len(ll), 78, device="cuda", generator=g)
    losses = []
    for _ in range(3):
        opt.zero_grad(set_to_none=True)
        loss = crit(model(x), y)
        loss.backward()
        losses.append(float(loss))
        assert all(torch.isfinite(q.grad).all() for q in model.parameters())
        opt.step()
    plan = model._train_engine.plan
    plan.status()
    # bar: the chunk budget (4 GiB, gw_train.cu) with a quarter of slack, and the mesh-sized terms: per processor block about
    # 12 tensors of the latent edges (tape and backward temporaries) at batch 1, 8 more for the encoder / decoder mesh sides
    El, De, nb = 41162, 256, 9
    bar = 1.25 * 4 * 2**30 + (12 * nb + 8) * El * De * 4 + 2**30
    print(f"0.25 deg: losses {losses}; train_peak_bytes {plan.train_peak_bytes() / 2**30:.2f} GiB (bar {bar / 2**30:.2f}); "
          f"plan {plan.device_bytes() / 2**20:.0f} MiB")
    assert plan.train_peak_bytes() < bar
    assert losses[2] < losses[1] < losses[0]
