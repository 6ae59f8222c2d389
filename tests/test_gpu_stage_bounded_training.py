"""-m gpu: the standalone Encoder, Decoder, AssimilatorEncoder and AssimilatorDecoder on the bounded-memory training step
(`train_precision` and use_checkpointing=True: a training-only plan whose forward keeps only the mesh-sized tensors and whose
backward recomputes each lat/lon chunk right before differentiating it, as GraphWeatherForecaster(use_checkpointing=True) does):
  * the flag selects the step at every training forward, and the Processor stays on the taped step;
  * each stage's forward equals its taped step's bit for bit, its gradients within 1e-5 (fp32_simt, bf16; many chunks);
  * Encoder -> Processor -> Decoder and the assimilator's stages, all bounded, held to the fp64 oracle and to the wrapper's bounded
    step (output, loss and d features bit for bit);
  * bit-repeatable under torch.use_deterministic_algorithms(True), two calls of one stage in one graph, memory that does not grow
    with the grid, one step on the 0.25-degree grid, and the refusals of the taped step."""
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import assimilator_oracle_step, check_bf16_bars, check_fp32_bars, forecaster_case, grid, rel_norm, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]

TPS = ["fp32_simt", "fp32", "bf16"]
PREFIXES = ("encoder", "processor", "decoder")


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture(scope="module")
def case10():
    """The seeded 10-degree, batch-2 step of tests/test_gpu_training.py and its oracle results (fp32 and fp64)."""
    return forecaster_case(10, 2, 21)


@pytest.fixture
def deterministic():
    """torch.use_deterministic_algorithms(True) for the test, restored afterwards."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _sub(sd, prefix):
    return {k[len(prefix) + 1 :]: v for k, v in sd.items() if k.startswith(prefix + ".")}


def _stages(ll, sd, tp, cp):
    from graph_weather_b200 import Decoder, Encoder, Processor

    mods = (Encoder(ll, input_dim=102, train_precision=tp, use_checkpointing=cp), Processor(train_precision=tp),
            Decoder(ll, train_precision=tp, use_checkpointing=cp))  # fmt: skip
    for m, p in zip(mods, PREFIXES):
        m.load_state_dict(_sub(sd, p))
    return [m.cuda().train() for m in mods]


def _grads(mods, prefixes=PREFIXES):
    return {f"{p}.{k}": q.grad.detach().cpu().clone() for m, p in zip(mods, prefixes) for k, q in m.named_parameters()}


def _composed_step(mods, x, target, crit):
    """test_end2end's composition + loss.backward(): (out, loss, d features, {name: grad}) on the host."""
    enc, proc, dec = mods
    for m in mods:
        m.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    h, ei, ea = enc(xc)
    out = dec(proc(h, ei, ea, batch_size=x.shape[0]), xc[..., :78])
    loss = crit(out, target.cuda())
    loss.backward()
    for m in mods:
        m._train_engine.plan.status()
    return out.detach().cpu(), float(loss), xc.grad.cpu(), _grads(mods)


def _randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).cuda()


# ---------------------------------------------------------------------------------------------------------------------------
# which step
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp", TPS)
def test_use_checkpointing_selects_the_step(tp):
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, Decoder, Encoder, Processor

    ll = grid(30)
    enc = Encoder(ll, input_dim=6, train_precision=tp, use_checkpointing=True).cuda().train()
    aenc = AssimilatorEncoder(train_precision=tp, use_checkpointing=True).cuda().train()
    proc = Processor(num_blocks=2, train_precision=tp, use_checkpointing=True).cuda().train()
    dec = Decoder(ll, output_dim=4, train_precision=tp, use_checkpointing=True).cuda().train()
    adec = AssimilatorDecoder(ll, output_dim=4, train_precision=tp, use_checkpointing=True).cuda().train()
    x = torch.randn(1, len(ll), 6, device="cuda")
    obs = torch.rand(40, 3, device="cuda") * torch.tensor([180.0, 360.0, 1.0], device="cuda") - torch.tensor([90.0, 0.0, 0.0], device="cuda")

    def step():
        h, ei, ea = enc(x)
        ha, _, eaa = aenc(torch.randn(1, 40, 2, device="cuda"), obs)
        y = proc(h, ei, ea)
        (dec(y, x[..., :4]).sum() + adec(proc(ha, ei, eaa), 1).sum()).backward()
        for m in (enc, aenc, proc, dec, adec):
            m._train_engine.plan.status()
            assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in m.parameters()), type(m).__name__

    for flag in (True, False, True):
        for m in (enc, aenc, proc, dec, adec):
            m.use_checkpointing = flag
            m.zero_grad(set_to_none=True)
        step()
        for m in (enc, aenc, dec, adec):
            assert m._train_engine.plan.train_only is flag, type(m).__name__
            other = m._train_engines.get(not flag)
            assert other is None or other.plan is None  # switching closed the other step's plan
        assert proc._train_engine.plan.train_only is False  # the processor stays on the taped step
    # a forward made under one step cannot run its backward after a switch: its plan is gone
    y = dec(torch.randn(dec.num_h3, 256, device="cuda", requires_grad=True), x[..., :4])
    dec.use_checkpointing = False
    dec(torch.randn(dec.num_h3, 256, device="cuda"), x[..., :4])
    with pytest.raises(RuntimeError, match="one backward per forward"):
        y.sum().backward()


# ---------------------------------------------------------------------------------------------------------------------------
# each stage against its taped step
# ---------------------------------------------------------------------------------------------------------------------------
def _encoder_run(enc, x, cot):
    enc.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    h, _, ea = enc(xc)
    ((h * cot[0]).sum() + (ea * cot[1]).sum()).backward()
    enc._train_engine.plan.status()
    return (h.detach(), ea.detach()), {"features": xc.grad, **_grads([enc], ["encoder"])}


def _decoder_run(dec, h, start, cot):
    dec.zero_grad(set_to_none=True)
    hc, sc = h.clone().requires_grad_(True), start.clone().requires_grad_(True)
    y = dec(hc, sc)
    (y * cot).sum().backward()
    dec._train_engine.plan.status()
    return (y.detach(),), {"x": hc.grad, "start": sc.grad, **_grads([dec], ["decoder"])}


CHUNKS = ["1", "37", "100000"]  # one point per chunk, a non-divisor of the 648 points, one chunk for everything


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_each_stage_equals_its_taped_step(case10, monkeypatch, tp, chunk):
    ll, sd, x = case10[:3]
    B = x.shape[0]
    runs = {}
    for cp in (False, True):
        if cp:
            monkeypatch.setenv("GW_B200_TRAIN_CHUNK", chunk)
        enc, _, dec = _stages(ll, sd, tp, cp)
        h = torch.randn(B * dec.num_h3, 256, generator=torch.Generator().manual_seed(4)).cuda()
        start = x[..., :78].cuda()
        ecot = (_randn((B * enc.num_h3, 256), 5), _randn((B * enc._g_lat.edge_index.shape[1], 256), 6))
        runs[cp] = (_encoder_run(enc, x, ecot), _decoder_run(dec, h, start, _randn((B, len(ll), 78), 7)))
        assert enc._train_engine.plan.train_only is cp and dec._train_engine.plan.train_only is cp
    for i, stage in enumerate(("encoder", "decoder")):
        (out_t, g_t), (out_l, g_l) = runs[False][i], runs[True][i]
        assert all(torch.equal(a, b) for a, b in zip(out_l, out_t)), stage
        worst = max((rel_norm(g_l[k], g), k) for k, g in g_t.items() if float(g.norm()) > 0)
        print(f"{stage} {tp} chunk {chunk}: worst norm-relative gradient difference to the taped step {worst}")
        assert worst[0] <= 1e-5, (stage, worst)


# ---------------------------------------------------------------------------------------------------------------------------
# compositions against the oracle and the wrappers' bounded step
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp", TPS)
def test_bounded_composition_matches_the_oracle_and_the_wrapper(case10, monkeypatch, tp):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var, ref32, ref64 = case10
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    crit = NormalizedMSELoss(var, ll, normalize=True)
    mods = _stages(ll, sd, tp, True)
    ours = _composed_step(mods, x, target, crit)
    assert [m._train_engine.plan.train_only for m in mods] == [True, False, True]
    tag = f"bounded composition {tp}"
    # (the bars of tests/test_gpu_stage_training.py's taped composition)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999, tag=tag)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=False, median=tp == "fp32_simt",
                        ill=None, skip_zero=False, norm_bar=None, tag=tag)  # fmt: skip
    wrapper = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=True).cuda().train()
    wrapper.load_state_dict(sd)
    theirs = train_step(wrapper, crit, x, target)
    assert wrapper._train_engine.plan.train_only
    worst = sorted(((rel_norm(ours[3][k], g), k) for k, g in theirs[3].items()), reverse=True)
    print(f"{tag} vs the wrapper's bounded step: worst parameters {worst[:3]}")
    assert torch.equal(ours[0], theirs[0]) and ours[1] == theirs[1] and torch.equal(ours[2], theirs[2])
    assert worst[0][0] < 1e-6, worst[0]


@pytest.fixture(scope="module")
def assim300():
    """The 300-observation assimilator case of tests/test_gpu_stage_training.py and its oracle steps."""
    from oracle import restate, weights

    out_ll = [(float(lat), float(lon)) for lat in range(-90, 90, 5) for lon in range(0, 360, 5)]
    sd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=24), 41)
    g_static = restate.build_assimilator_graphs(out_ll)
    n, seed = 300, 51
    rng = np.random.Generator(np.random.PCG64(seed))
    obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, n), rng.uniform(0, 360, n), rng.uniform(0, 1, n)], 1).astype(np.float32))
    x = weights.make_features(1, n, 2, seed)
    target = torch.randn(1, len(out_ll), 24, generator=torch.Generator().manual_seed(seed))
    refs = [assimilator_oracle_step(sd, g_static, x, obs, target, dt) for dt in (torch.float32, torch.float64)]
    return out_ll, sd, x, obs, target, *refs


@pytest.mark.parametrize("tp", TPS)
def test_bounded_assimilator_composition_matches_the_oracle_and_the_wrapper(assim300, monkeypatch, tp):
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, GraphWeatherAssimilator, Processor

    out_ll, sd, x, obs, target, ref32, ref64 = assim300
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    mods = (AssimilatorEncoder(train_precision=tp, use_checkpointing=True), Processor(train_precision=tp),
            AssimilatorDecoder(out_ll, output_dim=24, train_precision=tp, use_checkpointing=True))  # fmt: skip
    for m, p in zip(mods, PREFIXES):
        m.load_state_dict(_sub(sd, p))
    enc, proc, dec = [m.cuda().train() for m in mods]
    xc = x.cuda().requires_grad_(True)
    h, ei, ea = enc(xc, obs.cuda())
    out = dec(proc(h, ei, ea), 1)
    loss = torch.nn.functional.mse_loss(out, target.cuda())
    loss.backward()
    assert enc._train_engine.plan.train_only and dec._train_engine.plan.train_only
    ours = (out.detach().cpu(), float(loss), xc.grad.cpu(), _grads((enc, proc, dec)))
    # (the bars of tests/test_gpu_assimilator_training.py, as for the taped composition)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=214, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=0.98, total_cos=None, tag=tp)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=214, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=True, median=False, ill=None,
                        skip_zero=False, norm_bar=None, tag=tp)  # fmt: skip
    wrapper = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=24, train_precision=tp, use_checkpointing=True).cuda().train()
    wrapper.load_state_dict(sd)
    theirs = train_step(wrapper, torch.nn.functional.mse_loss, x, target, obs=obs)
    worst = max((rel_norm(ours[3][k], g), k) for k, g in theirs[3].items())
    print(f"assimilator {tp} bounded composition vs the wrapper's bounded step: worst parameter {worst}")
    assert torch.equal(ours[0], theirs[0]) and ours[1] == theirs[1] and torch.equal(ours[2], theirs[2])
    assert worst[0] < 1e-6, worst


# ---------------------------------------------------------------------------------------------------------------------------
# repeatability, two calls in one graph, memory
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp", TPS)
def test_bounded_stages_repeat(case10, monkeypatch, deterministic, tp):
    ll, sd, x, target, var = case10[:5]
    from graph_weather_b200 import NormalizedMSELoss

    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    mods = _stages(ll, sd, tp, True)
    crit = NormalizedMSELoss(var, ll, normalize=True)
    a, b = _composed_step(mods, x, target, crit), _composed_step(mods, x, target, crit)
    assert torch.equal(a[0], b[0]) and a[1] == b[1] and torch.equal(a[2], b[2])
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), k


@pytest.mark.parametrize("tp", TPS)
def test_two_calls_in_one_graph(monkeypatch, tp):
    """A bounded Decoder and a bounded Encoder each applied twice in one graph, at batch 2 and then 1 (the backward of each call
    cuts its own batch's chunk tables), against the same calls on the taped step."""
    from graph_weather_b200 import Decoder, Encoder

    ll = grid(10)
    torch.manual_seed(8)
    dec0, enc0 = Decoder(ll, output_dim=8), Encoder(ll, input_dim=8)
    hs = [torch.randn(b * dec0.num_h3, 256).cuda() for b in (2, 1)]
    starts = [torch.randn(b, len(ll), 8).cuda() for b in (2, 1)]
    xs = [torch.randn(b, len(ll), 8).cuda() for b in (2, 1)]
    runs = {}
    for cp in (False, True):
        if cp:
            monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
        dec = Decoder(ll, output_dim=8, train_precision=tp, use_checkpointing=cp)
        enc = Encoder(ll, input_dim=8, train_precision=tp, use_checkpointing=cp)
        dec.load_state_dict(dec0.state_dict())
        enc.load_state_dict(enc0.state_dict())
        dec, enc = dec.cuda().train(), enc.cuda().train()
        hc = [h.clone().requires_grad_(True) for h in hs]
        xc = [v.clone().requires_grad_(True) for v in xs]
        loss = sum((dec(h, s) * (i + 1)).square().mean() for i, (h, s) in enumerate(zip(hc, starts)))
        for i, v in enumerate(xc):
            h, _, ea = enc(v)
            loss = loss + (h * (i + 1)).square().mean() + ea.square().mean()
        assert len(dec._train_engine.plan.live_tapes()) == 2 and len(enc._train_engine.plan.live_tapes()) == 2
        loss.backward()
        assert sum(t.bytes() for t in dec._train_engine.plan.live_tapes()) == 0
        assert dec._train_engine.plan.train_only is cp and enc._train_engine.plan.train_only is cp
        for m in (dec, enc):
            m._train_engine.plan.status()
        runs[cp] = {"h0": hc[0].grad, "h1": hc[1].grad, "x0": xc[0].grad, "x1": xc[1].grad, **_grads([enc, dec], ["encoder", "decoder"])}
    worst = max((rel_norm(runs[True][k], g), k) for k, g in runs[False].items() if float(g.norm()) > 0)
    print(f"{tp}: two calls per stage, bounded vs taped: worst {worst}")
    # (fp32_simt: only the order of float sums differs; fp32 scales each chunk's operands from the chunk, and in bf16 a last-bit
    # difference of the chunk-ordered dPd can flip the rounding of single data-gradient operands)
    assert worst[0] <= (1e-5 if tp == "fp32_simt" else 1e-4), worst


def test_memory_does_not_grow_with_the_grid(monkeypatch):
    """Each bounded stage's train_peak_bytes at 2 and 1 degrees (GW_B200_TRAIN_CHUNK=2048, bf16, batch 1): equal up to the
    mesh- and output-sized terms, and well below the taped stage's at 1 degree."""
    from graph_weather_b200 import Decoder, Encoder

    def peaks(step, cp):
        ll = grid(step)
        enc = Encoder(ll, input_dim=102, train_precision="bf16", use_checkpointing=cp).cuda().train()
        dec = Decoder(ll, train_precision="bf16", use_checkpointing=cp).cuda().train()
        x = torch.randn(1, len(ll), 102, device="cuda", requires_grad=True)
        h, _, ea = enc(x)
        (h.square().mean() + ea.square().mean()).backward()
        y = dec(torch.randn(dec.num_h3, 256, device="cuda", requires_grad=True), x.detach()[..., :78])
        y.square().mean().backward()
        r = {}
        for name, m in (("encoder", enc), ("decoder", dec)):
            m._train_engine.plan.status()
            r[name] = (m._train_engine.plan.train_peak_bytes(), m._train_engine.plan.device_bytes())
        del enc, dec, x, h, ea, y
        torch.cuda.empty_cache()
        return r

    taped1 = peaks(1, False)
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "2048")
    lean1, lean2 = peaks(1, True), peaks(2, True)
    for s in ("encoder", "decoder"):
        print(f"{s} peak: taped 1 deg {taped1[s][0] / 2**20:.1f} MiB; bounded 1 deg {lean1[s][0] / 2**20:.1f} MiB, 2 deg "
              f"{lean2[s][0] / 2**20:.1f} MiB; plan bytes taped {taped1[s][1] / 2**20:.1f} MiB, training-only {lean1[s][1] / 2**20:.1f} MiB")
        # the mesh and its latent / mesh-side tensors are the same at both grids; the grid's points enter through one chunk only
        assert abs(lean1[s][0] - lean2[s][0]) < 0.05 * taped1[s][0], s
        assert lean1[s][0] < 0.5 * taped1[s][0], s


def test_quarter_degree_composition_equals_the_wrapper():
    """0.25 degrees (721 x 1440), batch 1, bf16: Encoder -> Processor -> Decoder on the bounded step, against the wrapper's bounded
    step (held to the fp64 grid oracle in tests/test_gpu_full_grid.py): output, loss and d features bit for bit."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    lat = np.linspace(-90.0, 90.0, 721)
    lon = np.arange(0.0, 360.0, 0.25)
    ll = [(float(a), float(b)) for a in lat for b in lon]
    torch.manual_seed(0)
    wrapper = GraphWeatherForecaster(ll, train_precision="bf16", use_checkpointing=True).cuda().train()
    sd = wrapper.state_dict()
    crit = NormalizedMSELoss([1.0] * 78, ll, normalize=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(1, len(ll), 102, device="cuda", generator=g)
    y = torch.randn(1, len(ll), 78, device="cuda", generator=g)

    xw = x.clone().requires_grad_(True)
    out_w = wrapper(xw)
    loss_w = crit(out_w, y)
    loss_w.backward()
    wrapper._train_engine.plan.status()
    peak_w = wrapper._train_engine.plan.train_peak_bytes()

    mods = _stages(ll, sd, "bf16", True)
    enc, proc, dec = mods
    xs = x.clone().requires_grad_(True)
    h, ei, ea = enc(xs)
    out_s = dec(proc(h, ei, ea), xs[..., :78])
    loss_s = crit(out_s, y)
    loss_s.backward()
    for m in mods:
        m._train_engine.plan.status()
    peaks = {p: m._train_engine.plan.train_peak_bytes() for p, m in zip(PREFIXES, mods)}
    print(f"0.25 deg bf16: loss composed {loss_s.item():.7f} wrapper {loss_w.item():.7f}; train_peak_bytes wrapper "
          f"{peak_w / 2**30:.2f} GiB, stages {({k: round(v / 2**30, 2) for k, v in peaks.items()})} GiB")
    assert all(m._train_engine.plan.train_only for m in (enc, dec))
    assert torch.equal(out_s.detach(), out_w.detach())
    assert loss_s.item() == loss_w.item()
    assert torch.equal(xs.grad, xw.grad)


# ---------------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_bounded_stages_refuse_non_finite_inputs(monkeypatch, tp):
    from graph_weather_b200 import Decoder, Encoder

    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    ll = grid(30)
    dec = Decoder(ll, output_dim=4, train_precision=tp, use_checkpointing=True).cuda().train()
    h = torch.randn(1, dec.num_h3, 256)
    h[0, 11, 5] = float("inf")
    with pytest.raises(RuntimeError, match="not finite"):
        dec(h.reshape(-1, 256).cuda().requires_grad_(True), torch.zeros(1, len(ll), 4, device="cuda"))
    assert dec._train_engine.plan.train_only
    enc = Encoder(ll, input_dim=6, train_precision=tp, use_checkpointing=True).cuda().train()
    x = torch.randn(1, len(ll), 6)
    x[0, 17, 2] = float("nan")
    with pytest.raises(RuntimeError, match="not finite"):
        enc(x.cuda().requires_grad_(True))
    assert enc._train_engine.plan.train_only


@pytest.mark.parametrize("tp", TPS)
def test_bounded_backward_refusals(monkeypatch, tp):
    """A backward after the weights were re-uploaded, or (AssimilatorEncoder) after the encoder graph changed, raises."""
    from graph_weather_b200 import AssimilatorEncoder, Decoder

    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    ll = grid(30)
    dec = Decoder(ll, output_dim=4, train_precision=tp, use_checkpointing=True).cuda().train()
    start = torch.zeros(1, len(ll), 4, device="cuda")
    y = dec(torch.randn(dec.num_h3, 256, device="cuda", requires_grad=True), start)
    with torch.no_grad():
        dec.node_decoder.model[0].weight.add_(0.01)
    dec(torch.randn(dec.num_h3, 256, device="cuda"), start)  # (re-uploads the weights)
    with pytest.raises(RuntimeError, match="weights were replaced"):
        y.sum().backward()
    enc = AssimilatorEncoder(train_precision=tp, use_checkpointing=True).cuda().train()
    gen = torch.Generator().manual_seed(3)

    def obs():
        return (torch.rand(40, 3, generator=gen) * torch.tensor([180.0, 360.0, 1.0]) - torch.tensor([90.0, 0.0, 0.0])).cuda()

    h1, _, _ = enc(torch.randn(1, 40, 2, device="cuda", requires_grad=True), obs())
    h2, _, _ = enc(torch.randn(1, 40, 2, device="cuda", requires_grad=True), obs())
    assert enc._train_engine.plan.train_only
    with pytest.raises(RuntimeError, match="encoder graph was replaced"):
        h1.sum().backward()
    h2.sum().backward()  # the later forward's backward runs
    enc._train_engine.plan.status()
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in enc.parameters())
