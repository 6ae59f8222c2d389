"""-m gpu: the standalone Encoder, Processor, Decoder, AssimilatorEncoder and AssimilatorDecoder trained on the CUDA step
(`train_precision`, gw_train_{encoder,processor,decoder}_*_tape), every train precision:
  * Encoder -> Processor -> Decoder composed as the reference's tests/test_model.py::test_end2end, one NormalizedMSE step held to
    the fp64 oracle with the bars of tests/test_gpu_training.py / tests/test_gpu_train_precision.py, and to the wrapper's step;
  * each stage alone against torch autograd of oracle/restate.py's stage function in float64 (on the GPU);
  * the processor on a random caller graph (the reference's test_processor_checkpointing shape): edge_attr.grad in the caller's
    order, and segments 0 / 1 / -1 giving the same outputs and gradients;
  * AssimilatorEncoder -> Processor -> AssimilatorDecoder against the assimilator oracle;
  * non-finite inputs refused in the tensor-core precisions, and the tapes' lifetime."""
import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import (ILL_CONDITIONED, assimilator_oracle_step, check_bf16_bars, check_fp32_bars, cos, forecaster_case, grid,
                             rel_norm)

pytestmark = [pytest.mark.gpu, pytest.mark.training]

TPS = ["fp32_simt", "fp32", "bf16"]
PREFIXES = ("encoder", "processor", "decoder")


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture(scope="module")
def case10():
    return forecaster_case(10, 2, 21)


def _sub(sd, prefix):
    return {k[len(prefix) + 1 :]: v for k, v in sd.items() if k.startswith(prefix + ".")}


def _stages(ll, sd, tp, eb=False):
    from graph_weather_b200 import Decoder, Encoder, Processor

    mods = (Encoder(ll, input_dim=102, efficient_batching=eb, train_precision=tp), Processor(train_precision=tp),
            Decoder(ll, train_precision=tp))  # fmt: skip
    for m, p in zip(mods, PREFIXES):
        m.load_state_dict(_sub(sd, p))
    return [m.cuda().train() for m in mods]


def _grads(mods, prefixes=PREFIXES):
    return {f"{p}.{k}": q.grad.detach().cpu().clone() for m, p in zip(mods, prefixes) for k, q in m.named_parameters()}


def _composed_step(mods, x, target, crit, eb):
    """test_end2end's composition + loss.backward(): (out, loss, d features, {name: grad}) on the host."""
    enc, proc, dec = mods
    for m in mods:
        m.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    h, ei, ea = enc(xc)
    h = proc(h, ei, ea, batch_size=x.shape[0], efficient_batching=eb)
    out = dec(h, xc[..., :78])
    loss = crit(out, target.cuda())
    loss.backward()
    for m in mods:
        m._train_engine.plan.status()
    return out.detach().cpu(), float(loss), xc.grad.cpu(), _grads(mods)


@pytest.mark.parametrize("eb", [False, True])
@pytest.mark.parametrize("tp", TPS)
def test_composed_stages_match_the_oracle_and_the_wrapper(case10, tp, eb):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss
    from training_oracle import train_step

    ll, sd, x, target, var, ref32, ref64 = case10
    crit = NormalizedMSELoss(var, ll, normalize=True)
    ours = _composed_step(_stages(ll, sd, tp, eb), x, target, crit, eb)
    tag = f"composed {tp} efficient_batching={eb}"
    # (bars of tests/test_gpu_training.py for fp32_simt and tests/test_gpu_train_precision.py for fp32 / bf16.  Measured on an H100,
    # both batchings alike: fp32_simt features 1.9e-6 (bar 1.4e-4), worst parameter 2.3e-4 max-relative on processor block 8's
    # edge model.2.weight (bar 2.6e-4); fp32 encoder.h3_nodes 5.3e-2 (bar 1.0e-1), worst processor parameter 1.1e-3 (floor 2e-3);
    # bf16 cosine 0.9858 for h3_nodes and 0.9895 for node_encoder.model.0.weight (bar 0.98), >= 0.998 for every other parameter)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999, tag=tag)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=False, median=tp == "fp32_simt",
                        ill=None, skip_zero=False, norm_bar=None, tag=tag)  # fmt: skip
    wrapper = GraphWeatherForecaster(ll, train_precision=tp).cuda().train()
    wrapper.load_state_dict(sd)
    theirs = train_step(wrapper, crit, x, target)
    # the same arithmetic: the output, the loss and the features' gradient bit for bit; the parameters' gradients up to the order
    # of float sums (atomics, and the per-sample copies of the latent edge features summed by autograd instead of in the step)
    # (measured on an H100: at most 6.7e-7 norm-relative, every precision and both batchings)
    worst = sorted(((rel_norm(ours[3][k], g), k) for k, g in theirs[3].items()), reverse=True)
    print(f"{tag} vs the wrapper: worst parameters {worst[:3]}")
    assert torch.equal(ours[0], theirs[0]) and ours[1] == theirs[1] and torch.equal(ours[2], theirs[2])
    assert worst[0][0] < 1e-5, worst[0]


def _graphs(ll, dt):
    from oracle import restate

    return {k: (v.to("cuda", dt) if torch.is_tensor(v) and v.is_floating_point() else (v.cuda() if torch.is_tensor(v) else v))
            for k, v in restate.build_forecaster_graphs(ll).items()}  # fmt: skip


def _autograd(sd, prefix, dt, inputs, fn, cotangents):
    """torch autograd of the restated stage fn(params, *inputs) -> outputs in dtype dt on the GPU, against `cotangents`:
    {input name or parameter name: gradient}."""
    s = {k: v.to("cuda", dt).requires_grad_(True) for k, v in sd.items() if k.startswith(prefix + ".")}
    ins = {k: v.detach().to("cuda", dt).requires_grad_(True) for k, v in inputs.items()}
    outs = fn(s, *ins.values())
    sum((o * c.to(dt)).sum() for o, c in zip(outs, cotangents)).backward()
    return {**{k: v.grad for k, v in ins.items()}, **{k: v.grad for k, v in s.items()}}


def _check_alone(tag, tp, got, want32, want64, floor):
    """{name: gradient} against fp64, norm-relative, as check_fp32_bars holds max-relative errors: below 10x the fp32 oracle's own
    error + 2e-5, or below `floor`, 5x that for the ILL_CONDITIONED parameters; bf16: cosine at least 0.99 (0.98 for those)."""
    fails, rows = [], []
    for k, w in want64.items():
        if float(w.abs().max()) == 0.0:
            continue
        ill = k.startswith(ILL_CONDITIONED)
        e, e32 = rel_norm(got[k], w), rel_norm(want32[k], w)
        if tp == "bf16":
            c = cos(got[k], w)
            rows.append((1 - c, k, e32))
            if not c >= (0.98 if ill else 0.99):
                fails.append((k, c))
        else:
            rows.append((e, k, e32))
            if not e < max(10 * e32 + 2e-5, floor) * (5 if ill else 1):
                fails.append((k, e, e32))
    print(tag, tp, "worst (error or 1 - cosine, name, fp32 oracle's error):", sorted(rows, reverse=True)[:3])
    assert not fails, fails


@pytest.mark.parametrize("tp", TPS)
def test_each_stage_alone_against_fp64(case10, tp):
    from oracle import restate

    ll, sd, x = case10[:3]
    enc, proc, dec = _stages(ll, sd, tp)
    gd = {dt: _graphs(ll, dt) for dt in (torch.float32, torch.float64)}
    gen = torch.Generator(device="cuda").manual_seed(5)
    B = x.shape[0]
    # encoder: random cotangents on x and edge_attr
    xc = x.cuda().requires_grad_(True)
    h, ei, ea = enc(xc)
    cot = (torch.randn(h.shape, generator=gen, device="cuda"), torch.randn(ea.shape, generator=gen, device="cuda"))
    ((h * cot[0]).sum() + (ea * cot[1]).sum()).backward()
    want = {dt: _autograd(sd, "encoder", dt, {"features": x}, lambda s, f: restate.encoder_forward(s, gd[dt], f)[0::2], cot)
            for dt in gd}  # fmt: skip
    # (fp32 mode: a 5e-3 floor, as a ReLU unit that switches between two fp32 implementations moves a gradient; measured worst 2.4e-3)
    floor = 5e-3 if tp == "fp32" else 0.0
    _check_alone("encoder", tp, {"features": xc.grad, **_grads([enc], ["encoder"])}, want[torch.float32], want[torch.float64], floor)
    # processor on the latent graph, per-sample edge features (the encoder's outputs)
    with torch.no_grad():
        h64, ei64, ea64 = restate.encoder_forward({k: v.to("cuda", torch.float64) for k, v in sd.items()}, gd[torch.float64], x.cuda().double())
    hp, ep = h64.float().requires_grad_(True), ea64.float().requires_grad_(True)
    out = proc(hp, ei64, ep)
    cot = (torch.randn(out.shape, generator=gen, device="cuda"),)
    (out * cot[0]).sum().backward()
    want = {dt: _autograd(sd, "processor", dt, {"x": hp, "edge_attr": ep}, lambda s, a, e: (restate.processor_forward(s, a, ei64, e),), cot)
            for dt in gd}  # fmt: skip
    # (random cotangents through nine blocks cancel heavily: the fp32 oracle's own error, which its scatter_add atomics make vary from
    # run to run, measured between 1e-6 and 1.7e-3 on the same parameter; ours is repeatable at 1.6e-3 in fp32_simt, 2.4e-3 in fp32:
    # a 5e-3 floor in both)
    _check_alone("processor", tp, {"x": hp.grad, "edge_attr": ep.grad, **_grads([proc], ["processor"])}, want[torch.float32],
                 want[torch.float64], 5e-3)  # fmt: skip
    # decoder, residual included
    hd = out.detach().requires_grad_(True)
    start = x[..., :78].cuda().requires_grad_(True)
    y = dec(hd, start)
    cot = (torch.randn(y.shape, generator=gen, device="cuda"),)
    (y * cot[0]).sum().backward()
    want = {dt: _autograd(sd, "decoder", dt, {"x": hd, "start": start},
                          lambda s, a, st: (restate.assimilator_decoder_forward(s, gd[dt], a, B) + st,), cot) for dt in gd}  # fmt: skip
    _check_alone("decoder", tp, {"x": hd.grad, "start": start.grad, **_grads([dec], ["decoder"])}, want[torch.float32],
                 want[torch.float64], floor)  # fmt: skip
    # (measured on an H100, worst of the three stages: fp32_simt 1.6e-3 on processor block 5's node model.0, the encoder and decoder
    # below 1e-6; fp32 2.4e-3 on processor block 4, 2.0e-3 on the decoder's x; bf16 cosine >= 0.992)


def _random_graph_case():
    torch.manual_seed(42)
    B, n, E = 2, 5882, 41162
    return B, torch.randn((B * n, 256)), torch.randint(0, n, (2, E)), torch.randn((E, 256))


@pytest.mark.parametrize("tp", TPS)
def test_processor_on_a_random_graph(tp):
    from graph_weather_b200 import Processor

    B, x, ei, ea = _random_graph_case()
    proc = Processor(train_precision=tp).cuda().train()
    runs = {}
    for seg in (0, 1, -1):
        proc.set_checkpoint_segments(seg)
        proc.zero_grad(set_to_none=True)
        xc, ec = x.cuda().requires_grad_(True), ea.cuda().requires_grad_(True)
        out = proc(xc, ei.cuda(), ec, batch_size=B, efficient_batching=True)
        go = torch.randn(out.shape, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
        (out * go).sum().backward()
        proc._train_engine.plan.status()
        assert ec.grad.shape == ea.shape and xc.grad.shape == x.shape
        runs[seg] = (out.detach(), xc.grad, ec.grad, {k: q.grad.clone() for k, q in proc.named_parameters()})
    # edge_attr.grad comes back in the caller's order: the same edges listed in another order (target-sorted, so that every
    # per-target sum adds the same rows in the same order) get the same gradients, permuted
    perm = torch.sort(ei[1], stable=True)[1]
    assert not torch.equal(perm, torch.arange(perm.numel()))
    proc.set_checkpoint_segments(0)
    proc.zero_grad(set_to_none=True)
    xc, ec = x.cuda().requires_grad_(True), ea[perm].cuda().requires_grad_(True)
    out = proc(xc, ei[:, perm].cuda(), ec, batch_size=B, efficient_batching=True)
    (out * go).sum().backward()
    assert torch.equal(out.detach(), runs[0][0]) and torch.equal(xc.grad, runs[0][1])
    assert torch.equal(ec.grad, runs[0][2][perm.cuda()])
    for seg in (1, -1):
        a, b = runs[0], runs[seg]
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), seg
        for k in a[3]:
            # (fp32_simt weight gradients and every LayerNorm's are summed with float atomics)
            if tp != "fp32_simt" and ".model.5." not in k:
                assert torch.equal(a[3][k], b[3][k]), (seg, k)
            else:
                assert rel_norm(b[3][k], a[3][k]) < 1e-5, (seg, k)


@pytest.fixture(scope="module")
def assim300():
    """The 300-observation case of tests/test_gpu_assimilator_training.py (its `_case(setup, 300, 51)`) and its oracle steps."""
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
def test_composed_assimilator_matches_the_oracle_and_the_wrapper(assim300, tp):
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, GraphWeatherAssimilator, Processor
    from training_oracle import train_step

    out_ll, sd, x, obs, target, ref32, ref64 = assim300
    mods = (AssimilatorEncoder(train_precision=tp), Processor(train_precision=tp), AssimilatorDecoder(out_ll, output_dim=24, train_precision=tp))
    for m, p in zip(mods, PREFIXES):
        m.load_state_dict(_sub(sd, p))
    enc, proc, dec = [m.cuda().train() for m in mods]
    xc = x.cuda().requires_grad_(True)
    h, ei, ea = enc(xc, obs.cuda())
    out = dec(proc(h, ei, ea), 1)
    loss = torch.nn.functional.mse_loss(out, target.cuda())
    loss.backward()
    ours = (out.detach().cpu(), float(loss), xc.grad.cpu(), _grads((enc, proc, dec)))
    # (the bars of tests/test_gpu_assimilator_training.py; 214 parameters: h3_nodes is a plain tensor.  Measured on an H100: the
    # features' gradient 6.6e-4 in fp32_simt and 3.5e-3 in fp32 (bar 6.6e-3), cosine 0.9809 in bf16 (bar 0.98) -- the wrapper's own)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=214, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=0.98, total_cos=None, tag=tp)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=214, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=True, median=False, ill=None,
                        skip_zero=False, norm_bar=None, tag=tp)  # fmt: skip
    wrapper = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=24, train_precision=tp).cuda().train()
    wrapper.load_state_dict(sd)
    theirs = train_step(wrapper, torch.nn.functional.mse_loss, x, target, obs=obs)
    # the same arithmetic: output, loss and the observation values' gradient bit for bit, the parameters' gradients up to the order
    # of float sums (measured on an H100: at most 6.3e-7 norm-relative)
    worst = max((rel_norm(ours[3][k], g), k) for k, g in theirs[3].items())
    print(f"assimilator {tp} composed vs the wrapper: worst parameter {worst}")
    assert torch.equal(ours[0], theirs[0]) and ours[1] == theirs[1] and torch.equal(ours[2], theirs[2])
    assert worst[0] < 1e-5, worst


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_cores_refuse_non_finite_stage_inputs(tp):
    from graph_weather_b200 import Decoder, Processor

    B, x, ei, ea = _random_graph_case()
    proc = Processor(num_blocks=2, train_precision=tp).cuda().train()
    for bad_x in (True, False):
        xc, ec = x.clone(), ea.clone()
        (xc if bad_x else ec)[7, 3] = float("nan") if bad_x else float("inf")
        with pytest.raises(RuntimeError, match="not finite"):
            proc(xc.cuda().requires_grad_(True), ei.cuda(), ec.cuda(), batch_size=B, efficient_batching=True)
    ll = grid(30)
    dec = Decoder(ll, output_dim=4, train_precision=tp).cuda().train()
    h = torch.randn(1, dec.num_h3, 256)
    h[0, 11, 5] = float("inf")
    with pytest.raises(RuntimeError, match="not finite"):
        dec(h.reshape(-1, 256).cuda().requires_grad_(True), torch.zeros(1, len(ll), 4, device="cuda"))


@pytest.mark.parametrize("tp", TPS)
def test_tape_lifetime(tp):
    from graph_weather_b200 import Encoder, Processor

    ll = grid(30)
    enc = Encoder(ll, input_dim=6, train_precision=tp).cuda().train()
    proc = Processor(num_blocks=2, train_precision=tp).cuda().train()
    x = torch.randn(1, len(ll), 6, device="cuda")
    # a processor applied twice in one graph back-propagates through both calls
    h, ei, ea = enc(x)
    y = proc(proc(h, ei, ea), ei, ea)
    plan = proc._train_engine.plan
    assert len(plan.live_tapes()) == 2 and all(t.bytes() > 0 for t in plan.live_tapes())
    y.sum().backward(retain_graph=True)
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in proc.parameters())
    assert all(q.grad is not None for q in enc.parameters())
    assert sum(t.bytes() for t in plan.live_tapes()) == 0
    # a second backward raises
    with pytest.raises(RuntimeError, match="one backward per forward"):
        y.sum().backward()
    # dropping the graph frees the tapes
    h, ei, ea = enc(x)
    y = proc(proc(h, ei, ea), ei, ea)
    assert sum(t.bytes() for t in plan.live_tapes()) > 0 and sum(t.bytes() for t in enc._train_engine.plan.live_tapes()) > 0
    del y, h, ea
    assert sum(t.bytes() for t in plan.live_tapes()) == 0
    assert sum(t.bytes() for t in enc._train_engine.plan.live_tapes()) == 0
    # without a train_precision the stages stay inference-only
    plain = Processor(num_blocks=2).cuda().train()
    plain.load_state_dict(proc.state_dict())
    h, ei, ea = enc(x)
    assert plain(h.detach(), ei, ea.detach()).grad_fn is None
