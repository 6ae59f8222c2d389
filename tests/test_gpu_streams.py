"""-m gpu: every entry point on the caller's own CUDA streams.

Torch users run modules under `with torch.cuda.stream(s)`, and torch makes its side streams non-blocking: they are not ordered
against the legacy default stream (handle 0) that the rest of the suite runs on.  So a copy, memset or kernel that the library put
on the wrong stream, or two calls on one plan that nothing orders, show up only here.  Every result is compared with the same call
on the default stream, on fresh objects and the same seeded data (the cases of test_non_finite_oracle.forecaster_base and
assimilator_base, whose default-stream results the rest of the suite checks against fp64): outputs, losses, the constraint layer and
the loss kernels bit for bit, and the training steps' gradients by the rule of `_step_fails`.

A delay is one `torch.cuda._sleep`, calibrated once against CUDA events; no test repeats a call to chase a race.
  * control: work queued behind a sleep on one side stream is not seen by another side stream, so the window below is real;
  * A, late producer: on a side stream the inputs are written after a sleep, then the call runs and its outputs are copied, still on
    that stream; only that stream is synchronised.  Work the library put on another stream would read the inputs too early;
  * B, legacy stream busy: the default stream sleeps ~1 s while a model is moved to the GPU, run, and its training forward made on
    a side stream; the results must be ready while the default stream still sleeps, and a second forward after the sleep must agree
    too (a legacy stream write that lands after the plan's own writes changes it);
  * C, one model on two streams: a call on a second stream is ordered after the plan's previous call on the first, and the loss
    gives each call its own result."""
import ctypes
import os
import time

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from test_non_finite_oracle import ASSIM_DIM, assimilator_base, forecaster_base
from training_oracle import rel_norm

pytestmark = pytest.mark.gpu

SLEEP_MS = 300  # the window of a late producer
BUSY_MS = 1000  # the legacy stream's sleep in case B


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture(scope="module")
def sleep():
    """sleep(ms): one torch.cuda._sleep of about `ms` milliseconds on the current stream (cycles calibrated once, with events)."""
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cycles = 50_000_000
    a.record()
    torch.cuda._sleep(cycles)
    b.record()
    b.synchronize()
    per_ms = cycles / a.elapsed_time(b)
    return lambda ms: torch.cuda._sleep(int(per_ms * ms))


def _cudart():
    """The CUDA runtime torch has loaded."""
    with open("/proc/self/maps") as f:
        paths = [ln.split()[-1] for ln in f if "libcudart.so" in ln]
    return ctypes.CDLL(paths[0] if paths else "libcudart.so.12")


def test_side_streams_are_non_blocking_and_the_default_stream_is_legacy():
    """The preconditions of every case below: a torch side stream is cudaStreamNonBlocking (not ordered against stream 0), and
    the default stream the rest of the suite runs on is the legacy stream 0."""
    flags = ctypes.c_uint(0)
    s = torch.cuda.Stream()
    assert _cudart().cudaStreamGetFlags(ctypes.c_void_p(s.cuda_stream), ctypes.byref(flags)) == 0
    assert flags.value & 1, "torch's side streams are expected to be cudaStreamNonBlocking"
    assert torch.cuda.current_stream().cuda_stream == 0 and torch.cuda.default_stream().cuda_stream == 0


def test_control_a_sleeping_stream_hides_its_writes(sleep):
    x = torch.zeros(1 << 16, device="cuda")
    new = torch.ones_like(x)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        sleep(SLEEP_MS)
        x.copy_(new)
    with torch.cuda.stream(s2):
        seen = x.clone()
    s2.synchronize()
    assert not bool(seen.any()), "the copy queued behind the sleep was visible: no window"
    s1.synchronize()
    assert bool(x.all())


# ---- helpers ---------------------------------------------------------------------------------------------------------------------------
def _randn(t, seed):
    """Other seeded finite data shaped like t, on the device."""
    return torch.randn(t.shape, generator=torch.Generator().manual_seed(seed)).to(t.dtype).cuda()


def _obs(n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return torch.from_numpy(np.stack([rng.uniform(-90, 90, n), rng.uniform(0, 360, n), rng.uniform(0, 1, n)], 1).astype(np.float32))


def _late(real, other, call, sleep):
    """Case A: on a fresh side stream, buffers prefilled with `other`, a sleep, the `real` inputs copied in, call(*buffers) (a list of
    tensors), its outputs copied into fresh tensors; then only that stream is synchronised.  Returns the copies on the host."""
    real, other = [r.cuda() for r in real], [o.cuda() for o in other]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        bufs = [o.clone() for o in other]
        sleep(SLEEP_MS)
        for b, r in zip(bufs, real):
            b.copy_(r)
        outs = [o.detach().clone() for o in call(*bufs)]
    s.synchronize()
    return [o.cpu() for o in outs]


def _assert_equal(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and torch.equal(g.cpu(), w.cpu()), f"{what}: output {i} differs"


def _forecaster(prec="fp32", tp="fp32_simt", bounded=False, model="forecaster", **kw):
    from graph_weather_b200 import GraphCast, GraphWeatherForecaster

    ll, sd = forecaster_base(model)[:2]
    cls = GraphCast if model == "graphcast" else GraphWeatherForecaster
    m = cls(ll, precision=prec, train_precision=tp, use_checkpointing=bounded, **kw).cuda()
    m.load_state_dict(sd)
    return m


def _assimilator(prec="fp32", tp="fp32_simt", bounded=False):
    from graph_weather_b200 import GraphWeatherAssimilator

    out_ll, sd = assimilator_base()[:2]
    m = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=ASSIM_DIM, precision=prec, train_precision=tp, use_checkpointing=bounded)
    m = m.cuda()
    m.load_state_dict(sd)
    return m


def _crit(model="forecaster"):
    from graph_weather_b200 import NormalizedMSELoss

    ll, _, _, _, var = forecaster_base(model)
    return NormalizedMSELoss(var, ll, normalize=True)


# ---- A: late producer, early consumer --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32_simt", "fp32", "bf16"])
def test_late_inputs_forecaster(prec, sleep):
    x = forecaster_base()[2]
    want = [_forecaster(prec).eval()(x.cuda())]
    model = _forecaster(prec).eval()
    model(_randn(x, 3))  # the plan and its weights exist before the window
    got = _late([x], [_randn(x, 4)], lambda xb: [model(xb)], sleep)
    _assert_equal(got, want, f"forecaster {prec}")


def test_late_inputs_rollout(sleep):
    """model.rollout(x, 3): three gw_forward_strided calls, each writing into the next step's input rows."""
    x = forecaster_base()[2]
    want = [_forecaster("fp32").eval().rollout(x.cuda(), 3)]
    model = _forecaster("fp32").eval()
    model(_randn(x, 3))
    got = _late([x], [_randn(x, 4)], lambda xb: [model.rollout(xb, 3)], sleep)
    _assert_equal(got, want, "rollout")


@pytest.mark.parametrize("host_graph", [False, True], ids=["device_obs_graph", "host_obs_graph"])
def test_late_inputs_assimilator(host_graph, sleep, monkeypatch):
    """The observation values and their coordinates are late: the device-built observation graph (and, with
    GW_B200_HOST_OBS_GRAPH=1, the host-built one) must read the coordinates on the caller's stream."""
    if host_graph:
        monkeypatch.setenv("GW_B200_HOST_OBS_GRAPH", "1")
    x, obs = assimilator_base()[3:5]
    want = [_assimilator().eval()(x.cuda(), obs.cuda())]
    model = _assimilator().eval()
    model(_randn(x, 5), _obs(obs.shape[0], 6).cuda())
    got = _late([x, obs], [_randn(x, 7), _obs(obs.shape[0], 8)], lambda xb, ob: [model(xb, ob)], sleep)
    _assert_equal(got, want, "assimilator")


def test_late_inputs_graphcast_bf16(sleep):
    x = forecaster_base("graphcast")[2]
    want = [_forecaster("bf16", model="graphcast").eval()(x.cuda())]
    model = _forecaster("bf16", model="graphcast").eval()
    model(_randn(x, 3))
    got = _late([x], [_randn(x, 4)], lambda xb: [model(xb)], sleep)
    _assert_equal(got, want, "GraphCast bf16")


def _regional():
    from oracle import weights

    from graph_weather_b200.regional import RegionalForecasterConfig

    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "regional_europe_b2.npz"))
    ll = [(float(a), float(b)) for a, b in z["lat_lons"]]
    cfg = RegionalForecasterConfig(num_blocks=2, precision="fp32")
    sd = weights.make_state_dict({k: tuple(v.shape) for k, v in cfg.build().state_dict().items()}, 71)
    return ll, cfg, sd, weights.make_features(2, len(ll), 102, 72)


def test_late_inputs_regional_fp32(sleep):
    """RegionalForecaster in fp32: its node decoder ends in a LayerNorm."""
    ll, cfg, sd, x = _regional()

    def build():
        m = cfg.build().cuda().eval()
        m.load_state_dict(sd)
        return m

    want = [build()(x.cuda(), ll)]
    model = build()
    model(_randn(x, 3), ll)
    got = _late([x], [_randn(x, 4)], lambda xb: [model(xb, ll)], sleep)
    _assert_equal(got, want, "RegionalForecaster fp32")


def test_late_inputs_stage_api(sleep):
    """Encoder (and the latent edge features it returns), Processor on a caller-supplied graph (gw_processor_forward_graph) and
    Decoder, each with late inputs."""
    from graph_weather_b200 import Decoder, Encoder, Processor

    ll, sd, x = forecaster_base()[:3]

    def stages():
        enc, proc, dec = Encoder(ll, input_dim=102, precision="fp32").cuda(), Processor(precision="fp32").cuda(), Decoder(ll, precision="fp32").cuda()
        for name, m in (("encoder", enc), ("processor", proc), ("decoder", dec)):
            m.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")})
        return enc, proc, dec

    enc, proc, dec = stages()
    ex, ei, ea = enc(x.cuda())
    px = proc(ex, ei, ea)
    want_enc, want_proc, want_dec = [ex, ea], [px], [dec(px, x.cuda()[..., :78])]
    enc, proc, dec = stages()  # fresh objects, warmed up on other data
    enc(_randn(x, 3))
    proc(_randn(ex, 4), ei, _randn(ea, 5))
    dec(_randn(px, 6), _randn(x, 7)[..., :78])
    _assert_equal(_late([x], [_randn(x, 8)], lambda xb: enc(xb)[::2], sleep), want_enc, "Encoder")
    # (the late edge index is a valid graph too: the real one with its two rows swapped)
    got = _late([ex, ei, ea], [_randn(ex, 9), ei.flip(0), _randn(ea, 10)], lambda xb, eib, eab: [proc(xb, eib, eab)], sleep)
    _assert_equal(got, want_proc, "Processor")
    start = x[..., :78].contiguous()
    _assert_equal(_late([px, start], [_randn(px, 11), _randn(start, 12)], lambda pb, sb: [dec(pb, sb)], sleep), want_dec, "Decoder")


@pytest.mark.training
def test_late_inputs_loss(sleep):
    """NormalizedMSELoss: the value and, through loss.backward() with the default stream current, its gradient."""
    _, _, x, target, _ = forecaster_base()
    pred = x[..., :78].contiguous()
    crit = _crit()

    def run(pb, tb, c=crit):
        pb.requires_grad_(True)
        return c(pb, tb), pb

    v, p = run(pred.cuda(), target.cuda(), _crit())
    v.backward()
    want = [v.detach(), p.grad]
    run(_randn(pred, 7), _randn(target, 8))  # (its constant tables on the device before the window)
    got_v = _late([pred, target], [_randn(pred, 3), _randn(target, 4)], lambda pb, tb: [run(pb, tb)[0]], sleep)
    _assert_equal(got_v, want[:1], "loss value")
    # the gradient: the forward on the side stream, backward() from the default stream, the gradient read on the side stream
    real = [pred.cuda(), target.cuda()]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        pb, tb = _randn(pred, 5), _randn(target, 6)
        sleep(SLEEP_MS)
        pb.copy_(real[0])
        tb.copy_(real[1])
        v, p = run(pb, tb)
    v.backward()
    with torch.cuda.stream(s):
        g = p.grad.clone()
    s.synchronize()
    _assert_equal([v.detach(), g], want, "loss and its gradient")


@pytest.mark.training
def test_late_inputs_constraint_layer(sleep):
    """PhysicalConstraintLayer apply (no autograd) and backward (autograd.grad on the side stream)."""
    from graph_weather_b200.constraint import PhysicalConstraintLayer

    _, _, x, target, _ = forecaster_base()
    hr, lr, dy = x[..., :78].contiguous(), x[..., 24:102].contiguous(), target

    def both(hb, lb, db, layer):
        with torch.no_grad():
            out = layer(hb, lb)
        h = hb.detach().requires_grad_(True)
        l = lb.detach().requires_grad_(True)  # noqa: E741
        gh, gl = torch.autograd.grad(layer(h, l), (h, l), db)
        return [out, gh, gl]

    def fresh():
        model = _forecaster("fp32")
        return PhysicalConstraintLayer(model, model.grid_shape, 1, "additive")

    want = both(hr.cuda(), lr.cuda(), dy.cuda(), fresh())
    layer = fresh()
    both(_randn(hr, 6), _randn(lr, 7), _randn(dy, 8), layer)  # (the grid mapping on the device before the window)
    got = _late([hr, lr, dy], [_randn(hr, 3), _randn(lr, 4), _randn(dy, 5)], lambda hb, lb, db: both(hb, lb, db, layer), sleep)
    _assert_equal(got, want, "constraint layer")


def _step_fails(a, b, tp):
    """Two training steps agree: output and loss bit for bit; with tensor cores, the gradients of Linear weights with more than 16
    inputs bit for bit (tensor-core weight gradients are repeatable: tests/test_gpu_train_precision.py); every other gradient, and
    all of fp32_simt's (float atomics), within 1e-5 norm-relative."""
    out, loss, gx, grads = a
    out_b, loss_b, gx_b, grads_b = b
    fails = [] if torch.equal(out, out_b) and torch.equal(loss, loss_b) else ["output or loss differ"]
    assert set(grads) == set(grads_b)
    for k, g in grads.items():
        if tp != "fp32_simt" and k.endswith(".weight") and g.dim() == 2 and g.shape[1] > 16:
            same = torch.equal(g, grads_b[k])
        else:
            same = rel_norm(g, grads_b[k]) <= 1e-5
        if not same:
            fails.append(k)
    if gx is not None and not rel_norm(gx, gx_b) <= 1e-5:
        fails.append("d features")
    return fails


def _plain(model, crit, bufs):
    """One training forward + loss of the forecaster: bufs = (features, target)."""
    out = model(bufs[0])
    return out, crit(out, bufs[1])


def _two_steps(model, crit, bufs):
    """A two-tape rollout in multi_step(): the second forward is fed the first's forecast and the auxiliary columns."""
    x, t = bufs
    with model.multi_step():
        y1 = model(x)
        y2 = model(torch.cat([y1, x[..., 78:]], -1))
    return torch.stack([y1, y2]), crit(y1, t) + crit(y2, t)


def _assim_step(model, crit, bufs):
    out = model(bufs[0], bufs[2])
    return out, torch.nn.functional.mse_loss(out, bufs[1])


def _step(model, crit, real, fwd, sleep=None, other=None):
    """One training step from cleared gradients: (out, loss, d features, {name: grad}) on the host.  With `sleep`, case A: on a
    side stream the inputs are prefilled with `other`, written after a sleep, and the forward runs there; backward() is called with
    the default stream current (autograd runs the backward on the side stream); the results are copied on the side stream, and
    only that stream is synchronised.  Without it, everything runs on the current stream."""
    model.zero_grad(set_to_none=True)
    real = [r.cuda() for r in real]
    s = torch.cuda.Stream() if sleep is not None else torch.cuda.current_stream()
    if sleep is not None:
        other = [o.cuda() for o in other]
        torch.cuda.synchronize()
    with torch.cuda.stream(s):
        if sleep is not None:
            bufs = [o.clone() for o in other]
            sleep(SLEEP_MS)
            with torch.no_grad():
                for b, r in zip(bufs, real):
                    b.copy_(r)
        else:
            bufs = [r.clone() for r in real]
        bufs[0].requires_grad_(True)
        out, loss = fwd(model, crit, bufs)
    loss.backward()
    with torch.cuda.stream(s):
        res = (out.detach().clone(), loss.detach().clone(), bufs[0].grad.clone(),
               {k: q.grad.detach().clone() for k, q in model.named_parameters()})  # fmt: skip
    s.synchronize()
    return res[0].cpu(), res[1].cpu(), res[2].cpu(), {k: g.cpu() for k, g in res[3].items()}


def _warm(model, crit, real, fwd):
    """A training step on other features on the default stream: the training plan, its weights and the loss's tables exist
    before the window."""
    _step(model, crit, [_randn(real[0], 90)] + list(real[1:]), fwd)
    torch.cuda.synchronize()


@pytest.mark.training
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_late_inputs_taped_step(tp, sleep):
    _, _, x, target, _ = forecaster_base()
    want = _step(_forecaster(tp=tp).train(), _crit(), [x, target], _plain)
    model, crit = _forecaster(tp=tp).train(), _crit()
    _warm(model, crit, [x, target], _plain)
    got = _step(model, crit, [x, target], _plain, sleep, [_randn(x, 3), _randn(target, 4)])
    fails = _step_fails(got, want, tp)
    assert not fails, fails


@pytest.mark.training
@pytest.mark.parametrize("what", ["forecaster", "assimilator"])
def test_late_inputs_bounded_step(what, sleep, monkeypatch):
    """use_checkpointing=True, many chunks: the assimilator's encoder chunk tables are rebuilt from the late observation graph on
    every call."""
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    if what == "forecaster":
        _, _, x, target, _ = forecaster_base()
        real, other, fwd = [x, target], [_randn(x, 3), _randn(target, 4)], _plain
        build = lambda: _forecaster(tp="fp32", bounded=True).train()  # noqa: E731
    else:
        _, _, _, x, obs, target = assimilator_base()
        real, other, fwd = [x, target, obs], [_randn(x, 3), _randn(target, 4), _obs(obs.shape[0], 5)], _assim_step
        build = lambda: _assimilator(tp="fp32", bounded=True).train()  # noqa: E731
    want = _step(build(), _crit(), real, fwd)
    model, crit = build(), _crit()
    _warm(model, crit, real[:2] + [_obs(real[2].shape[0], 6)] if what == "assimilator" else real, fwd)
    got = _step(model, crit, real, fwd, sleep, other)
    fails = _step_fails(got, want, "fp32")
    assert not fails, fails


@pytest.mark.training
def test_late_inputs_multi_step(sleep):
    _, _, x, target, _ = forecaster_base()
    want = _step(_forecaster(tp="fp32").train(), _crit(), [x, target], _two_steps)
    model, crit = _forecaster(tp="fp32").train(), _crit()
    _warm(model, crit, [x, target], _two_steps)
    got = _step(model, crit, [x, target], _two_steps, sleep, [_randn(x, 3), _randn(target, 4)])
    fails = _step_fails(got, want, "fp32")
    assert not fails, fails


# ---- B: the legacy default stream held busy ----------------------------------------------------------------------------------------------
@pytest.mark.training
@pytest.mark.parametrize("prec,bounded", [("fp32", False), ("bf16", False), ("fp32", True)], ids=["fp32", "bf16", "fp32-bounded"])
def test_legacy_stream_busy(prec, bounded, sleep, monkeypatch):
    """While the default stream sleeps, on a side stream: move a model to the GPU, run a forward (the inference plan is created,
    its graphs and weights uploaded, in the window) and a training forward and loss (the training plan likewise; the bounded
    variant also builds its chunk tables there).  They must be complete while the default stream still sleeps: no call may wait
    for the legacy stream.  The backward then runs on the side stream after the window: its first call sizes the weight-gradient
    workspace, and growing a device buffer frees the old one with cudaFree, which synchronises the device.  After the sleep the
    same forward runs again: a legacy-stream write that landed after the plan's own writes would change it.  (fp32_simt is left
    out: its first forward grows a scratch buffer in the same way.)"""
    from graph_weather_b200 import GraphWeatherForecaster

    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    ll, sd, x, target, var = forecaster_base()
    with torch.no_grad():
        want_out = _forecaster(prec).eval()(x.cuda()).cpu()
    want_step = _step(_forecaster(prec, prec, bounded).train(), _crit(), [x, target], _plain)
    crit = _crit()
    crit(want_out.cuda(), target.cuda())  # (its constant tables on the device)
    model = GraphWeatherForecaster(ll, precision=prec, train_precision=prec, use_checkpointing=bounded)  # (the graphs: host work)
    model.load_state_dict(sd)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    t0 = time.perf_counter()
    sleep(BUSY_MS)  # on the legacy default stream
    busy = torch.cuda.Event()
    busy.record()
    with torch.cuda.stream(s):
        model = model.cuda().eval()
        xs, ts = x.cuda(), target.cuda()
        with torch.no_grad():
            out = model(xs).clone()
        model.train()
        xr = xs.clone().requires_grad_(True)
        y = model(xr)
        loss = crit(y, ts)
        s.synchronize()
    read, took = busy.query(), time.perf_counter() - t0
    torch.cuda.synchronize()
    assert not read, f"a call on the side stream waited for the legacy default stream (the window took {took:.2f} s)"
    with torch.cuda.stream(s):
        loss.backward()
        step = (y.detach().cpu(), loss.detach().cpu(), xr.grad.cpu(), {k: q.grad.cpu() for k, q in model.named_parameters()})
    assert torch.equal(out.cpu(), want_out), "the forward made in the window differs"
    fails = _step_fails(step, want_step, prec)
    assert not fails, fails
    with torch.cuda.stream(s):
        with torch.no_grad():
            again = model.eval()(xs).clone()
    s.synchronize()
    assert torch.equal(again.cpu(), want_out), "the forward after the legacy stream's sleep differs"


# ---- C: one model, two streams -----------------------------------------------------------------------------------------------------------
def test_two_streams_inference(sleep, monkeypatch):
    """model(x1) on S1 behind a sleep, then model(x2) on S2: S2's call must be ordered after S1's (they share the plan's scratch),
    so once S2's work is complete, so is S1's; both results are their own."""
    monkeypatch.setenv("GW_B200_CHECK", "0")
    x = forecaster_base()[2]
    x1, x2 = x.cuda(), _randn(x, 3)
    ref = _forecaster("fp32").eval()
    want1, want2 = ref(x1).cpu(), ref(x2).cpu()
    model = _forecaster("fp32").eval()
    model(_randn(x, 4))
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    e1, e2 = torch.cuda.Event(), torch.cuda.Event()
    with torch.cuda.stream(s1):
        sleep(SLEEP_MS)
        y1 = model(x1)
        e1.record()
    with torch.cuda.stream(s2):
        y2 = model(x2)
        e2.record()
    e2.synchronize()
    done1 = e1.query()
    torch.cuda.synchronize()
    assert done1, "the call on the second stream was not ordered after the plan's call on the first"
    assert torch.equal(y1.cpu(), want1) and torch.equal(y2.cpu(), want2)


@pytest.mark.training
def test_two_streams_training(sleep, monkeypatch):
    """A training forward on S1 behind a sleep; then on S2 an inference and a training step, whose forward closes S1's tape
    (stream-ordered memory that S1's forward may still be writing).  S2's step must be ordered after S1's forward, and every
    result must be its own."""
    monkeypatch.setenv("GW_B200_CHECK", "0")
    _, _, x, target, _ = forecaster_base()
    x2 = _randn(x, 3)
    with torch.no_grad():
        want_inf = _forecaster("fp32", "fp32").eval()(x2).cpu()
    want1 = _step(_forecaster("fp32", "fp32").train(), _crit(), [x, target], _plain)
    want2 = _step(_forecaster("fp32", "fp32").train(), _crit(), [x2, target], _plain)
    model = _forecaster("fp32", "fp32").train()
    crit = _crit()
    _warm(model, crit, [x, target], _plain)
    with torch.no_grad():
        model(x2)
    x1 = x.cuda().requires_grad_(True)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    e1 = torch.cuda.Event()
    with torch.cuda.stream(s1):
        sleep(SLEEP_MS)
        y1 = model(x1)
        e1.record()  # (right behind the forward: what the second stream's step must wait for)
        out1 = y1.detach().clone()
    with torch.cuda.stream(s2):
        with torch.no_grad():
            inf2 = model(x2).clone()
        step2 = _step(model, crit, [x2, target], _plain)  # (synchronises s2 only)
    done1 = e1.query()
    torch.cuda.synchronize()
    assert done1, "the training step on the second stream was not ordered after the training forward on the first"
    assert torch.equal(out1.cpu(), want1[0]), "the first stream's training forward differs"
    assert torch.equal(inf2.cpu(), want_inf), "the second stream's inference differs"
    fails = _step_fails(step2, want2, "fp32")
    assert not fails, fails


def test_two_streams_loss(sleep):
    """NormalizedMSELoss.local_sum on S1, read after a sleep, while S2 evaluates the loss of other data: S1 reads its own sum."""
    _, _, x, target, _ = forecaster_base()
    p1, t1 = x[..., :78].contiguous().cuda(), target.cuda()
    p2, t2 = _randn(p1, 3), _randn(t1, 4)
    want1, want2 = _crit().local_sum(p1, t1).clone(), _crit().local_sum(p2, t2).clone()
    crit = _crit()
    crit.local_sum(p2, t2)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        s = crit.local_sum(p1, t1)
        sleep(SLEEP_MS)
        got1 = s.clone()
    with torch.cuda.stream(s2):
        got2 = crit(p2, t2)
    torch.cuda.synchronize()
    assert torch.equal(got1, want1), "the first stream read another call's loss"
    assert torch.equal(got2, (want2 / (p2.shape[0] * p2.shape[1])).float().reshape(()))
