"""-m gpu: bit-repeatable training under torch.use_deterministic_algorithms(True).

With the flag set when a backward runs, the training step sums every parameter gradient in an order fixed by the shapes
(gw_train_set_deterministic): the CUDA-core weight gradient and the LayerNorm backward switch from float atomics to fixed-order
partials, and the rest of the step already sums in a fixed order.  Checked, in every train precision on the taped and the
bounded step, with no parameter exempt:
  * two identical steps give the same output, features' gradient and parameter gradients bit for bit;
  * processor segments S in {-1, 1, 2, 3, 9} give the bits of S = 0 -- the forecaster, the assimilator, GraphCast under each
    GraphCastConfig strategy and RegionalForecaster (nudging off);
  * a 3-forward multi_step() window repeats bit for bit, and so do the five standalone stages composed;
  * two fresh processes give the same SHA-256 over every gradient (no state one process reuses between its runs);
  * the gradients meet the fp64 oracle's bars of the default mode, and the flag's value when the backward runs is what counts;
  * inference repeats bit for bit in every precision (it has no float atomics; nothing changes there);
  * the fixed-order workspace stays within its 32 MiB budget, and a plan that never trains under the flag allocates none."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import check_bf16_bars, check_fp32_bars, forecaster_case, train_step

pytestmark = [pytest.mark.gpu, pytest.mark.training]

PRECISIONS = ["fp32_simt", "fp32", "bf16"]
SEGMENTS = (-1, 1, 2, 3, 9)
DET_WS_BUDGET = 32 << 20
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


@pytest.fixture
def deterministic():
    """torch.use_deterministic_algorithms(True) for the test, restored afterwards."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


def _randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _plans(model):
    """The training plans a step of `model` (a wrapper or a list of stages) used."""
    mods = model if isinstance(model, (list, tuple)) else [model]
    return [m._train_engine.plan for m in mods]


def _step(model, x, *args):
    """One training forward + a seeded linear loss + backward from cleared gradients: (out, d features, {name: grad}) on the host."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    out = model(xc, *args)
    (out * _randn(out.shape, 5).cuda()).sum().backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters() if q.grad is not None}
    return out.detach().cpu(), xc.grad.cpu(), grads


def _assert_same(res, ref, tag):
    """Every tensor of `res` equals `ref` bit for bit (parameters included, none exempt)."""
    out, gx, grads = res
    assert torch.equal(out.view(torch.int32), ref[0].view(torch.int32)), f"{tag}: output"
    assert torch.equal(gx.view(torch.int32), ref[1].view(torch.int32)), f"{tag}: features' gradient"
    assert grads.keys() == ref[2].keys(), tag
    bad = [k for k in grads if not torch.equal(grads[k].view(torch.int32), ref[2][k].view(torch.int32))]
    assert not bad, f"{tag}: {len(bad)} of {len(grads)} gradients differ: {bad[:5]}"


def _check_workspace(plans, tag):
    for plan in plans:
        b = plan.deterministic_bytes()
        assert 0 < b <= DET_WS_BUDGET, f"{tag}: fixed-order workspace {b} bytes"


def _forecaster(tp, bounded, num_blocks=9):
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(0)
    return GraphWeatherForecaster(_grid(30), num_blocks=num_blocks, train_precision=tp, use_checkpointing=bounded).cuda().train()


# ---- repeatability and processor segments -------------------------------------------------------------------------------------
@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_forecaster_repeats_and_segments_are_bit_identical(deterministic, monkeypatch, tp, bounded):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")  # (the bounded step: several chunks on the 72-point grid)
    model = _forecaster(tp, bounded)
    x = _randn((2, len(_grid(30)), 102), 1)
    ref = _step(model, x)
    assert model._train_engine.plan.train_only == bounded
    _assert_same(_step(model, x), ref, f"{tp} bounded={bounded} repeated")
    for s in SEGMENTS:
        model.processor.set_checkpoint_segments(s)
        _assert_same(_step(model, x), ref, f"{tp} bounded={bounded} S={s}")
    _check_workspace(_plans(model), tp)


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_assimilator_repeats_and_segments_are_bit_identical(deterministic, tp, bounded):
    from graph_weather_b200 import GraphWeatherAssimilator

    torch.manual_seed(0)
    model = GraphWeatherAssimilator(output_lat_lons=_grid(20), analysis_dim=24, num_blocks=4, train_precision=tp,
                                    use_checkpointing=bounded).cuda().train()  # fmt: skip
    rng = np.random.Generator(np.random.PCG64(3))
    n = 200
    obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, n), rng.uniform(0, 360, n), rng.uniform(0, 1, n)], 1).astype(np.float32)).cuda()
    x = _randn((1, n, 2), 2)
    ref = _step(model, x, obs)
    _assert_same(_step(model, x, obs), ref, f"assimilator {tp} bounded={bounded} repeated")
    for s in SEGMENTS:
        model.processor.set_checkpoint_segments(s)
        _assert_same(_step(model, x, obs), ref, f"assimilator {tp} bounded={bounded} S={s}")


STRATEGIES = ["no_checkpointing", "full_checkpointing", "balanced_checkpointing", "processor_only_checkpointing",
              "fine_grained_checkpointing"]  # fmt: skip


@pytest.mark.parametrize("tp", PRECISIONS)
def test_graphcast_strategies_repeat_and_segments_are_bit_identical(deterministic, tp):
    """Under each strategy (the step it selects, taped or bounded): the strategy's own step twice, and every S against S = 0."""
    from graph_weather_b200 import GraphCast, GraphCastConfig

    torch.manual_seed(0)
    model = GraphCast(_grid(30), train_precision=tp).cuda().train()
    x = _randn((2, len(_grid(30)), 78), 4)
    for strategy in STRATEGIES:
        getattr(GraphCastConfig, strategy)(model)
        own = _step(model, x)
        _assert_same(_step(model, x), own, f"GraphCast {tp} {strategy} repeated")
        bounded = model._bounded_step()
        model.set_checkpoint_processor(0)
        assert model._bounded_step() == bounded
        ref = _step(model, x)
        _assert_same(own, ref, f"GraphCast {tp} {strategy} against S = 0")
        for s in SEGMENTS:
            model.set_checkpoint_processor(s)
            _assert_same(_step(model, x), ref, f"GraphCast {tp} {strategy} S={s}")


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_regional_repeats_and_segments_are_bit_identical(deterministic, tp, bounded):
    """RegionalForecaster (nudging off): its h3_embeddings gradient goes through an index_put, which torch runs deterministically."""
    from graph_weather_b200.regional import RegionalForecasterConfig

    torch.manual_seed(0)
    model = RegionalForecasterConfig(num_blocks=3, train_precision=tp, use_checkpointing=bounded).build().cuda().train()
    ll = [(float(lat), float(lon)) for lat in range(36, 70, 3) for lon in range(-10, 30, 3)]
    x = _randn((2, len(ll), 102), 6)
    ref = _step(model, x, ll)
    assert "h3_embeddings" in ref[2]
    _assert_same(_step(model, x, ll), ref, f"regional {tp} bounded={bounded} repeated")
    for s in SEGMENTS:
        model.processor.set_checkpoint_segments(s)
        _assert_same(_step(model, x, ll), ref, f"regional {tp} bounded={bounded} S={s}")


# ---- multi-step and stages ----------------------------------------------------------------------------------------------------
def _window(model, x, auxs):
    """Three chained forwards in multi_step() and one backward over the summed loss."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    inp, outs = xc, []
    with model.multi_step():
        for j in range(3):
            outs.append(model(inp))
            if j < 2:
                inp = torch.cat([outs[-1], auxs[j].cuda()], -1)
    sum((o * _randn(o.shape, 7 + j).cuda()).sum() for j, o in enumerate(outs)).backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters()}
    return torch.stack([o.detach().cpu() for o in outs]), xc.grad.cpu(), grads


@pytest.mark.parametrize("bounded", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", PRECISIONS)
def test_multi_step_window_repeats(deterministic, tp, bounded):
    model = _forecaster(tp, bounded, num_blocks=4)
    N = len(_grid(30))
    x = _randn((2, N, 102), 8)
    auxs = [_randn((2, N, 24), 9 + j) for j in range(2)]
    ref = _window(model, x, auxs)
    _assert_same(_window(model, x, auxs), ref, f"window {tp} bounded={bounded}")
    model.processor.set_checkpoint_segments(1)
    _assert_same(_window(model, x, auxs), ref, f"window {tp} bounded={bounded} S=1")


def _sub(sd, prefix):
    return {k[len(prefix) + 1 :]: v for k, v in sd.items() if k.startswith(prefix + ".")}


def _stage_step(mods, run, x):
    """`run(mods, features)` -> output; a seeded linear loss and its backward: (out, d features, {name: grad})."""
    for m in mods:
        m.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(True)
    out = run(mods, xc)
    (out * _randn(out.shape, 13).cuda()).sum().backward()
    for m in mods:
        m._train_engine.plan.status()
    grads = {f"{i}.{k}": q.grad.detach().cpu().clone() for i, m in enumerate(mods) for k, q in m.named_parameters() if q.grad is not None}
    return out.detach().cpu(), xc.grad.cpu(), grads


@pytest.mark.parametrize("tp", PRECISIONS)
def test_stages_repeat(deterministic, tp):
    """Encoder -> Processor -> Decoder (the processor with segments on the second pass too) and AssimilatorEncoder -> Processor ->
    AssimilatorDecoder, each composition twice: the same bits.  The stage API's edge_attr gather / repeat run under the flag."""
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, Decoder, Encoder, Processor
    from oracle import weights

    ll = _grid(10)
    sd = weights.make_state_dict(weights.forecaster_shapes(), 21)
    mods = [Encoder(ll, input_dim=102, train_precision=tp), Processor(train_precision=tp), Decoder(ll, train_precision=tp)]
    for m, p in zip(mods, ("encoder", "processor", "decoder")):
        m.load_state_dict(_sub(sd, p))
    mods = [m.cuda().train() for m in mods]

    def run(ms, xc):
        enc, proc, dec = ms
        h, ei, ea = enc(xc)
        return dec(proc(h, ei, ea, batch_size=xc.shape[0]), xc[..., :78])

    x = weights.make_features(2, len(ll), 102, 21)
    ref = _stage_step(mods, run, x)
    _assert_same(_stage_step(mods, run, x), ref, f"stages {tp}")
    mods[1].set_checkpoint_segments(2)
    _assert_same(_stage_step(mods, run, x), ref, f"stages {tp} processor S=2")
    _check_workspace(_plans(mods), f"stages {tp}")

    out_ll = [(float(lat), float(lon)) for lat in range(-90, 90, 5) for lon in range(0, 360, 5)]
    asd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=24), 41)
    amods = [AssimilatorEncoder(train_precision=tp), Processor(train_precision=tp), AssimilatorDecoder(out_ll, output_dim=24, train_precision=tp)]
    for m, p in zip(amods, ("encoder", "processor", "decoder")):
        m.load_state_dict(_sub(asd, p))
    amods = [m.cuda().train() for m in amods]
    rng = np.random.Generator(np.random.PCG64(51))
    n = 300
    obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, n), rng.uniform(0, 360, n), rng.uniform(0, 1, n)], 1).astype(np.float32)).cuda()

    def arun(ms, xc):
        enc, proc, dec = ms
        h, ei, ea = enc(xc, obs)
        return dec(proc(h, ei, ea), 1)

    xa = weights.make_features(1, n, 2, 51)
    aref = _stage_step(amods, arun, xa)
    _assert_same(_stage_step(amods, arun, xa), aref, f"assimilator stages {tp}")


# ---- fresh processes ------------------------------------------------------------------------------------------------------------
_CHILD = r"""
import hashlib, json, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import torch
import __graft_entry__ as ge
ge.build()
from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss
from training_oracle import grid, train_step
from oracle import weights
ll = grid(10)
sd = weights.make_state_dict(weights.forecaster_shapes(), 21)
x = weights.make_features(2, len(ll), 102, 21)
torch.manual_seed(0)
target = torch.randn(2, len(ll), 78)
torch.use_deterministic_algorithms(True)
model = GraphWeatherForecaster(ll, train_precision=sys.argv[2], use_checkpointing=sys.argv[3] == "1").cuda().train()
model.load_state_dict(sd)
out, loss, gx, grads = train_step(model, NormalizedMSELoss([1.0] * 78, ll, normalize=True), x, target)
h = hashlib.sha256()
for t in [out, gx] + [grads[k] for k in sorted(grads)]:
    h.update(t.contiguous().numpy().tobytes())
print(json.dumps({"sha256": h.hexdigest(), "n": len(grads)}))
"""


def _child(tp, bounded):
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, tp, "1" if bounded else "0"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("tp,bounded", [("fp32_simt", False), ("bf16", False), ("fp32_simt", True)])
def test_fresh_processes_give_the_same_gradients(tp, bounded):
    """Two fresh interpreters train the seeded 10-degree, batch-2 step: the same SHA-256 over the output, the features' gradient
    and every parameter gradient."""
    a, b = _child(tp, bounded), _child(tp, bounded)
    assert a["n"] == 215 and a == b, (a, b)


# ---- the oracle's bars, and when the flag is read --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def case10():
    return forecaster_case(10, 2, 21)


def _oracle_step(tp, case, bounded=False):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = case[:5]
    model = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=bounded).cuda().train()
    model.load_state_dict(sd)
    return model, train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target)


@pytest.mark.parametrize("tp", PRECISIONS)
def test_deterministic_gradients_meet_the_oracle_bars(deterministic, case10, tp):
    """The bars of tests/test_gpu_training.py (fp32_simt) and tests/test_gpu_train_precision.py (fp32, bf16)."""
    ref32, ref64 = case10[5:]
    model, ours = _oracle_step(tp, case10)
    if tp == "fp32_simt":
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=0.0, feat_floor=False, median=True, ill=None, skip_zero=False,
                        norm_bar=None, tag=tp)  # fmt: skip
    elif tp == "fp32":
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3, feat_floor=False, median=False, ill=None, skip_zero=False,
                        norm_bar=None, tag=tp)  # fmt: skip
    else:
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999, tag=tp)
    _check_workspace(_plans(model), tp)


@pytest.mark.parametrize("tp", PRECISIONS)
def test_the_flag_counts_when_the_backward_runs(case10, tp):
    """A forward without the flag and a backward with it gives the bits of a step run wholly under the flag; a plan that never
    ran a backward under the flag holds no fixed-order workspace."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = case10[:5]
    crit = NormalizedMSELoss(var, ll, normalize=True)
    model, _ = _oracle_step(tp, case10)
    assert model._train_engine.plan.deterministic_bytes() == 0
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        ref = train_step(model, crit, x, target)
        model.zero_grad(set_to_none=True)
        torch.use_deterministic_algorithms(False)
        xc = x.cuda().requires_grad_(True)
        out = model(xc)
        loss = crit(out, target.cuda())
        torch.use_deterministic_algorithms(True)
        loss.backward()
    finally:
        torch.use_deterministic_algorithms(was)
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu() for k, q in model.named_parameters()}
    _assert_same((out.detach().cpu(), xc.grad.cpu(), grads), (ref[0], ref[2], ref[3]), f"{tp} flag set before the backward only")
    assert 0 < model._train_engine.plan.deterministic_bytes() <= DET_WS_BUDGET


# ---- inference ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32_simt", "fp32", "bf16"])
def test_inference_repeats(deterministic, precision):
    from graph_weather_b200 import GraphWeatherForecaster
    from oracle import weights

    ll = _grid(10)
    model = GraphWeatherForecaster(ll, precision=precision).cuda().eval()
    model.load_state_dict(weights.make_state_dict(weights.forecaster_shapes(), 1))
    x = weights.make_features(2, len(ll), 102, 1).cuda()
    with torch.no_grad():
        a, b = model(x).cpu(), model(x).cpu()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
