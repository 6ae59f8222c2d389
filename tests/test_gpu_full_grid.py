"""-m gpu: the grids the project is built for against the fp64 reference arithmetic -- the 0.25-degree ERA5 grid (721 x 1440 =
1 038 240 points, up to 9 142 points in one mesh cell, 7.27 M decoder edges) and the 1-degree grid -- through the chunked oracle
of tests/grid_oracle.py, which runs oracle/restate.py's ops on the GPU in fp64 (and in fp32 without TF32, the yardstick of the
training bars).

  * forward at 0.25 degrees, batch 4 (BASELINE configs[2]'s grid): every precision on every row of every sample, with the worst
    error on the polar rows, on the lon 0 / 359.75 seam and in the 9 142-point mesh cell printed apart;
  * the bounded training step (use_checkpointing=True, default chunk budget) at 0.25 degrees, batch 1, fp32 and bf16, and bf16 at
    batch 2 with and without processor segments;
  * the taped training step at 1 degree, batch 2, in every train precision;
  * the forward bars against faults a chunked kernel could make, put into the fp64 oracle's graph (nothing is provoked on the
    device): one of the 9 142 rows of the dense cell's encoder sum dropped; the source cells of two decoder edges of one point
    swapped; a chunk boundary inside the dense cell that does not carry the cell's sum (the 4 571 rows before it lost).
Each test prints its time and its peak memory: torch's allocator (the oracle, and the tensors handed to and returned by the model),
held under 30 GB, and beside it the model's own plan and training working set while it ran.

Measured values beside the bars are from an H100 80GB HBM3 at its 700 W power limit."""
import contextlib
import copy
import time

import numpy as np
import pytest
import torch
from torch import nn

import __graft_entry__ as ge
import grid_oracle
from training_oracle import ILL_CONDITIONED, check_bf16_bars, check_fp32_bars, cos, grid, rel_max, rel_norm, train_step

pytestmark = pytest.mark.gpu
TOL, BF16_TOL = 1e-4, 2e-2  # tests/test_gpu_parity.py's forward bars
# The 0.25-degree forward of the fp32-type precisions against fp64, max-abs over 4 x 1 038 240 x 78 outputs: measured 4.7e-7
# (fp32_simt) and 8.5e-7 (fp32).  TOL would not see two swapped decoder edges of one point (6.4e-5), so this grid holds them to
# 1e-5.
FULL_TOL = 1e-5
CHUNK = 8192  # grid rows per oracle chunk: a few GB of fp64 activations at batch 4
MEM_BAR = 30e9
ATOMIC_BAR = 1e-6  # tests/test_gpu_processor_checkpointing.py


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def quarter_degree():
    """bench.py's grid_quarter_deg: lat = -90 + 0.25 i (i < 721, both poles), lon = 0.25 j (j < 1440), latitude-major."""
    lat = -90.0 + 0.25 * np.arange(721)
    lon = 0.25 * np.arange(1440)
    return [tuple(p) for p in np.stack(np.meshgrid(lat, lon, indexing="ij"), axis=-1).reshape(-1, 2).tolist()]


def _dense_cell(graphs):
    """The mesh slot that collects the most points in the encoder, and those points."""
    counts = np.bincount(graphs["enc"].mesh_local, minlength=graphs["enc"].num_h3)
    slot = int(counts.argmax())
    return np.flatnonzero(graphs["enc"].mesh_local == slot), slot


@pytest.fixture(scope="module")
def quarter():
    ll = quarter_degree()
    graphs = grid_oracle.build_graphs(ll)
    dense_pts, slot = _dense_cell(graphs)
    counts = np.bincount(graphs["enc"].mesh_local, minlength=graphs["enc"].num_h3)
    assert len(ll) == 1038240 and len(dense_pts) == 9142 and counts.min() > 8  # every encoder sum takes the segment-sum kernels
    return ll, graphs, dense_pts, slot


@contextlib.contextmanager
def _budget(tag):
    """Peak memory and time of the block; `models` collects the device bytes of the models it ran (plan + training working set)."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0, models = time.perf_counter(), []
    yield models
    torch.cuda.synchronize()
    torch_peak, model_peak = torch.cuda.max_memory_allocated(), max(models, default=0)
    print(f"{tag}: peak {torch_peak / 1e9:.1f} GB in torch's allocator; while a model ran, its plan and training working set + "
          f"torch's tensors {model_peak / 1e9:.1f} GB; {time.perf_counter() - t0:.0f} s")  # fmt: skip
    assert torch_peak < MEM_BAR


def _model_bytes(model):
    """Device bytes while `model` is alive: its plan, its training step's working set, and torch's tensors (the oracle's results
    among them)."""
    plan = (model._train_engine if model.training else model._engine).plan
    return plan.device_bytes() + (plan.train_peak_bytes() if model.training else 0) + torch.cuda.memory_allocated()


def _drop_encoder_rows(graphs, pts):
    """The graphs with the encoder edges of points `pts` removed: their rows are missing from their mesh cells' sums."""
    e = copy.copy(graphs["enc"])
    keep = ~np.isin(np.arange(e.num_latlons), pts)
    e.edge_index, e.edge_attr = e.edge_index[:, keep], e.edge_attr[keep]
    return dict(graphs, enc=e)


def _faults(graphs, dense_pts):
    p = int(dense_pts[len(dense_pts) // 2])
    return {"one row dropped from the dense cell's encoder sum": _drop_encoder_rows(graphs, [p]),
            "two decoder edges of one point swapped": _swap_decoder_edges(graphs, p),
            "the dense cell's sum not carried over a chunk boundary": _drop_encoder_rows(graphs, dense_pts[: len(dense_pts) // 2])}  # fmt: skip


def _swap_decoder_edges(graphs, p):
    """The graphs with the source cells of point p's first two decoder edges swapped (their attributes stay)."""
    d = copy.copy(graphs["dec"])
    e0 = int(d.ptr[p])
    d.edge_index = d.edge_index.copy()
    d.edge_index[0, [e0, e0 + 1]] = d.edge_index[0, [e0 + 1, e0]]
    return dict(graphs, dec=d)


# ---- the dense cell's own gradients ----------------------------------------------------------------------------------------------
# A fault in one mesh cell is lost in a bar over a whole gradient tensor (losing half the dense cell's rows moves no parameter's
# gradient by more than 0.07x check_fp32_bars' bar).  These bars look at the cell itself, each relative to its fp64 magnitude there:
#   * the features' gradient on the cell's points in the auxiliary channels (F: of F + A), which reach the loss only through the
#     encoder's sum over the cell, and
#   * the cell's row of the h3_nodes gradient.
# fp32-type steps: 10x the fp32 oracle's own error there + 2e-5, or LOCAL_FLOOR, check_fp32_bars' form with fp32 mode's floor.
# (The fp32 oracle on the GPU sums with atomics, so its own error there changes from run to run: 1e-4 .. 1e-3 at 1 degree.  At 0.25
# degrees it is 2.0e-2 on the features; fp32 mode measured 8.8e-2 there, and at most 6.5e-4 everywhere else.)  bf16: measured 0.24 on the features
# (1 degree; 0.22 at 0.25 degrees), so 0.3.  On the h3_nodes row bf16 measures 0.12, above every fault's change there (at most
# 1.0e-2), so bf16 has no bar on that row: it would see nothing.
FEAT, H3ROW = "d features, auxiliary channels of the dense cell", "h3_nodes row of the dense cell"
LOCAL_BF16 = {FEAT: 0.3, H3ROW: None}
LOCAL_FLOOR = 2e-3


def _local_errors(res, ref64, pts, slot, F=78):
    return {FEAT: rel_max(res[2][:, pts, F:], ref64[2][:, pts, F:]),
            H3ROW: rel_max(res[3]["encoder.h3_nodes"][slot], ref64[3]["encoder.h3_nodes"][slot])}  # fmt: skip


def _local_bars(ref32, ref64, pts, slot):
    """{region: (fp32-type bar, bf16 bar or None)}."""
    return {k: (max(10 * e + 2e-5, LOCAL_FLOOR), LOCAL_BF16[k]) for k, e in _local_errors(ref32, ref64, pts, slot).items()}


def _check_local(ours, ref32, ref64, pts, slot, tp, tag):
    bars = _local_bars(ref32, ref64, pts, slot)
    fails = []
    for k, e in _local_errors(ours, ref64, pts, slot).items():
        bar = bars[k][1 if tp == "bf16" else 0]
        print(f"  {tag} {k}: max-rel err vs fp64 {e:.2e} (bar {'none' if bar is None else f'{bar:.2e}'})")
        if bar is not None and not e < bar:
            fails.append((tag, k, e, bar))
    assert not fails, fails


def _atomic(model):
    """Parameters whose gradients the tensor-core step sums with float atomics: LayerNorms and Linear layers with <= 16 inputs."""
    names = set()
    for mname, m in model.named_modules():
        if isinstance(m, nn.LayerNorm) or (isinstance(m, nn.Linear) and m.in_features <= 16):
            names |= {f"{mname}.{k}" for k, _ in m.named_parameters(recurse=False)}
    return names


# ---- forward at 0.25 degrees -----------------------------------------------------------------------------------------------------
def test_quarter_degree_forward(quarter):
    """Batch 4, every precision, every row against the fp64 oracle: fp32_simt and fp32 within FULL_TOL, bf16 within BF16_TOL
    (measured 4.0e-3; 2.0e-3 on the polar rows, 2.9e-3 on the seam, 3.6e-3 in the dense cell).  Then the fp32-type bar against
    the faults: it sees two swapped decoder edges (measured 6.4e-5, 6.4x the bar) and a sum not carried over a chunk boundary
    (2.9e-5, 2.9x).  One row dropped from the 9 142-row sum moves the output by 4.2e-7, the size of fp32 rounding, and no fault
    of one cell reaches the bf16 bar (at most 0.003x): no end-to-end bar sees those; the exact-integer kernel tests of
    tests/test_gpu_kernels.py see a dropped or repeated row in every precision."""
    from graph_weather_b200 import GraphWeatherForecaster
    from oracle import weights

    ll, graphs, dense_pts, _ = quarter
    N = len(ll)
    sd = weights.make_state_dict(weights.forecaster_shapes(), 10)
    x = weights.make_features(4, N, 102, 10)
    lon_j = np.arange(N) % 1440
    where = {"polar rows": torch.from_numpy(np.r_[0:1440, N - 1440:N]).cuda(),
             "lon 0 / 359.75 seam": torch.from_numpy(np.flatnonzero((lon_j == 0) | (lon_j == 1439))).cuda(),
             f"the {len(dense_pts)}-point mesh cell": torch.from_numpy(dense_pts).cuda()}  # fmt: skip
    with _budget("0.25 deg forward, batch 4") as models:
        t0 = time.perf_counter()
        ref = grid_oracle.forward(sd, graphs, x, torch.float64, "cuda", CHUNK)
        print(f"fp64 oracle forward: {time.perf_counter() - t0:.1f} s")
        faults = {}
        for name, bad in _faults(graphs, dense_pts).items():  # the largest change each fault makes to the output
            faults[name] = float((grid_oracle.forward(sd, bad, x, torch.float64, "cuda", CHUNK) - ref).abs().max())
            print(f"fault '{name}': max|faulty - true| = {faults[name]:.3e} ({faults[name] / FULL_TOL:.1f}x the fp32-type bar, "
                  f"{faults[name] / BF16_TOL:.2g}x the bf16 bar)")  # fmt: skip
        xg = x.cuda()
        fails = []
        for precision, bar in (("fp32_simt", FULL_TOL), ("fp32", FULL_TOL), ("bf16", BF16_TOL)):
            model = GraphWeatherForecaster(ll, precision=precision).cuda().eval()
            model.load_state_dict(sd)
            out = model(xg)
            model._engine.plan.status()
            models.append(_model_bytes(model))
            del model
            assert out.shape == (4, N, 78)
            err = {k: 0.0 for k in ["all rows", *where]}
            for b in range(4):
                d = (out[b].double() - ref[b]).abs().amax(-1)
                err["all rows"] = max(err["all rows"], float(d.max()))
                for k, idx in where.items():
                    err[k] = max(err[k], float(d[idx].max()))
            print(f"0.25 deg [{precision}] max|gpu - fp64 oracle|: " + ", ".join(f"{k} {v:.3e}" for k, v in err.items()))
            if not err["all rows"] < bar:
                fails.append((precision, err["all rows"]))
            del out
    assert not fails, fails
    assert faults["two decoder edges of one point swapped"] > FULL_TOL
    assert faults["the dense cell's sum not carried over a chunk boundary"] > FULL_TOL


# ---- bounded training step at 0.25 degrees ------------------------------------------------------------------------------------
def _quarter_case(quarter, batch, seed):
    from oracle import weights

    ll, graphs = quarter[:2]
    sd = weights.make_state_dict(weights.forecaster_shapes(), seed)
    x = weights.make_features(batch, len(ll), 102, seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    target = torch.from_numpy(rng.standard_normal((batch, len(ll), 78)).astype(np.float32))
    var = rng.uniform(0.5, 2.0, 78).astype(np.float32).tolist()
    refs = []
    for dtype in (torch.float32, torch.float64):
        t0 = time.perf_counter()
        refs.append(grid_oracle.train_step(sd, graphs, x, target, var, ll, dtype, "cuda", CHUNK))
        print(f"0.25 deg batch {batch} {dtype} oracle step: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 1e9:.1f} GB")
    return ll, graphs, sd, x, target, var, *refs


@pytest.fixture(scope="module")
def quarter_b1(quarter):
    with _budget("0.25 deg oracle steps, batch 1"):
        return _quarter_case(quarter, 1, 31)


def _bounded_step(ll, sd, x, target, var, tp, segments=0):
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    model = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=True).cuda().train()
    model.load_state_dict(sd)
    model.processor.set_checkpoint_segments(segments)
    res = train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target)
    assert model._train_engine.plan.train_only
    return model, res


def _groups(model, ours, ref32, ref64, tag):
    """The float-atomic parameters and the ILL_CONDITIONED group, printed apart: worst max-relative error against fp64 next to
    the fp32 oracle's and worst cosine."""
    grads, g32, g64 = ours[3], ref32[3], ref64[3]
    for name, keys in (("float-atomic", sorted(_atomic(model))), ("ILL_CONDITIONED", sorted(k for k in grads if k.startswith(ILL_CONDITIONED)))):
        e = max((rel_max(grads[k], g64[k]), rel_max(g32[k], g64[k]), k) for k in keys)
        c = min((cos(grads[k], g64[k]), k) for k in keys)
        print(f"  {tag} {name} ({len(keys)} tensors): worst max-rel err vs fp64 {e[0]:.2e} on {e[2]} (fp32 oracle {e[1]:.2e}); "
              f"lowest cosine {c[0]:.5f} on {c[1]}")  # fmt: skip


@pytest.mark.training
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_quarter_degree_bounded_step(quarter, quarter_b1, tp):
    """Batch 1, the default chunk budget, against the fp64 oracle step with the 10-degree bounded step's bars
    (tests/test_gpu_lean_training.py::test_gradients_match_the_oracle).  Measured: fp32 -- features 6.4e-5 max-relative (fp32
    oracle 4.1e-5), h3_nodes 2.2e-2 (oracle 1.7e-2), the float-atomic parameters at most 5.3e-5, every other parameter below
    4e-4; bf16 -- lowest cosine 0.9932 (h3_nodes), >= 0.9993 for every other parameter, float-atomic ones included."""
    ll, graphs, sd, x, target, var, ref32, ref64 = quarter_b1
    with _budget(f"0.25 deg bounded step [{tp}]") as models:
        model, ours = _bounded_step(ll, sd, x, target, var, tp)
        models.append(_model_bytes(model))
        tag = f"0.25 deg bounded [{tp}]"
        _groups(model, ours, ref32, ref64, tag)
        _check_local(ours, ref32, ref64, *quarter[2:], tp, tag)
        if tp == "bf16":
            check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=None, tag=tag)
        else:
            check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3, feat_floor=False, median=False, ill=None, skip_zero=False,
                            norm_bar=None, tag=tag)  # fmt: skip


@pytest.mark.training
def test_gradient_bars_see_the_faults(quarter, quarter_b1):
    """The fp64 oracle step on the faulty graphs of the dense cell, held to the bars the GPU steps are held to.  The bars over whole
    gradient tensors cannot see a fault in one cell of 5 882 (printed: the largest ratio of change to bar).  Of the dense cell's
    own bars, each one, fp32-type and bf16, must see at least one fault, and the features' bars must see both -- a single dropped
    row among them.  Measured: the features change by 0.37 (one row; 1.9x the fp32-type bar, 1.2x the bf16 bar) and 1.0 (the
    sum not carried; 5.1x, 3.4x); the h3_nodes row by 4.7e-4 (one row: below the floor) and 1.0e-2 (5x the floor); no
    whole-tensor bar reaches more than 0.065x."""
    ll, graphs, sd, x, target, var, ref32, ref64 = quarter_b1
    pts, slot = quarter[2:]
    bars = _local_bars(ref32, ref64, pts, slot)
    faults = _faults(graphs, pts)
    change = {}
    for name in ("one row dropped from the dense cell's encoder sum", "the dense cell's sum not carried over a chunk boundary"):
        with _budget(f"0.25 deg fault step: {name}"):
            bad = grid_oracle.train_step(sd, faults[name], x, target, var, ll, torch.float64, "cuda", CHUNK)
        whole = max((rel_max(g, ref64[3][k]) / max(10 * rel_max(ref32[3][k], ref64[3][k]) + 2e-5, 2e-3), k) for k, g in bad[3].items())
        print(f"fault '{name}': whole-tensor gradient change / bar, largest {whole[0]:.3f} ({whole[1]})")
        change[name] = _local_errors(bad, ref64, pts, slot)
        for k, e in change[name].items():
            print(f"  {k}: change {e:.2e} = " + ", ".join(f"{e / b:.1f}x the {t} bar" for b, t in zip(bars[k], ("fp32-type", "bf16")) if b))
    fails = [(k, i) for k in bars for i in (0, 1) if bars[k][i] is not None and not max(c[k] for c in change.values()) > bars[k][i]]
    fails += [(name, FEAT) for name, c in change.items() if not c[FEAT] > max(bars[FEAT])]
    assert not fails, fails


@pytest.mark.training
def test_quarter_degree_processor_segments(quarter):
    """bf16, batch 2: the step without processor segments (S = 0) against the fp64 oracle, and S = 1 against S = 0 -- bit for
    bit except the float-atomic gradients (<= 1e-6 norm-relative), as tests/test_gpu_processor_checkpointing.py states at 10 and
    30 degrees.  Measured: S = 0 lowest cosine 0.9952 (h3_nodes); S = 1 equal bit for bit, float-atomic gradients within 5.3e-7."""
    with _budget("0.25 deg bf16 batch 2, S = 0 and S = 1") as models:
        ll, graphs, sd, x, target, var, ref32, ref64 = _quarter_case(quarter, 2, 33)
        model, s0 = _bounded_step(ll, sd, x, target, var, "bf16")
        models.append(_model_bytes(model))
        atomic = _atomic(model)
        del model
        tag = "0.25 deg bounded bf16 batch 2, S = 0"
        check_bf16_bars(s0, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=None, tag=tag)
        del ref32, ref64
        model, s1 = _bounded_step(ll, sd, x, target, var, "bf16", segments=1)
        models.append(_model_bytes(model))
    assert torch.equal(s1[0], s0[0]) and s1[1] == s0[1] and torch.equal(s1[2], s0[2])
    bad = [k for k in s0[3] if k not in atomic and not torch.equal(s1[3][k], s0[3][k])]
    worst = max((rel_norm(s1[3][k], s0[3][k]), k) for k in atomic if float(s0[3][k].norm()) > 0)
    print(f"S = 1 vs S = 0: {len(s0[3]) - len(atomic)} gradients compared bit for bit, {len(bad)} differ; float-atomic worst "
          f"norm-relative difference {worst[0]:.2e} ({worst[1]})")  # fmt: skip
    assert not bad, bad[:5]
    assert worst[0] <= ATOMIC_BAR, worst


# ---- taped training step at 1 degree ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def one_degree():
    from oracle import weights

    ll = grid(1)
    graphs = grid_oracle.build_graphs(ll)
    sd = weights.make_state_dict(weights.forecaster_shapes(), 5)
    x = weights.make_features(2, len(ll), 102, 5)
    rng = np.random.Generator(np.random.PCG64(5))
    target = torch.from_numpy(rng.standard_normal((2, len(ll), 78)).astype(np.float32))
    var = rng.uniform(0.5, 2.0, 78).astype(np.float32).tolist()
    with _budget("1 deg batch 2 oracle steps"):
        refs = [grid_oracle.train_step(sd, graphs, x, target, var, ll, dt, "cuda", CHUNK) for dt in (torch.float32, torch.float64)]
    return ll, sd, x, target, var, *refs, _dense_cell(graphs)


@pytest.mark.training
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_one_degree_taped_step(one_degree, tp):
    """Batch 2, the taped step, against the fp64 oracle step with the 10-degree bars (tests/test_gpu_training.py,
    tests/test_gpu_train_precision.py).  Measured: fp32_simt -- every gradient within 1.1x the fp32 oracle's error (h3_nodes
    1.0e-2); fp32 -- features 1.2e-4 (oracle 4.9e-5), h3_nodes 1.1e-2, every other parameter below 5e-4, float-atomic ones at
    most 7.7e-5; bf16 -- lowest cosine 0.9937 (h3_nodes), >= 0.9992 for every other parameter."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var, ref32, ref64, dense = one_degree
    with _budget(f"1 deg taped step [{tp}]") as models:
        model = GraphWeatherForecaster(ll, train_precision=tp).cuda().train()
        model.load_state_dict(sd)
        ours = train_step(model, NormalizedMSELoss(var, ll, normalize=True), x, target)
        assert not model._train_engine.plan.train_only
        models.append(_model_bytes(model))
        tag = f"1 deg taped [{tp}]"
        _groups(model, ours, ref32, ref64, tag)
        _check_local(ours, ref32, ref64, *dense, tp, tag)
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999, tag=tag)
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3 if tp == "fp32" else 0.0, feat_floor=False, median=False, ill=None,
                        skip_zero=False, norm_bar=None, tag=tag)  # fmt: skip
