"""-m gpu: model shapes beyond the reference defaults, against the fp64 / fp32 CPU oracle (oracle/restate.py).  Every other test runs
node_dim == edge_dim, equal processor hidden widths and two hidden layers per MLP, where a swapped width, a wrong column offset of
a concatenated first layer or an off-by-one in a hidden-layer loop cannot show.  The shapes:

  * mixed      the forecaster_mixed_shapes fixture's configuration: node 48 / edge 80, processor hidden 96 / 64, hidden layers
               1 (node) / 3 (edge) / 3 (decoder), decoder hidden 40, 7 + 5 input channels, 2 blocks;
  * unaligned  widths that are not multiples of four: node 37 / edge 30, processor hidden 50 / 27, decoder hidden 19, hidden
               layers 3 (node) / 1 (edge), 5 + 2 input channels, 2 blocks;
  * one_layer  64 wide, one hidden layer in every MLP, 2 blocks;
  * the node decoder variants of the tensor-core trunk (256 wide, 2 blocks) as (hidden_dim_decoder, hidden_layers_decoder,
    feature_dim): (64, 2, 78), (192, 2, 77) (an odd output), (96, 2, 78) (not a multiple of 64), (128, 1, 78), (128, 3, 78).

Per shape: inference in every precision the shape takes against restate.forecaster_forward (max-abs 1e-4 fp32 / fp32_simt, 2e-2
bf16, the bars of tests/test_gpu_parity.py), the mixed shape also against the reference's own output and per stage (standalone
Encoder / Processor / Decoder); one training step against forecaster_case's oracle -- fp32_simt taped and bounded (several
chunks) for the trunk shapes with the bars of tests/test_gpu_training.py, fp32 and bf16 for the decoder variants with those of
tests/test_gpu_train_precision.py, widened where these shapes measured beyond them (comments at each bar) -- and one SGD step that lowers the loss.  GraphCast with three hidden layers, and the
RegionalForecaster and GraphWeatherAssimilator in the mixed shape, run against their restatements (another GraphCast hidden_dim is
refused: tests/test_wrapper_training_config.py).  The row movement of the training step (launch_segsum, launch_gather_rows) is
checked bit for bit at widths 1 .. 64, dense and odd strides, aligned and unaligned base pointers.

Each case prints its worst error next to its bar.  Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit:
  * inference max-abs against the oracle: trunk shapes 2.4e-7 .. 3.6e-7 (fp32_simt); decoder variants 4.8e-7 .. 7.2e-7
    (fp32_simt), 4.8e-7 .. 1.2e-6 (fp32), 7.4e-4 .. 5.6e-3 (bf16); mixed against the reference 2.4e-7, per stage 1.4e-6 /
    1.9e-6 / 2.4e-7; GraphCast 2.4e-7, regional 9.5e-7, assimilator 7.5e-8;
  * fp32_simt training, taped and bounded alike: features 1.2e-7 .. 1.6e-7 max-relative error against fp64, median parameter
    error 2.4e-7 .. 4.1e-7 (the fp32 oracle's 1.6e-7 .. 3.8e-7); the training bars' comments give the rest.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
from training_oracle import check_bf16_bars, check_fp32_bars, forecaster_case, grid, train_step

pytestmark = pytest.mark.gpu
TOL, BF16_TOL = 1e-4, 2e-2  # tests/test_gpu_parity.py

MIXED = dict(node_dim=48, edge_dim=80, hidden_dim_processor_node=96, hidden_dim_processor_edge=64, hidden_layers_processor_node=1,
             hidden_layers_processor_edge=3, hidden_dim_decoder=40, hidden_layers_decoder=3, feature_dim=7, aux_dim=5, num_blocks=2)
TRUNK = {
    "mixed": MIXED,
    "unaligned": dict(node_dim=37, edge_dim=30, hidden_dim_processor_node=50, hidden_dim_processor_edge=27, hidden_layers_processor_node=3,
                      hidden_layers_processor_edge=1, hidden_dim_decoder=19, feature_dim=5, aux_dim=2, num_blocks=2),
    "one_layer": dict(node_dim=64, edge_dim=64, hidden_dim_processor_node=64, hidden_dim_processor_edge=64, hidden_dim_decoder=64,
                      hidden_layers_processor_node=1, hidden_layers_processor_edge=1, hidden_layers_decoder=1, feature_dim=10, aux_dim=4,
                      num_blocks=2),
}  # fmt: skip
DECODER = {f"dec_{h}x{n}_f{f}": dict(hidden_dim_decoder=h, hidden_layers_decoder=n, feature_dim=f, num_blocks=2)
           for h, n, f in [(64, 2, 78), (192, 2, 77), (96, 2, 78), (128, 1, 78), (128, 3, 78)]}  # fmt: skip
SHAPES = {**TRUNK, **DECODER}


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _hl(kw):
    """restate's hidden-layer arguments of a forecaster configuration."""
    return dict(hl_node=kw.get("hidden_layers_processor_node", 2), hl_edge=kw.get("hidden_layers_processor_edge", 2),
                hl_dec=kw.get("hidden_layers_decoder", 2))  # fmt: skip


def _case(name):
    """The 10-degree, batch-2 case of a shape and its oracle step (fp32 and fp64), seed 21 as in tests/test_gpu_training.py."""
    return forecaster_case(10, 2, 21, **SHAPES[name])


def _n_params(kw):
    from oracle import weights

    return len(weights.forecaster_shapes(**kw))


def _forecaster(ll, sd, kw, **model_kw):
    from graph_weather_b200 import GraphWeatherForecaster

    model = GraphWeatherForecaster(ll, **kw, **model_kw).cuda()
    model.load_state_dict(sd)
    return model


def _max_abs(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


# ---- inference --------------------------------------------------------------------------------------------------------------
INFER = [(n, p) for n in TRUNK for p in ["fp32_simt"]] + [(n, p) for n in DECODER for p in ["fp32_simt", "fp32", "bf16"]]


@pytest.mark.parametrize("name,precision", INFER)
def test_inference_matches_the_oracle(name, precision):
    from oracle import restate

    from oracle import weights

    kw = SHAPES[name]
    ll = grid(10)  # (forecaster_case's weights and features, without its oracle step)
    sd = weights.make_state_dict(weights.forecaster_shapes(**kw), 21)
    x = weights.make_features(2, len(ll), kw["feature_dim"] + kw.get("aux_dim", 24), 21)
    model = _forecaster(ll, sd, kw, precision=precision).eval()
    with torch.no_grad():
        out = model(x.cuda())
    assert model._engine.resolved_precision == precision
    ref = restate.forecaster_forward(sd, restate.build_forecaster_graphs(ll), x, feature_dim=kw["feature_dim"], num_blocks=kw["num_blocks"],
                                     **_hl(kw))  # fmt: skip
    assert out.shape == ref.shape
    err, bar = _max_abs(out, ref), BF16_TOL if precision == "bf16" else TOL
    print(f"{name} [{precision}] max|gpu - oracle| = {err:.3e} (bar {bar:.0e})")
    assert err < bar


def _fixture(golden_dir):
    from oracle import weights

    z = np.load(os.path.join(golden_dir, "forecaster_mixed_shapes.npz"))
    cfg = json.loads(str(z["config"]))
    assert cfg["kw"] == MIXED
    ll = grid(cfg["step"])
    sd = weights.make_state_dict(weights.forecaster_shapes(**MIXED), cfg["seed"])
    x = weights.make_features(cfg["batch"], len(ll), MIXED["feature_dim"] + MIXED["aux_dim"], cfg["seed"])
    return z, ll, sd, x


def test_mixed_shape_matches_the_reference_fixture(golden_dir):
    z, ll, sd, x = _fixture(golden_dir)
    model = _forecaster(ll, sd, MIXED, precision="fp32_simt").eval()
    with torch.no_grad():
        out = model(x.cuda()).cpu().numpy()
    assert out.shape == z["out"].shape
    err = float(np.abs(out - z["out"]).max())
    print(f"mixed [fp32_simt] max|gpu - reference| = {err:.3e} (bar {TOL:.0e})")
    assert err < TOL


def test_mixed_shape_stage_api_matches_the_reference_fixture(golden_dir):
    """Encoder -> Processor -> Decoder built on their own with the mixed shape's arguments, checked per stage."""
    from graph_weather_b200 import Decoder, Encoder, Processor

    z, ll, sd, x = _fixture(golden_dir)
    m = MIXED
    common = dict(hidden_dim_processor_node=m["hidden_dim_processor_node"], hidden_dim_processor_edge=m["hidden_dim_processor_edge"],
                  hidden_layers_processor_node=m["hidden_layers_processor_node"],
                  hidden_layers_processor_edge=m["hidden_layers_processor_edge"], precision="fp32_simt")  # fmt: skip
    enc = Encoder(ll, input_dim=m["feature_dim"] + m["aux_dim"], output_dim=m["node_dim"], output_edge_dim=m["edge_dim"], **common).cuda()
    proc = Processor(input_dim=m["node_dim"], edge_dim=m["edge_dim"], num_blocks=m["num_blocks"], **common).cuda()
    dec = Decoder(ll, input_dim=m["node_dim"], output_dim=m["feature_dim"], output_edge_dim=m["edge_dim"], hidden_dim_decoder=m["hidden_dim_decoder"],
                  hidden_layers_decoder=m["hidden_layers_decoder"], **common).cuda()  # fmt: skip
    for name, stage in (("encoder", enc), ("processor", proc), ("decoder", dec)):
        stage.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")})
    xg = x.cuda()
    with torch.no_grad():
        ex, ei, ea = enc(xg)
        assert ex.shape == (5882 * 2, 48) and ea.shape == (41162 * 2, 80)
        px = proc(ex, ei, ea)
        out = dec(px, xg[..., : m["feature_dim"]])
    errs = dict(encoder=float(np.abs(ex.cpu().numpy()[::53] - z["enc_x_sub"]).max()),
                processor=float(np.abs(px.cpu().numpy()[::53] - z["proc_x_sub"]).max()),
                decoder=float(np.abs(out.cpu().numpy() - z["out"]).max()))  # fmt: skip
    print(f"mixed stage API max|gpu - reference|: {errs} (bar {TOL:.0e})")
    assert all(e < TOL for e in errs.values()), errs


# ---- training ---------------------------------------------------------------------------------------------------------------
def _inference_loss(model, crit, x, target):
    model.eval()
    with torch.no_grad():
        loss = float(crit(model(x.cuda()), target.cuda()))
    model.train()
    return loss


def _sgd_lowers_the_loss(model, crit, x, target):
    """One SGD step (lr 0.1) on the gradients of the training step just taken lowers the loss, evaluated by inference before and
    after (an fp32-faithful forward in every precision: the decrease is ~1e-4 relative on some shapes, below a bf16 forward's
    error).  lr 0.1 lowers the fp32 oracle's loss on every shape here; lr 1e-2 does too, but by as little as 1e-5."""
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in model.parameters())
    loss0 = _inference_loss(model, crit, x, target)
    torch.optim.SGD(model.parameters(), lr=0.1).step()
    loss1 = _inference_loss(model, crit, x, target)
    print(f"  loss {loss0:.6f} -> {loss1:.6f} after one SGD step")
    assert loss1 < loss0


# tests/test_gpu_training.py's bar (no floor), except where a ReLU unit sits at the edge of its mask: five layer-0 pre-activations
# of the mixed shape's processor block 1 edge MLP are within 1e-6 of zero in fp64 (the smallest 1.6e-7), so an fp32 step may switch
# one.  Measured on an H100 (700 W): 7.8e-5 / 7.4e-5 max-relative error on that layer's bias / weight (fp32 oracle 8.9e-8 / 1.0e-7),
# taped and bounded alike; every other parameter of every trunk shape within 10x the fp32 oracle's error + 2e-5.
TRUNK_FLOOR = {"mixed": 2e-4, "unaligned": 0.0, "one_layer": 0.0}


@pytest.mark.training
@pytest.mark.parametrize("step", ["taped", "bounded"])
@pytest.mark.parametrize("name", list(TRUNK))
def test_trunk_shapes_train_like_the_oracle(monkeypatch, name, step):
    """fp32_simt, the taped step and the bounded one (37-point chunks: 18 decoder chunks on the 648-point grid)."""
    from graph_weather_b200 import NormalizedMSELoss

    kw = SHAPES[name]
    ll, sd, x, target, var, ref32, ref64 = _case(name)
    if step == "bounded":
        monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")  # (read at plan creation)
    model = _forecaster(ll, sd, kw, use_checkpointing=step == "bounded").train()
    crit = NormalizedMSELoss(var, ll, normalize=True)
    ours = train_step(model, crit, x, target)
    assert model._train_engine.plan.train_only == (step == "bounded")
    check_fp32_bars(ours, ref32, ref64, n_params=_n_params(kw), floor=TRUNK_FLOOR[name], feat_floor=False, median=True, ill=None,
                    skip_zero=False, norm_bar=None, tag=f"{name} fp32_simt {step}")  # fmt: skip
    _sgd_lowers_the_loss(model, crit, x, target)


@pytest.mark.training
@pytest.mark.parametrize("tp", ["fp32", "bf16"])
@pytest.mark.parametrize("name", list(DECODER))
def test_decoder_variants_train_like_the_oracle(name, tp):
    from graph_weather_b200 import NormalizedMSELoss

    kw = SHAPES[name]
    ll, sd, x, target, var, ref32, ref64 = _case(name)
    model = _forecaster(ll, sd, kw, train_precision=tp).train()
    crit = NormalizedMSELoss(var, ll, normalize=True)
    ours = train_step(model, crit, x, target)
    assert model._train_engine.resolved_precision == tp
    # Bars.  tests/test_gpu_train_precision.py's (fp32: floor 2e-3; bf16: cosine 0.99 / 0.98, all parameters 0.999), widened where
    # these shapes measured beyond them on an H100 (700 W) -- the 2-block trunk spreads the encoder's ill-conditioned gradients
    # further than the 9-block default does, and the deeper decoders add layers:
    #   fp32: features 3.2e-5 .. 5.7e-5 max-relative error (fp32 oracle 2.8e-7 .. 2.1e-6); the encoder's edge encoder and block
    #     edge MLP up to 5.4e-3 (fp32 oracle <= 1.1e-4); (128, 3) one decoder node-MLP unit switches its ReLU: 5.1e-3 on
    #     node_decoder.model.2 (fp32 oracle 3.0e-7), as tests/test_gpu_graphcast_training.py measures on GraphCast's decoder.
    #     Floor 8e-3, the features' gradient included: a 1 % error in one gradient still fails it (tests/test_training_oracle.py).
    #   bf16: (128, 3) gives cosines 0.984 (h3_nodes), 0.986 (encoder.edge_encoder.model.0), 0.989 (processor block 1 edge MLP
    #     layer 0) and 0.9966 over all parameters; the other variants >= 0.9868 / 0.9956 / 0.998.
    if tp == "bf16":
        check_bf16_bars(ours, ref32, ref64, n_params=_n_params(kw), cos_bar=0.98, ill_cos_bar=0.975, feat_cos=None, total_cos=0.995,
                        tag=f"{name} bf16")  # fmt: skip
    else:
        check_fp32_bars(ours, ref32, ref64, n_params=_n_params(kw), floor=8e-3, feat_floor=True, median=False, ill=None, skip_zero=False,
                        norm_bar=None, tag=f"{name} fp32")  # fmt: skip
    _sgd_lowers_the_loss(model, crit, x, target)


# ---- the wrappers -----------------------------------------------------------------------------------------------------------
GRAPHCAST = dict(feature_dim=78, aux_dim=0, hidden_dim_decoder=256, hidden_layers_processor_node=3, hidden_layers_processor_edge=3,
                 hidden_layers_decoder=3, num_blocks=2)  # fmt: skip


@pytest.mark.training
def test_graphcast_three_hidden_layers():
    """GraphCast(hidden_layers=3, num_processor_blocks=2): its node decoder gets hidden_dim and hidden_layers too (256 x 3).
    Inference against the restatement, one fp32_simt training step against the oracle with tests/test_gpu_training.py's bars.
    (Another hidden_dim leaves the reference's decoder with 256-wide edges and the rest of the network with hidden_dim-wide ones,
    which the plan's single edge width cannot hold: tests/test_wrapper_training_config.py checks that it is refused.)"""
    from graph_weather_b200 import GraphCast, NormalizedMSELoss
    from oracle import restate

    ll, sd, x, target, var, ref32, ref64 = forecaster_case(10, 2, 21, **GRAPHCAST)
    model = GraphCast(ll, hidden_layers=3, num_processor_blocks=2).cuda()
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        out = model(x.cuda())
    ref = restate.forecaster_forward(sd, restate.build_forecaster_graphs(ll), x, feature_dim=78, num_blocks=2, **_hl(GRAPHCAST))
    err = _max_abs(out, ref)
    print(f"graphcast 3 hidden layers [{model._engine.resolved_precision}] max|gpu - oracle| = {err:.3e} (bar {TOL:.0e})")
    assert err < TOL
    model.train()
    crit = NormalizedMSELoss(var, ll, normalize=True)
    ours = train_step(model, crit, x, target)
    check_fp32_bars(ours, ref32, ref64, n_params=_n_params(GRAPHCAST), floor=0.0, feat_floor=False, median=True, ill=None,
                    skip_zero=False, norm_bar=None, tag="graphcast 3 hidden layers fp32_simt")  # fmt: skip
    _sgd_lowers_the_loss(model, crit, x, target)


def _mixed_kw():
    """MIXED as keyword arguments of the wrappers that have no feature_dim / aux_dim."""
    return {k: v for k, v in MIXED.items() if k not in ("feature_dim", "aux_dim")}


def test_regional_forecaster_mixed_shape():
    from graph_weather_b200.regional import RegionalForecasterConfig
    from oracle import restate, weights

    ll = [(38.0 + 0.5 * i, -12.0 + 0.5 * j) for i in range(20) for j in range(31)] + [(58.1, 10.9), (63.0, -20.0)]
    model = RegionalForecasterConfig(feature_dim=7, aux_dim=5, **_mixed_kw()).build().cuda().eval()
    sd = weights.make_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, 23)
    model.load_state_dict(sd)
    x = weights.make_features(2, len(ll), 12, 23)
    with torch.no_grad():
        out = model(x.cuda(), ll)
    ref = restate.regional_forward(sd, restate.regional_graphs(ll), x, output_dim=7, num_blocks=2, **_hl(MIXED))
    assert out.shape == ref.shape == (2, len(ll), 7)
    err = _max_abs(out, ref)
    print(f"regional mixed [auto] max|gpu - oracle| = {err:.3e} (bar {TOL:.0e})")
    assert err < TOL


def test_assimilator_mixed_shape():
    from graph_weather_b200 import GraphWeatherAssimilator
    from oracle import restate, weights

    out_ll = grid(10)
    model = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=7, **_mixed_kw()).cuda().eval()
    sd = weights.make_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, 24)
    model.load_state_dict(sd)
    rng = np.random.Generator(np.random.PCG64(24))
    obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, 500), rng.uniform(0, 360, 500), rng.uniform(0, 1, 500)], 1).astype(np.float32))
    x = weights.make_features(2, obs.shape[0], 2, 24)
    with torch.no_grad():
        out = model(x.cuda(), obs.cuda())
    assert out.shape == (2, len(out_ll), 7)
    # one sample at a time: the reference offsets sample i of its replicated observation graph by i * max(edge_index) + i
    # (assimilator_encoder.py:148), which is the node count only when the highest cell id receives an observation
    g = restate.build_assimilator_graphs(out_ll)
    err = max(_max_abs(out[b : b + 1], restate.assimilator_forward(sd, g, x[b : b + 1], obs, num_blocks=2, **_hl(MIXED))) for b in range(2))
    print(f"assimilator mixed [auto] max|gpu - oracle| = {err:.3e} (bar {TOL:.0e})")
    assert err < TOL


# ---- row movement at any width ----------------------------------------------------------------------------------------------
WIDTHS = [1, 2, 3, 27, 30, 37, 50, 64]
# (ld of the rows read, ld of the rows written, elements the base pointers are moved by): dense rows; odd strides; 4-aligned strides
# behind base pointers one float off a 16-byte boundary (float4 could address the strides but not the rows)
LAYOUTS = {"dense": (0, 0, 0), "odd_ld": (3, 5, 0), "offset_base": (4, 8, 1)}


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)

    tk.HK = tk._compile_harness(tmp_path_factory.mktemp("gw_shape_harness"))
    return tk.HK


def _layout(width, layout):
    pad_in, pad_out, off = LAYOUTS[layout]
    return width + pad_in, width + pad_out, off


def _at(t, elems):
    return ctypes.c_void_p(t.data_ptr() + t.element_size() * elems)


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("width", WIDTHS)
def test_segsum_any_width(hk, width, layout, accumulate):
    """launch_segsum (through h_segsum_range: a CSR slice with ptr_base, optionally adding to out) with a permutation, empty and
    700-row segments, three samples: each segment's sum is the sequential float32 sum of its rows, added to the previous value
    of out when accumulating; columns >= width and rows past the output keep their bits."""
    from test_gpu_kernels import _csr, _ok, _p, _seq_sum, _st

    rng = np.random.Generator(np.random.PCG64(100 * width + 7 * list(LAYOUTS).index(layout) + accumulate))
    lengths = rng.integers(0, 9, 60)
    lengths[[5, 6, 40]] = 0
    lengths[20] = 700
    ptr = _csr(lengths)
    s0, s1 = 3, 55
    r0, r1 = int(ptr[s0]), int(ptr[s1])
    n, ns, B = r1 - r0, s1 - s0, 3
    ld, ldo, off = _layout(width, layout)
    base = rng.standard_normal((B * n, ld)).astype(np.float32)
    perm = rng.permutation(n).astype(np.int32)
    out0 = rng.standard_normal((B * ns + 1, ldo)).astype(np.float32)
    out0[:, width:] = np.nan
    if not accumulate:
        out0[::3, :width] = np.nan
    tb = torch.from_numpy(np.concatenate([np.zeros(off, np.float32), base.ravel()])).cuda()
    tout = torch.from_numpy(np.concatenate([np.zeros(off, np.float32), out0.ravel()])).cuda()
    tp, tperm = torch.from_numpy(ptr).cuda(), torch.from_numpy(perm).cuda()
    _ok(hk.h_segsum_range(_at(tb, off), ld, width, _at(tp, s0), _p(tperm), n, ns, B, _at(tout, off), ldo, r0, int(accumulate), _st()))
    torch.cuda.synchronize()
    want = out0.copy()
    for b in range(B):
        for i in range(ns):
            j = perm[np.arange(ptr[s0 + i], ptr[s0 + i + 1]) - r0]
            part = _seq_sum(base[b * n + j, :width])
            want[b * ns + i, :width] = out0[b * ns + i, :width] + part if accumulate else part
    got = tout.cpu().numpy()[off:].reshape(B * ns + 1, ldo)
    bad = _bits(got) != _bits(want)
    assert not bad.any(), f"segsum width {width} {layout}: {int(bad.sum())} floats differ, first at {np.argwhere(bad)[0].tolist()}"
    if layout == "dense" and not accumulate:  # the plain entry point (ptr_base 0, no accumulate) on the whole table
        tfull = torch.full((B * len(lengths), width), float("nan"), device="cuda")
        full_base = torch.from_numpy(rng.standard_normal((B * int(ptr[-1]), width)).astype(np.float32)).cuda()
        _ok(hk.h_segsum(_p(full_base), width, width, _p(tp), None, int(ptr[-1]), len(lengths), B, _p(tfull), width, _st()))
        torch.cuda.synchronize()
        fb = full_base.cpu().numpy()
        E = int(ptr[-1])
        want_full = np.stack([_seq_sum(fb[b * E + ptr[i]: b * E + ptr[i + 1]]) for b in range(B) for i in range(len(lengths))])
        assert np.array_equal(_bits(tfull.cpu().numpy()), _bits(want_full)), f"h_segsum width {width}"


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("width", WIDTHS)
def test_gather_rows_any_width(hk, width, layout, accumulate):
    """launch_gather_rows (through h_gather_rows_base: a table holding targets r0 .. r0 + n - 1) over three samples and enough
    rows for several grid-stride passes at the narrow widths: out = (out +) the target's row, bit for bit; columns >= width keep
    their bits."""
    from test_gpu_kernels import _ok, _p, _st

    rng = np.random.Generator(np.random.PCG64(200 * width + 7 * list(LAYOUTS).index(layout) + accumulate))
    n_pts, r0, n, B = 4000, 911, 1500, 3
    ld_in, ld_out, off = _layout(width, layout)
    dst = np.sort(rng.integers(0, n_pts, 12000)).astype(np.int32)
    e0, e1 = int(np.searchsorted(dst, r0)), int(np.searchsorted(dst, r0 + n))
    ne = e1 - e0
    table = rng.standard_normal((B * n, ld_in)).astype(np.float32)
    out0 = rng.standard_normal((B * ne, ld_out)).astype(np.float32)
    out0[:, width:] = np.nan
    tt = torch.from_numpy(np.concatenate([np.zeros(off, np.float32), table.ravel()])).cuda()
    tout = torch.from_numpy(np.concatenate([np.zeros(off, np.float32), out0.ravel()])).cuda()
    td = torch.from_numpy(dst).cuda()
    _ok(hk.h_gather_rows_base(_at(tt, off), ld_in, n, _at(td, e0), ne, width, B, _at(tout, off), ld_out, int(accumulate), r0, _st()))
    torch.cuda.synchronize()
    rows = (np.arange(B)[:, None] * n + (dst[e0:e1] - r0)[None, :]).reshape(-1)
    want = out0.copy()
    want[:, :width] = out0[:, :width] + table[rows, :width] if accumulate else table[rows, :width]
    got = tout.cpu().numpy()[off:].reshape(B * ne, ld_out)
    bad = _bits(got) != _bits(want)
    assert not bad.any(), f"gather_rows width {width} {layout}: {int(bad.sum())} floats differ, first at {np.argwhere(bad)[0].tolist()}"
    if layout == "dense":  # the plain entry point (idx_base 0)
        src_rows = 300
        idx = rng.integers(0, src_rows, 2000).astype(np.int32)
        tin = torch.from_numpy(rng.standard_normal((B * src_rows, width)).astype(np.float32)).cuda()
        g0 = rng.standard_normal((B * 2000, width)).astype(np.float32)
        gout, tidx = torch.from_numpy(g0).cuda(), torch.from_numpy(idx).cuda()
        _ok(hk.h_gather_rows(_p(tin), width, src_rows, _p(tidx), 2000, width, B, _p(gout), width, int(accumulate), _st()))
        torch.cuda.synchronize()
        src = tin.cpu().numpy()[(np.arange(B)[:, None] * src_rows + idx[None, :]).reshape(-1)]
        assert np.array_equal(_bits(gout.cpu().numpy()), _bits(g0 + src if accumulate else src)), f"h_gather_rows width {width}"
