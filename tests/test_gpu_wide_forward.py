"""-m gpu: the tensor-core forward of trunks wider than 256 (precision "fp32" | "bf16" on a layer-by-layer plan): every row op of
the forward runs as tensor-core column blocks of at most 256 outputs, and a LayerNorm over more than 256 columns -- or one whose
bound the next layer needs -- is finished by gw_ln_rows_kernel, which also writes that bound (max |out|).

Kernels, one row op at a time through tests/kernels/gw_wide_forward_harness.cu (gw::run_op on a layer-by-layer plan), against
float64: LayerNorm'd row ops of N in {257, 512, 597, 1024} outputs, K in {300, 1024}, with and without a residual, and one whose
operand is assembled from two sources of 300 and 256 columns; in fp32 and bf16.  On exact-integer data the value entering the
LayerNorm equals float64 bit for bit, the LayerNorm'd rows equal the CUDA-core path's bit for bit (the same values through the
same kernel), and both are within 1e-5 of float64; on random data the rows are within the row-op bars of tests/test_gpu_kernels.py.
Every written bound equals the true max |out|.

Models: train/run.py's (605 + 40 features, node / edge / processor-hidden / decoder-hidden widths of 1024) with 2 blocks on the
10-degree grid, and a mixed trunk (node 300, edge 256, processor hidden 512 / 384, 3 / 1 hidden layers, decoder 200 wide with 3
hidden layers), against the CPU oracle (oracle/restate.py): the forecast, the additive-constrained forecast (the model's constraint layer
on the oracle's forecast), the assimilator, the RegionalForecaster, and the Encoder, Processor and Decoder alone, in fp32
(1e-4, the bar of tests/test_gpu_parity.py) and bf16 (2e-2, see BF16_LN_TOL).  Also: resolved precisions; bit-repeatable calls and
rollouts; refusal of non-finite features and weights with a clean next call; a call on a non-default stream; and the refusal of
the fused multi-GPU boundary store."""
import ctypes
import os
import subprocess

import pytest
import torch

import __graft_entry__ as ge
import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import BARS, Data, RowOp, bcast, stream
from training_oracle import grid

pytestmark = pytest.mark.gpu
TOL, BF16_TOL = 1e-4, 2e-2  # tests/test_gpu_parity.py
# bf16 outputs that leave a 1024-wide LayerNorm unchanged (the Encoder's and Processor's latent rows, the RegionalForecaster's
# LayerNorm'd node decoder): rows of unit variance after 1024-term bf16 products measured 4.0e-2 / 4.1e-2 / 4.8e-2 against the
# oracle (Encoder / Processor / RegionalForecaster) on one NVIDIA H100 80GB HBM3 at 700 W, a few % of their magnitude: bf16's own
# rounding accumulated over K = 1024.  The forecast itself (the decoder's residual output) stays within 2e-2 (measured 3.2e-3).
BF16_LN_TOL = 6e-2
BIT3 = "a magnitude bound is not finite"  # _capi.Plan.status' text for status bit 3

WIDE = dict(node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024, hidden_dim_decoder=1024,
            feature_dim=605, aux_dim=40, num_blocks=2)  # fmt: skip
MIXED_WIDE = dict(node_dim=300, edge_dim=256, hidden_dim_processor_node=512, hidden_dim_processor_edge=384, hidden_layers_processor_node=3,
                  hidden_layers_processor_edge=1, hidden_dim_decoder=200, hidden_layers_decoder=3, feature_dim=77, aux_dim=24,
                  num_blocks=2)  # fmt: skip
SHAPES = {"run_py": WIDE, "mixed": MIXED_WIDE}
SEED = 31


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _bar(prec, ln_rows=False):
    return (BF16_LN_TOL if ln_rows else BF16_TOL) if prec == "bf16" else TOL


def _max_abs(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def _hl(kw):
    """restate's hidden-layer arguments of a forecaster configuration."""
    return dict(hl_node=kw.get("hidden_layers_processor_node", 2), hl_edge=kw.get("hidden_layers_processor_edge", 2),
                hl_dec=kw.get("hidden_layers_decoder", 2))  # fmt: skip


def _case(shape="run_py"):
    from oracle import weights

    kw = SHAPES[shape]
    ll = grid(10)
    sd = weights.make_state_dict(weights.forecaster_shapes(**kw), SEED)
    x = weights.make_features(2, len(ll), kw["feature_dim"] + kw["aux_dim"], SEED)
    return ll, sd, x


def _forecaster(prec, shape="run_py", sd=None, **kw):
    from graph_weather_b200 import GraphWeatherForecaster

    ll, sd0, _ = _case(shape)
    m = GraphWeatherForecaster(ll, **SHAPES[shape], precision=prec, **kw).cuda()
    m.load_state_dict(sd0 if sd is None else sd, strict=False)
    return m.eval()


def _oracle_forecast(shape="run_py"):
    from oracle import restate

    ll, sd, x = _case(shape)
    kw = SHAPES[shape]
    return restate.forecaster_forward(sd, restate.build_forecaster_graphs(ll), x, feature_dim=kw["feature_dim"], num_blocks=kw["num_blocks"],
                                      **_hl(kw))  # fmt: skip


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_forecaster_matches_the_oracle(prec, shape):
    x = _case(shape)[2]
    model = _forecaster(prec, shape)
    with torch.no_grad():
        out = model(x.cuda())
    assert model._engine.resolved_precision == prec
    ref = _oracle_forecast(shape)
    assert out.shape == ref.shape
    err = _max_abs(out, ref)
    print(f"{shape} forecaster [{prec}] max|gpu - oracle| = {err:.3e} (bar {_bar(prec):.0e})")
    assert err < _bar(prec)


def test_auto_still_resolves_to_simt():
    model = _forecaster("auto")
    with torch.no_grad():
        model(_case()[2].cuda())
    assert model._engine.resolved_precision == "fp32_simt"


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_constrained_forecaster_matches_the_oracle(prec):
    """The oracle of a constrained forecast: the model's constraint layer (checked against the reference by
    tests/test_gpu_constraints_rollout.py) applied to the oracle's forecast and the same input."""
    x = _case()[2]
    model = _forecaster(prec, constraint_type="additive")
    with torch.no_grad():
        got = model(x.cuda())
        want = model._constrain(_oracle_forecast().cuda().float(), x.cuda())
    err = _max_abs(got, want)
    print(f"run_py additive-constrained [{prec}] max|gpu - oracle| = {err:.3e} (bar {_bar(prec):.0e})")
    assert err < _bar(prec)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_stages_alone_match_the_oracle(prec):
    """The forecaster's Encoder, Processor and Decoder called one by one, each against restate's stage on the same input (the
    Processor and the Decoder get the GPU's previous stage's output on both sides)."""
    from oracle import restate

    ll, sd, x = _case()
    g = restate.build_forecaster_graphs(ll)
    B, F = x.shape[0], WIDE["feature_dim"]
    tc = _forecaster(prec)
    with torch.no_grad():
        xh, ei, ea = tc.encoder(x.cuda())
        ref = restate.encoder_forward(sd, g, x)[0]
        err = _max_abs(xh.reshape(ref.shape), ref)
        print(f"run_py Encoder [{prec}] max|gpu - oracle| = {err:.3e}")
        assert err < _bar(prec, ln_rows=True)
        px = tc.processor(xh, ei, ea)
        ref = restate.processor_forward(sd, xh.cpu(), ei.cpu(), ea.cpu(), WIDE["num_blocks"])
        err = _max_abs(px.reshape(ref.shape), ref)
        print(f"run_py Processor [{prec}] max|gpu - oracle| = {err:.3e}")
        assert err < _bar(prec, ln_rows=True)
        start = x[..., :F]
        out = tc.decoder(px, start.cuda())
        ref = restate.assimilator_decoder_forward(sd, g, px.cpu(), B) + start
        err = _max_abs(out.reshape(ref.shape), ref)
        print(f"run_py Decoder [{prec}] max|gpu - oracle| = {err:.3e}")
        assert err < _bar(prec)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_assimilator_matches_the_oracle(prec):
    import numpy as np

    from oracle import restate, weights

    from graph_weather_b200 import GraphWeatherAssimilator

    out_ll = grid(10)
    kw = dict(node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024, num_blocks=2)
    model = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=24, precision=prec, **kw).cuda().eval()
    sd = weights.make_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, SEED)
    model.load_state_dict(sd)
    rng = np.random.Generator(np.random.PCG64(SEED))
    obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, 400), rng.uniform(0, 360, 400), rng.uniform(0, 1, 400)], 1).astype(np.float32))
    x = weights.make_features(1, obs.shape[0], 2, SEED)
    with torch.no_grad():
        out = model(x.cuda(), obs.cuda())
    ref = restate.assimilator_forward(sd, restate.build_assimilator_graphs(out_ll), x, obs, num_blocks=2)
    err = _max_abs(out, ref)
    print(f"1024-wide assimilator [{prec}] max|gpu - oracle| = {err:.3e} (bar {_bar(prec):.0e})")
    assert err < _bar(prec)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_regional_matches_the_oracle(prec):
    from oracle import restate, weights

    from graph_weather_b200.regional import RegionalForecasterConfig

    ll = [(38.0 + 0.5 * i, -12.0 + 0.5 * j) for i in range(20) for j in range(31)] + [(58.1, 10.9), (63.0, -20.0)]
    kw = dict(num_blocks=2, node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024,
              hidden_dim_decoder=1024, feature_dim=7, aux_dim=5)  # fmt: skip
    model = RegionalForecasterConfig(precision=prec, **kw).build().cuda().eval()
    sd = weights.make_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, SEED)
    model.load_state_dict(sd)
    x = weights.make_features(2, len(ll), 12, SEED)
    with torch.no_grad():
        out = model(x.cuda(), ll)
    ref = restate.regional_forward(sd, restate.regional_graphs(ll), x, output_dim=7, num_blocks=2)
    err = _max_abs(out, ref)
    print(f"1024-wide regional [{prec}] max|gpu - oracle| = {err:.3e} (bar {_bar(prec, ln_rows=True):.0e})")
    assert err < _bar(prec, ln_rows=True)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_repeatable_and_rollout_equals_the_manual_loop(prec):
    x = _case()[2].cuda()
    model = _forecaster(prec)
    with torch.no_grad():
        a, b = model(x), model(x)
        assert torch.equal(_bits(a), _bits(b)), "two identical calls differ"
        roll = model.rollout(x, 3)
        cur, manual = x, []
        for _ in range(3):
            y = model(cur)
            manual.append(y)
            cur = torch.cat([y, x[..., y.shape[-1]:]], dim=-1)
    got = roll if isinstance(roll, torch.Tensor) else torch.stack(list(roll))
    want = torch.stack(manual).reshape(got.shape)
    assert torch.equal(_bits(got), _bits(want)), "rollout differs from the manual loop"


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
def test_non_finite_features_raise_and_the_next_call_is_clean(prec, value):
    x = _case()[2].cuda()
    model = _forecaster(prec)
    bad = x.clone()
    bad[1, 5, 90] = float(value)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match=BIT3):
            model(bad)
        again = model(x)
        fresh = _forecaster(prec)(x)
    assert torch.equal(_bits(again), _bits(fresh)), "the model computes differently after a refused call"


POISONED_WEIGHT = "processor.graph_processor.blocks.1.edge_model.edge_mlp.model.2.weight"  # read in full by every path


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_non_finite_weight_raises_and_clean_weights_compute_as_fresh(prec, value):
    """One non-finite entry in a processor edge-MLP weight: the first call after the upload (which packs the weight images)
    raises the error of status bit 3; after reloading the clean weights the model computes what a fresh one does."""
    _, sd, x = _case()
    x = x.cuda()
    bad = {k: v.clone() for k, v in sd.items()}
    bad[POISONED_WEIGHT][7, 11] = float(value)
    model = _forecaster(prec, sd=bad)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match=BIT3):
            model(x)
        model.load_state_dict(sd, strict=False)
        again = model(x)
        fresh = _forecaster(prec)(x)
    assert torch.equal(_bits(again), _bits(fresh)), "the model computes differently after a refused call"


def test_non_default_stream():
    x = _case()[2].cuda()
    model = _forecaster("fp32")
    with torch.no_grad():
        want = model(x)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            got = model(x)
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want))


def test_forward_into_with_peers_raises():
    x = _case()[2].cuda()
    model = _forecaster("fp32")
    out = torch.empty(x.shape[0], x.shape[1], WIDE["feature_dim"], device="cuda")
    with torch.no_grad():
        model.forward_into(x, out)  # without peers: the plain forward
        with pytest.raises(Exception, match="256-wide trunk"):
            model.forward_into(x, out, peers=(2, [0]))


# ---- one row op of a layer-by-layer plan, against float64 ------------------------------------------------------------------------
WIDE_HARNESS = os.path.join(tk.ROOT, "tests", "kernels", "gw_wide_forward_harness.cu")
SIMT, FP32, BF16 = tk.SIMT, tk.FP32, tk.BF16


def compile_wide_harness(out_dir):
    """Builds the package, then gw_wide_forward_harness.cu against its libgwb200.so (undefined symbols are link errors)."""
    ge.build()
    so = os.path.join(str(out_dir), "libgwwideharness.so")
    cmd = [ge.NVCC, "-shared", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", WIDE_HARNESS, "-o", so,
           "-L" + tk.PKG, "-lgwb200", "-lcudart", "-Xlinker", "-rpath," + tk.PKG, "-Xlinker", "--no-undefined"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"harness build failed:\n{r.stdout}{r.stderr}"
    lib = ctypes.CDLL(so)
    lib.h_sizeof_op.restype, lib.h_sizeof_op.argtypes = ctypes.c_int, []
    lib.h_layered_row_op.restype = ctypes.c_int
    lib.h_layered_row_op.argtypes = [ctypes.c_int, ctypes.POINTER(tk.HOp), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def wh(tmp_path_factory):
    return compile_wide_harness(tmp_path_factory.mktemp("gw_wide_forward_harness"))


def _run(wh, prec, op):
    """op (a test_gpu_kernels.RowOp) through h_layered_row_op: (out [R, ldo], the written bound or None)."""
    R = op.rows * op.batch
    out = torch.full((R, op.ldo), float("nan"), device="cuda")
    h = tk.HOp()
    h.rows, h.batch = op.rows, op.batch
    for j, s in enumerate(op.a):
        h.a[j] = s.h()
    h.W, h.K, h.N, h.ldw = op.W.data_ptr(), op.K, op.N, op.W.shape[1]
    h.bias = op.bias.data_ptr() if op.bias is not None else None
    h.relu = int(op.relu)
    if op.ln is not None:
        h.ln_g, h.ln_b = op.ln[0].data_ptr(), op.ln[1].data_ptr()
    if op.residual is not None:
        h.residual = op.residual.h()
    h.out, h.ldo = out.data_ptr(), op.ldo
    bound = torch.zeros(1, device="cuda") if (prec != SIMT and op.ln is not None) else None
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    err = ctypes.create_string_buffer(256)
    rc = wh.h_layered_row_op(prec, ctypes.byref(h), tk._p(bound), tk._p(status), err, tk._st())
    torch.cuda.synchronize()
    assert rc == 0, err.value.decode()
    assert int(status.item()) == 0, f"status word {int(status.item())}"
    return out, (float(bound.item()) if bound is not None else None)


def _ln_op(d, N, K, residual, two_source, rows=300, batch=2):
    R = rows * batch
    if two_source:  # [x (broadcast, 300 columns) ; aggregate (256)]: assembled into one operand before the blocks
        a = [bcast(d.operand(rows, 300)), stream(d.operand(R, K - 300), rows)]
    else:
        a = [stream(d.operand(R, K), rows)]
    g = torch.rand(N, generator=d.g, device="cuda") + 0.5
    b = torch.randn(N, generator=d.g, device="cuda") * 0.1
    res = stream(d.addend(R, N), rows) if residual else None
    return RowOp(rows, batch, a, d.weight(N, K), K, N, bias=d.addend(N), ln=(g, b), residual=res)


LN_CASES = [pytest.param(N, K, False, id=f"N{N}_K{K}") for N in (257, 512, 597, 1024) for K in (300, 1024)] + [
    pytest.param(597, 556, True, id="N597_two_source")]


def _check_bound(out, bound, tag):
    m = float(out.abs().max())
    return [] if bound == m else [f"{tag}: bound {bound!r}, max |out| {m!r}"]


@pytest.mark.parametrize("prec", [FP32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("residual", [False, True], ids=["plain", "residual"])
@pytest.mark.parametrize("N,K,two_source", LN_CASES)
def test_ln_row_op_exact(wh, N, K, two_source, residual, prec):
    """Exact-integer data: the column blocks' value entering the LayerNorm equals float64 bit for bit; the LayerNorm'd rows equal
    the CUDA-core path's bit for bit and float64 within 1e-5; the bound is max |out|."""
    d = Data(7000 + N + K, exact=True, s=0)
    op = _ln_op(d, N, K, residual, two_source)
    tag = f"N {N} K {K} {tk.PREC_NAME[prec]}{' residual' if residual else ''}"
    plain = RowOp(op.rows, op.batch, op.a, op.W, K, N, bias=op.bias)  # the same op without LayerNorm and residual
    pre, _ = _run(wh, prec, plain)
    fails = []
    if not torch.equal(pre.double(), plain.ref()[0]):
        fails.append(f"{tag}: the value entering the LayerNorm differs from float64")
    out, bound = _run(wh, prec, op)
    simt, _ = _run(wh, SIMT, op)
    if not torch.equal(out.view(torch.int32), simt.view(torch.int32)):
        fails.append(f"{tag}: {int((out != simt).sum())} LayerNorm'd values differ from the CUDA-core path's")
    y64 = op.ref()[0]
    ef = float((out.double() - y64).norm() / y64.norm())
    if not ef < 1e-5:
        fails.append(f"{tag}: eps_F {ef:.2e} against float64")
    fails += _check_bound(out, bound, tag)
    assert not fails, fails


@pytest.mark.parametrize("prec", [FP32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("data", tk.FLOAT)
@pytest.mark.parametrize("N,K,two_source", LN_CASES)
def test_ln_row_op_float(wh, N, K, two_source, data, prec):
    """Random data (normal, an outlier column, gradients of 1e-8, raw values of 1e5) with a residual: the LayerNorm'd rows within
    the row-op bars (eps_F) of tests/test_gpu_kernels.py, the bound max |out|."""
    d = Data(8000 + N + K, **data)
    op = _ln_op(d, N, K, True, two_source)
    out, bound = _run(wh, prec, op)
    y64 = op.ref()[0]
    ef = float((out.double() - y64).norm() / y64.norm())
    tag = f"N {N} K {K} {tk.PREC_NAME[prec]}"
    print(f"{tag} {data}: eps_F {ef:.2e} (bar {BARS[prec][0]:.0e})")
    fails = [] if ef < BARS[prec][0] else [f"{tag}: eps_F {ef:.2e}"]
    fails += _check_bound(out, bound, tag)
    assert not fails, fails
