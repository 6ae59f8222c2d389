"""-m gpu: the training step at the reference's ERA5 widths (above 256).

Kernels, one at a time, against float64 (the style and helpers of tests/test_gpu_kernels.py: exact-integer data bit for bit,
random floats under the per-precision bars):
  * the wide LayerNorm backward (rows of 257 .. 1024 columns);
  * weight gradients with N and K in {597, 621, 1024} on CUDA cores and on tensor cores (K blocks of 256, o blocks of 128),
    written into a column slice of a wider prefilled buffer;
  * one-layer row ops of N = 597 / 621 as column blocks of at most 256 outputs (residual, mask, addend, misaligned output rows),
    on both chain paths, and stage 0 with K0 = 640 from 597- / 621-wide misaligned rows;
  * the memory-bound primitives and the loss gradient at 597 .. 1024 channels.
The model: a train/run_fulll.py-shaped forecaster (597 + 24 features, 2 blocks, 10-degree grid) in every train precision, and a
train/run.py-shaped one (1024-wide, 605 + 40 features, 2 blocks, 30-degree grid) in fp32_simt, against torch.autograd on the
CPU oracle."""
import ctypes

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import BCAST, BF16, FP32, RUNS, SIMT, STREAM, Data, Src, _eps, _ok, _p, _st, bcast, stream

PREC_NAME = tk.PREC_NAME
EXACT = [pytest.param(dict(exact=True, s=s), id=f"int_s{s}") for s in (-40, 0, 20)]
FLOAT = tk.FLOAT


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    lib = tk._compile_harness(tmp_path_factory.mktemp("gw_wide_harness"))
    tk.HK = lib  # (the helpers of test_gpu_kernels call through it)
    return lib


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


# ---- LayerNorm backward -------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("R", [5, 3001])
@pytest.mark.parametrize("offset", [0.0, 1000.0])
@pytest.mark.parametrize("N", [257, 512, 597, 1024])
def test_ln_bwd_wide(N, offset, R):
    """Rows wider than 256 against float64 autograd of layer_norm(eps=1e-5); dgamma / dbeta accumulate into prefilled buffers and
    dz rows have a stride wider than N (columns beyond N untouched)."""
    g = torch.Generator(device="cuda").manual_seed(N + R)
    ld = N + 3
    z = torch.randn(R, ld, generator=g, device="cuda") + offset
    dy = torch.randn(R, ld, generator=g, device="cuda")
    gamma = torch.rand(N, generator=g, device="cuda") + 0.5
    beta = torch.randn(N, generator=g, device="cuda")
    dg0, db0 = torch.randn(N, generator=g, device="cuda"), torch.randn(N, generator=g, device="cuda")
    dg, dbt = dg0.clone(), db0.clone()
    dz = torch.full((R, ld), float("nan"), device="cuda")
    _ok(tk.HK.h_ln_bwd(_p(dy), ld, _p(z), ld, N, _p(gamma), R, _p(dz), ld, _p(dg), _p(dbt), _st()))
    torch.cuda.synchronize()
    with torch.enable_grad():
        z64 = z[:, :N].double().requires_grad_()
        g64 = gamma.double().requires_grad_()
        b64 = beta.double().requires_grad_()
        y = torch.nn.functional.layer_norm(z64, (N,), g64, b64, eps=1e-5)
        y.backward(dy[:, :N].double())
    ez = float((dz[:, :N].double() - z64.grad).norm() / z64.grad.norm())
    eg = float((dg.double() - dg0.double() - g64.grad).norm() / g64.grad.norm())
    eb = float((dbt.double() - db0.double() - b64.grad).norm() / b64.grad.norm())
    print(f"ln_bwd N {N} R {R} offset {offset}: dz {ez:.2e} dgamma {eg:.2e} dbeta {eb:.2e}")
    # the bars of the 256-wide kernel (tests/test_gpu_kernels.py::test_ln_bwd)
    bar = 2e-6 if offset == 0.0 else 2e-4
    assert ez < bar and eg < bar and eb < 2e-6, (ez, eg, eb)
    assert torch.isnan(dz[:, N:]).all(), "dz columns beyond N were written"


@gpu
def test_ln_bwd_refuses_rows_beyond_its_limit():
    t = torch.zeros(4, 1025, device="cuda")
    g = torch.ones(1025, device="cuda")
    rc = tk.HK.h_ln_bwd(_p(t), 1025, _p(t), 1025, 1025, _p(g), 4, _p(t), 1025, _p(g), _p(g), _st())
    assert rc != 0


# ---- weight gradients ---------------------------------------------------------------------------------------------------------
WG_KINDS = ["fp32", "bf16", "simt"]
# (rows, batch, N, K, A kind): the wide layers of the reference's ERA5 models
WG_SHAPES = {
    "dec_out_n597_k128": (700, 2, 597, 128, STREAM),       # decoder output layer (run_fulll)
    "enc_in_n256_k621": (700, 2, 256, 621, STREAM),        # node encoder Linear 0 on the 597 + 24 features
    "n621_k597": (300, 3, 621, 597, BCAST),                # both wide, a batch-shared A
    "n1024_k1024": (1000, 1, 1024, 1024, STREAM),          # run.py's hidden layers
    "n1024_k645": (555, 2, 1024, 645, STREAM),             # run.py's node encoder Linear 0 (605 + 40 features)
}


def _wg_case(name, d, rows=None, batch=None):
    r0, b0, N, K, kind = WG_SHAPES[name]
    rows, batch = rows or r0, batch or b0
    dY = d.operand(rows * batch, N, outlier=False)
    if kind == STREAM:
        a = Src(STREAM, d.operand(rows * batch, K + 5), K, 3, rows)  # a misaligned column window of wider rows
    else:
        a = Src(BCAST, d.operand(rows, K), K)
    return rows, batch, N, K, dY, a


def _wg_check(kind, rows, batch, N, K, dY, a, d, col=7):
    """One weight gradient into columns col .. col + K of a prefilled [N, K + 20] buffer: (dW slice, db, untouched outside)."""
    ldw = K + 20
    dW = d.addend(N, ldw)
    db = d.operand(N)
    dW0, db0 = dW.clone(), db.clone()
    _ok(tk._wgrad(kind, dY, a, K, rows, batch, dW, col, db))
    torch.cuda.synchronize()
    outside = torch.ones_like(dW, dtype=torch.bool)
    outside[:, col:col + K] = False
    untouched = torch.equal(dW[outside].view(torch.int32), dW0[outside].view(torch.int32))
    return dW[:, col:col + K].double() - dW0[:, col:col + K].double(), db.double() - db0.double(), dW, db, dW0, db0, untouched


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("name", list(WG_SHAPES))
def test_wide_wgrad_exact(name, data):
    """Exact integers: every K block, every o block and the bias sum bit for bit, only the slice written."""
    d = Data(6000 + list(WG_SHAPES).index(name), **data)
    rows, batch, N, K, dY, a = _wg_case(name, d)
    g64, b64, _ = tk._wg_ref(rows, batch, dY, a)
    fails = []
    for kind in WG_KINDS:
        _, _, dW, db, dW0, db0, untouched = _wg_check(kind, rows, batch, N, K, dY, a, d)
        got, want = dW[:, 7:7 + K].double(), dW0[:, 7:7 + K].double() + g64
        if not torch.equal(got, want):
            bad = (got != want)
            fails.append(f"{name} {kind}: {int(bad.sum())} of {got.numel()} dW values differ (columns {sorted(set(bad.nonzero()[:, 1].tolist()))[:8]}...)")
        if not torch.equal(db.double(), db0.double() + b64):
            fails.append(f"{name} {kind}: {int((db.double() != db0.double() + b64).sum())} of {N} db values differ")
        if not untouched:
            fails.append(f"{name} {kind}: values outside the slice changed")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("rows,batch", [(1, 1), (63, 1), (64, 1), (65, 3), (127, 1), (128, 2), (129, 1)])
def test_wide_wgrad_exact_row_counts(rows, batch):
    d = Data(6100 + rows + batch, exact=True, s=0)
    fails = []
    for name in ("n621_k597", "enc_in_n256_k621"):
        _, _, N, K, dY, a = _wg_case(name, d, rows, batch)
        g64, b64, _ = tk._wg_ref(rows, batch, dY, a)
        for kind in WG_KINDS:
            gd, bd, *_, untouched = _wg_check(kind, rows, batch, N, K, dY, a, d)
            if not (torch.equal(gd, g64) and torch.equal(bd, b64) and untouched):
                fails.append(f"{name} {kind}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("name", list(WG_SHAPES))
def test_wide_wgrad_float(name, data):
    d = Data(6200 + list(WG_SHAPES).index(name), **data)
    rows, batch, N, K, dY, a = _wg_case(name, d)
    g64, b64, c = tk._wg_ref(rows, batch, dY, a)
    fails = []
    for kind in WG_KINDS:
        dW = torch.zeros(N, K, device="cuda")
        db = torch.zeros(N, device="cuda")
        _ok(tk._wgrad(kind, dY, a, K, rows, batch, dW, 0, db))
        torch.cuda.synchronize()
        bf, bel = tk.BARS[{"fp32": FP32, "bf16": BF16, "simt": SIMT}[kind]]
        ef, eel = _eps(dW, g64, c)
        _, eelb = _eps(db, b64, dY.double().abs().sum(0))
        print(f"{name} {kind}: dW eps_F {ef:.2e} (bar {bf:.0e}) eps_el {eel:.2e} (bar {bel:.1e})  db eps_el {eelb:.2e} (bar 1e-6)")
        if not (ef < bf and eel < bel):
            fails.append(f"{name} {kind}: dW eps_F {ef:.2e} eps_el {eel:.2e}")
        if not eelb < 1e-6:
            fails.append(f"{name} {kind}: db eps_el {eelb:.2e}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("kind", ["fp32", "bf16"])
def test_wide_wgrad_tc_is_repeatable(kind):
    d = Data(63, exact=False)
    rows, batch, N, K, dY, a = _wg_case("n1024_k645", d, 20_000, 2)
    out = []
    for _ in range(2):
        dW = torch.zeros(N, K, device="cuda")
        db = torch.zeros(N, device="cuda")
        _ok(tk._wgrad(kind, dY, a, K, rows, batch, dW, 0, db))
        torch.cuda.synchronize()
        out.append((dW, db))
    assert torch.equal(out[0][0].view(torch.int32), out[1][0].view(torch.int32))
    assert torch.equal(out[0][1].view(torch.int32), out[1][1].view(torch.int32))


# ---- column-blocked row ops ---------------------------------------------------------------------------------------------------
class BlockedOp(tk.RowOp):
    """A training row op of any N: h_row_op runs the column blocks train_op runs, and run() returns their lean mask."""


def _bshape(name, d, rows=300, batch=2):
    R = rows * batch
    if name == "out597_res":  # decoder output layer: 597 columns + the first 597 of the 621-wide features (odd ldo)
        res = stream(d.addend(R, 621), rows, width=597)
        return BlockedOp(rows, batch, [stream(d.operand(R, 128), rows)], d.weight(597, 128), 128, 597, bias=d.addend(597), residual=res)
    if name == "out597_ldo603":  # the same into rows of stride 603, residual from column 2 of wider rows
        res = stream(d.addend(R, 610), rows, width=597, col0=2)
        return BlockedOp(rows, batch, [stream(d.operand(R, 128), rows)], d.weight(597, 128), 128, 597, bias=d.addend(597), residual=res,
                         ldo=603)  # fmt: skip
    if name == "dgrad621":  # data gradient into the 621 features: dY [R, 256] . W0 (W^T [621, 256])
        return BlockedOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(621, 256), 256, 621)
    if name == "dgrad_mask_add621":  # masked data gradient with an addend, 621 columns (three blocks: 256, 256, 109)
        return BlockedOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(621, 256), 256, 621, add=(stream(d.addend(R, 621), rows),),
                         mask=stream(d.relu_rows(R, 621), rows))  # fmt: skip
    if name == "dgrad_mask597_bcast":  # broadcast mask and addend, relu rows of the batch-shared tables
        return BlockedOp(rows, batch, [stream(d.operand(R, 128), rows)], d.weight(597, 128), 128, 597, add=(bcast(d.addend(rows, 597)),),
                         mask=bcast(d.relu_rows(rows, 597)))  # fmt: skip
    if name == "enc_k621":  # node encoder Linear 0: K0 = 640 from 621-wide (misaligned) feature rows, relu
        return BlockedOp(rows, batch, [stream(d.operand(R, 621), rows)], d.weight(256, 621), 621, 256, bias=d.addend(256), relu=True)
    if name == "dgrad_out_k597":  # data gradient of the output layer: K0 = 640 from 597-wide dY rows, masked by the hidden rows
        return BlockedOp(rows, batch, [stream(d.operand(R, 597), rows)], d.weight(128, 597), 597, 128, mask=stream(d.relu_rows(R, 128), rows))
    raise KeyError(name)


BSHAPES = ["out597_res", "out597_ldo603", "dgrad621", "dgrad_mask_add621", "dgrad_mask597_bcast", "enc_k621", "dgrad_out_k597"]


def _blocked_fails(name, op, y64, prec, nofast, out, lean):
    tag = f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
    fails = []
    if op.ldo > op.N and not torch.isnan(out[:, op.N:]).all():
        fails.append(f"{tag}: columns beyond N written")
    if prec != SIMT and nofast and lean != 0:
        fails.append(f"{tag}: lean mask {lean} under GW_TC3_NOFAST")
    return tag, fails


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("name", BSHAPES)
def test_blocked_row_op_exact(name, data):
    """Exact integers: every column block, both chain paths and every precision reproduce float64 bit for bit."""
    d = Data(7000 + BSHAPES.index(name), **data)
    op = _bshape(name, d)
    y64, _, _ = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, _, lean = op.run(prec, nofast)
        tag, f = _blocked_fails(name, op, y64, prec, nofast, out, lean)
        fails += f
        bad = out[:, :op.N].double() != y64
        if bad.any():
            cols = sorted(set(bad.nonzero()[:, 1].tolist()))
            fails.append(f"{tag}: {int(bad.sum())} of {y64.numel()} values differ (columns {cols[0]} .. {cols[-1]})")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("rows,batch", [(1, 1), (63, 2), (65, 1), (127, 3), (128, 1), (129, 3)])
@pytest.mark.parametrize("name", ["out597_res", "dgrad_mask_add621", "enc_k621"])
def test_blocked_row_op_exact_row_counts(name, rows, batch):
    d = Data(71 + rows + batch, exact=True, s=0)
    op = _bshape(name, d, rows, batch)
    y64, _, _ = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, _, _ = op.run(prec, nofast)
        if not torch.equal(out[:, :op.N].double(), y64):
            fails.append(f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("name", BSHAPES)
def test_blocked_row_op_float(name, data):
    d = Data(7100 + BSHAPES.index(name), **data)
    op = _bshape(name, d)
    y64, _, c = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, _, lean = op.run(prec, nofast)
        tag, f = _blocked_fails(name, op, y64, prec, nofast, out, lean)
        fails += f
        bf, bel = tk.BARS[prec]
        ef, eel = _eps(out[:, :op.N], y64, c)
        print(f"{tag}: eps_F {ef:.2e} (bar {bf:.0e}) eps_el {eel:.2e} (bar {bel:.1e})")
        if not (ef < bf and eel < bel):
            fails.append(f"{tag}: eps_F {ef:.2e} eps_el {eel:.2e}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("prec", [FP32, BF16])
def test_blocked_row_op_refuses_a_split_layernorm(prec):
    """A LayerNorm row cannot be cut into column blocks: the launch fails instead of normalising each block on its own."""
    d = Data(8, exact=False)
    R = 64
    g, b = torch.ones(300, device="cuda"), torch.zeros(300, device="cuda")
    op = BlockedOp(R, 1, [stream(d.operand(R, 256), R)], d.weight(300, 256), 256, 300, ln=(g, b), save_pre=True)
    with pytest.raises(AssertionError, match="CUDA error"):
        op.run(prec)


# ---- CUDA-core row ops and memory-bound primitives at 1024 ----------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["ln_res_save_pre", "mask_add"])
def test_simt_row_op_1024(name):
    """launch_rowop_simt's wide path: the taped pre-LayerNorm value bit for bit (exact data) and the LayerNorm'd output under the
    fp32 bar; a masked data gradient with an addend bit for bit."""
    d = Data(9, exact=True, s=0)
    rows, batch = 300, 2
    R = rows * batch
    if name == "ln_res_save_pre":
        g = torch.rand(1024, generator=d.g, device="cuda") + 0.5
        b = torch.randn(1024, generator=d.g, device="cuda") * 0.1
        op = tk.RowOp(rows, batch, [stream(d.operand(R, 1024), rows)], d.weight(1024, 1024), 1024, 1024, bias=d.addend(1024), ln=(g, b),
                      residual=stream(d.addend(R, 1024), rows), save_pre=True)  # fmt: skip
    else:
        op = tk.RowOp(rows, batch, [stream(d.operand(R, 1024), rows)], d.weight(1024, 1024), 1024, 1024, add=(stream(d.addend(R, 1024), rows),),
                      mask=stream(d.relu_rows(R, 1024), rows))  # fmt: skip
    y64, pre64, _ = op.ref()
    out, pre, _ = op.run(SIMT)
    if op.ln is None:
        assert torch.equal(out.double(), y64)
    else:
        assert torch.equal(pre.double(), pre64)
        ef = float((out.double() - y64).norm() / y64.norm())
        print(f"simt LayerNorm 1024: output eps_F {ef:.2e} (bar 1e-5)")
        assert ef < 1e-5


def _seq_sum(rows_f32):
    if rows_f32.shape[0] == 0:
        return np.zeros(rows_f32.shape[1], np.float32)
    return np.cumsum(rows_f32, axis=0, dtype=np.float32)[-1]


@gpu
def test_segsum_1024():
    """The one-level per-segment sum the training step runs, on 1024-wide edge rows: bit for bit a sequential float32 sum."""
    rng = np.random.Generator(np.random.PCG64(21))
    lengths = rng.integers(0, 9, 100)
    lengths[[0, 40]] = 0
    lengths[7] = 300
    ptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    E, S, B, W = int(ptr[-1]), len(lengths), 2, 1024
    base = rng.standard_normal((B * E, W)).astype(np.float32)
    perm = rng.permutation(E).astype(np.int32)
    out = torch.full((B * S, W), float("nan"), device="cuda")
    tb, tp, tperm = torch.from_numpy(base).cuda(), torch.from_numpy(ptr).cuda(), torch.from_numpy(perm).cuda()
    _ok(tk.HK.h_segsum(_p(tb), W, W, _p(tp), _p(tperm), E, S, B, _p(out), W, _st()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for b in range(B):
        for i in range(S):
            want = _seq_sum(base[b * E + perm[ptr[i]:ptr[i + 1]]])
            assert np.array_equal(got[b * S + i], want), f"sample {b} segment {i}"


@gpu
@pytest.mark.parametrize("width", [605, 1024])
def test_batch_reduce_gather_rows_transpose_wide(width):
    rng = np.random.Generator(np.random.PCG64(width))
    rows, B, src_rows = 501, 3, 257
    x = rng.standard_normal((B * rows, width)).astype(np.float32)
    out = torch.full((rows, width), float("nan"), device="cuda")
    tx = torch.from_numpy(x).cuda()
    _ok(tk.HK.h_batch_reduce(_p(tx), width, rows, width, B, _p(out), width, 0, _st()))
    torch.cuda.synchronize()
    acc = np.zeros((rows, width), np.float32)
    for b in range(B):
        acc = acc + x[b * rows:(b + 1) * rows]
    assert np.array_equal(out.cpu().numpy(), acc)
    gw = width // 4 * 4  # (row gathers move float4s: widths are multiples of 4)
    tin = torch.from_numpy(rng.standard_normal((B * src_rows, 1024)).astype(np.float32)).cuda()
    idx = torch.from_numpy(rng.integers(0, src_rows, rows).astype(np.int32)).cuda()
    gout = torch.full((B * rows, gw), float("nan"), device="cuda")
    _ok(tk.HK.h_gather_rows(_p(tin), 1024, src_rows, _p(idx), rows, gw, B, _p(gout), gw, 0, _st()))
    torch.cuda.synchronize()
    sel = (torch.arange(B, device="cuda")[:, None] * src_rows + idx.long()[None, :]).reshape(-1)
    assert torch.equal(gout, tin[sel, :gw])
    W = torch.randn(width, 3 * 1024 if width == 1024 else 128, device="cuda")
    WT = torch.full((W.shape[1], W.shape[0]), float("nan"), device="cuda")
    _ok(tk.HK.h_transpose(_p(W), W.shape[0], W.shape[1], _p(WT), _st()))
    torch.cuda.synchronize()
    assert torch.equal(WT, W.T)


@gpu
@pytest.mark.parametrize("F", [597, 605])
def test_normalized_mse_loss_and_grad_wide(F):
    from graph_weather_b200 import _capi

    lib = _capi.load()
    g = torch.Generator(device="cuda").manual_seed(F)
    B, Nn = 2, 1003
    pred = torch.randn(B, Nn, F, generator=g, device="cuda")
    target = torch.randn(B, Nn, F, generator=g, device="cuda")
    w = torch.rand(Nn, generator=g, device="cuda")
    iv = torch.rand(F, generator=g, device="cuda") + 0.5
    scale = 1.0 / (B * Nn)
    grad = torch.full_like(pred, float("nan"))
    _capi._check(lib.gw_normalized_mse_loss_grad(_p(pred), _p(target), _p(iv), _p(w), B, Nn, F, None, ctypes.c_float(scale), _p(grad), _st()))
    ws = torch.empty(int(lib.gw_loss_workspace_bytes()), dtype=torch.uint8, device="cuda")
    s = torch.zeros(1, dtype=torch.float64, device="cuda")
    _capi._check(lib.gw_normalized_mse_loss_sum(_p(pred), _p(target), _p(iv), _p(w), B, Nn, F, _p(s), _p(ws), _st()))
    torch.cuda.synchronize()
    d = pred.double() - target.double()
    want = d * 2.0 / F * scale * w.double()[None, :, None] * iv.double()
    err = float(((grad.double() - want).abs() / want.abs().clamp_min(1e-30)).max())
    want_sum = float(((d * d * iv.double()).mean(-1) * w.double()[None, :]).sum())
    serr = abs(float(s.item()) - want_sum) / abs(want_sum)
    print(f"loss F {F}: grad max relative error {err:.2e} (bar 1e-5), sum relative error {serr:.2e} (bar 1e-5)")
    assert err < 1e-5 and serr < 1e-5


# ---- the model ----------------------------------------------------------------------------------------------------------------
def _grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


def _oracle_step(sd, ll, x, target, var, feature_dim, num_blocks, dtype):
    """One training step of the reference arithmetic on the CPU under torch.autograd (fp32: what the reference runs; fp64: the
    ground truth the tolerances are measured against)."""
    from oracle import restate

    sd_g = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    xg = x.to(dtype).clone().requires_grad_(True)
    g = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in restate.build_forecaster_graphs(ll).items()}
    ex, ei, ea = restate.encoder_forward(sd_g, g, xg)
    px = restate.processor_forward(sd_g, ex, ei, ea, num_blocks)
    out = restate.assimilator_decoder_forward(sd_g, g, px, x.shape[0]) + xg[..., :feature_dim]
    loss = restate.normalized_mse_loss(out, target.to(dtype), var, ll, True)
    loss.backward()
    return out.detach(), float(loss.detach()), xg.grad, {k: v.grad for k, v in sd_g.items()}


RUN_FULLL = dict(feature_dim=597, aux_dim=24, num_blocks=2)
RUN_WIDE = dict(feature_dim=605, aux_dim=40, node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024,
                hidden_dim_decoder=1024, num_blocks=2)  # fmt: skip


def _case(cfg, step, batch, seed):
    from oracle import weights

    ll = _grid(step)
    shape_kw = {k: v for k, v in cfg.items()}
    sd = weights.make_state_dict(weights.forecaster_shapes(**shape_kw), seed)
    F, A = cfg["feature_dim"], cfg["aux_dim"]
    x = weights.make_features(batch, len(ll), F + A, seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    target = torch.from_numpy(rng.standard_normal((batch, len(ll), F)).astype(np.float32))
    var = rng.uniform(0.5, 2.0, F).astype(np.float32).tolist()
    ref32 = _oracle_step(sd, ll, x, target, var, F, cfg["num_blocks"], torch.float32)
    ref64 = _oracle_step(sd, ll, x, target, var, F, cfg["num_blocks"], torch.float64)
    return ll, sd, x, target, var, ref32, ref64


@pytest.fixture(scope="module")
def case_fulll():
    return _case(RUN_FULLL, 10, 2, 31)


@pytest.fixture(scope="module")
def case_wide():
    return _case(RUN_WIDE, 30, 1, 32)


def _model(cfg, ll, sd, tp):
    from graph_weather_b200 import GraphWeatherForecaster

    model = GraphWeatherForecaster(ll, train_precision=tp, **cfg).cuda().train()
    model.load_state_dict(sd)
    return model


def _step(model, crit, x, target):
    xc = x.cuda().requires_grad_(True)
    out = model(xc)
    loss = crit(out, target.cuda())
    loss.backward()
    model._train_engine.plan.status()  # raises on a flagged status word
    grads = {k: q.grad.detach().clone() for k, q in model.named_parameters()}
    return out.detach().cpu(), float(loss), xc.grad, grads


def _rel(a, b):
    return float((a.double().cpu() - b).abs().max()) / (float(b.abs().max()) + 1e-30)


def _rel_norm(a, b):
    return float((a.double().cpu() - b.double()).norm()) / (float(b.double().norm()) + 1e-30)


# node encoder, h3_nodes, latent edge encoder, encoder block node MLP: the gradients summed over the whole graph
# (tests/test_gpu_train_precision.py)
ILL_CONDITIONED = ("encoder.h3_nodes", "encoder.node_encoder.", "encoder.latent_edge_encoder.", "encoder.graph_processor.blocks.0.node_model.")


def _check_against_oracle(tp, out, loss, gx, grads, ref32, ref64):
    out32, loss32, gx32, g32 = ref32
    _, _, gx64, g64 = ref64
    assert gx is not None and gx.shape == gx64.shape, "features.grad was not produced"
    assert set(grads) == set(g64)
    fails = []
    if tp == "bf16":
        assert float((out - out32).abs().max()) < 2e-2 and abs(loss - loss32) <= 1e-2 * abs(loss32)
        big = max(float(g.abs().max()) for g in g64.values())
        worst = []
        for k, g in grads.items():
            ref = g64[k].double().flatten()
            if float(ref.abs().max()) <= 1e-6 * big:
                continue
            worst.append((float(torch.nn.functional.cosine_similarity(g.double().cpu().flatten(), ref, dim=0)), k))
        worst.sort()
        for cos, k in worst[:6]:
            print(f"  {k}: cosine vs fp64 {cos:.5f} (bar {0.98 if k.startswith(ILL_CONDITIONED) else 0.99})")
        fails += [(k, cos) for cos, k in worst if cos < (0.98 if k.startswith(ILL_CONDITIONED) else 0.99)]
        return fails
    assert float((out - out32).abs().max()) < 1e-4 and abs(loss - loss32) <= 1e-5 * abs(loss32)
    e_ours, e_ref = _rel(gx, gx64), _rel(gx32, gx64)
    print(f"d loss / d features: rel err vs fp64 {e_ours:.2e} (fp32 oracle {e_ref:.2e}; bar {10 * e_ref + 2e-5:.2e})")
    if not e_ours < 10 * e_ref + 2e-5:
        fails.append(("features", e_ours, e_ref))
    errs = sorted(((_rel(grads[k], g64[k]), _rel(g32[k], g64[k]), k) for k in grads), reverse=True)
    # An isolated ReLU unit within ~1e-6 of zero switches between two fp32 implementations (tests/test_gpu_train_precision.py): a
    # 2e-3 floor on the max-relative error, in both fp32 modes here (measured on an H100: fp32_simt 7.1e-5 on the run_fulll shape's
    # decoder edge MLP where the fp32 oracle has 2.5e-7).  The gradients summed over the whole graph (ILL_CONDITIONED) are held to
    # 5x the bar on the norm-relative error instead (the 1024-wide node encoder's Linear 0: max-relative 3.5e-2 against the fp32
    # oracle's 6.8e-4).
    for eo, er, k in errs[:6]:
        print(f"  {k}: max-rel err vs fp64 {eo:.2e} (fp32 oracle {er:.2e}; bar {max(10 * er + 2e-5, 2e-3):.2e})")
    for eo, er, k in errs:
        if k.startswith(ILL_CONDITIONED):
            no, nr = _rel_norm(grads[k], g64[k]), _rel_norm(g32[k], g64[k])
            print(f"  {k}: norm-rel err vs fp64 {no:.2e} (fp32 oracle {nr:.2e}; bar {5 * (10 * nr + 2e-5):.2e})")
            if not no < 5 * (10 * nr + 2e-5):
                fails.append((k, "norm", no, nr))
        elif not eo < max(10 * er + 2e-5, 2e-3):
            fails.append((k, eo, er))
    med_o, med_r = sorted(e[0] for e in errs)[len(errs) // 2], sorted(e[1] for e in errs)[len(errs) // 2]
    print(f"median rel err vs fp64: ours {med_o:.2e}, fp32 oracle {med_r:.2e}")
    if tp == "fp32_simt" and not med_o < 3 * med_r + 1e-5:
        fails.append(("median", med_o, med_r))
    return fails


def _train_checks(cfg, case, tp):
    from graph_weather_b200 import NormalizedMSELoss

    ll, sd, x, target, var, ref32, ref64 = case
    model = _model(cfg, ll, sd, tp)
    crit = NormalizedMSELoss(var, ll, normalize=True)
    out, loss, gx, grads = _step(model, crit, x, target)
    assert model._train_engine.resolved_precision == tp
    fails = _check_against_oracle(tp, out, loss, gx, grads, ref32, ref64)
    if tp != "fp32_simt":  # tensor-core weight gradients sum in a fixed order: a second step on the same weights repeats them
        model.zero_grad(set_to_none=True)
        _, loss_b, gx_b, grads_b = _step(model, crit, x, target)
        assert loss_b == loss and torch.equal(gx, gx_b)
        # the Linear layers (model.0 / .2 / .4) and h3_nodes (a data gradient); not the LayerNorm parameters (CUDA-core atomics) nor
        # the first layer of the 2-wide edge encoders (K = 2: the CUDA-core kernel, float atomics across row slabs)
        keys = [k for k in grads if k == "encoder.h3_nodes" or (any(f".model.{i}." in k for i in (0, 2, 4)) and not
                (".model.0." in k and "edge_encoder" in k))]  # fmt: skip
        assert len(keys) > 50
        diff = [k for k in keys if not torch.equal(grads[k].view(torch.int32), grads_b[k].view(torch.int32))]
        assert not diff, diff[:5]
    # a few optimiser steps on the fixed batch: the weights are re-uploaded every step and the loss goes down
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    losses = []
    for _ in range(4):
        opt.zero_grad(set_to_none=True)
        lo = crit(model(x.cuda()), target.cuda())
        lo.backward()
        opt.step()
        losses.append(float(lo))
    model._train_engine.plan.status()
    print(f"{tp}: losses over 4 AdamW steps {[f'{v:.5f}' for v in losses]}")
    assert all(np.isfinite(losses)) and losses[-1] < losses[1] < losses[0], losses
    assert all(q.grad is not None and torch.isfinite(q.grad).all() for q in model.parameters())
    assert not fails, fails


@pytest.mark.gpu
@pytest.mark.training
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_run_fulll_shaped_training_step(case_fulll, tp):
    """597 + 24 features, 597 outputs on the default 256-wide trunk, 2 blocks, 10-degree grid, batch 2."""
    ge.build()
    _train_checks(RUN_FULLL, case_fulll, tp)


@pytest.mark.gpu
@pytest.mark.training
def test_1024_wide_training_step(case_wide):
    """run.py's 1024-wide widths (605 + 40 features), 2 blocks, 30-degree grid, batch 1, exact fp32."""
    ge.build()
    _train_checks(RUN_WIDE, case_wide, "fp32_simt")
