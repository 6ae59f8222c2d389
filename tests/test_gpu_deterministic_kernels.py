"""-m gpu: the fixed-order weight gradient and LayerNorm backward (gw_train_set_deterministic) one at a time, against float64.

The CUDA-core weight gradient and the LayerNorm backward sum their per-slab / per-CTA parts with float atomics by default; their
fixed-order variants store those parts in a workspace and add them in an order that follows from the shapes.  Checked here, in
the style of tests/test_gpu_kernels.py:
  * exact-integer inputs reproduce the float64 result bit for bit (a dropped, repeated or misplaced partial is a mismatch);
  * random floats stay within the fp32 bars of the atomic kernels;
  * repeated launches, on the current stream and on another one, give identical bits;
  * the workspace stays within its fixed budget, also for train/run.py's 1024 x 1024 weights.
Shapes: K in {2, 3, 256, 621} x N in {64, 256, 1024} over 12 345 x 3 rows (several slabs of rows, not a multiple of them), and
LayerNorm rows of N in {78, 256, 300, 1024} (both kernels: N <= 256 and wider)."""
import ctypes
import os
import subprocess

import pytest
import torch

import __graft_entry__ as ge
import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import BARS, SIMT, Data, _eps, _ok, _p, _st, stream

WG_ROWS, WG_BATCH = 12_345, 3
WG_SHAPES = [(N, K) for N in (64, 256, 1024) for K in (2, 3, 256, 621)]
LN_N = [78, 256, 300, 1024]


DET_HARNESS = os.path.join(tk.ROOT, "tests", "kernels", "gw_det_harness.cu")
DK = None  # the fixed-order kernels' harness (fixture `hk`); tk.HK: tests/kernels/gw_kernel_harness.cu, for the atomic kernels


def _compile_det_harness(out_dir):
    """Builds the package (and gw_kernel_harness.cu, tk.HK), then gw_det_harness.cu against the same libgwb200.so."""
    tk.HK = tk._compile_harness(out_dir)
    so = os.path.join(str(out_dir), "libgwdetharness.so")
    cmd = [ge.NVCC, "-shared", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", DET_HARNESS, "-o", so,
           "-L" + tk.PKG, "-lgwb200", "-lcudart", "-Xlinker", "-rpath," + tk.PKG, "-Xlinker", "--no-undefined"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"harness build failed:\n{r.stdout}{r.stderr}"
    lib = ctypes.CDLL(so)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    pws = ctypes.POINTER(ctypes.c_longlong)
    lib.h_sizeof_src.restype, lib.h_sizeof_src.argtypes = ctypes.c_int, []
    lib.h_det_ws_bytes.restype, lib.h_det_ws_bytes.argtypes = ctypes.c_longlong, []
    lib.h_wgrad_det.restype = ctypes.c_int
    lib.h_wgrad_det.argtypes = [vp, i32, i32, ctypes.POINTER(tk.HSrc), i32, i32, i32, vp, i32, vp, pws, vp]
    lib.h_ln_bwd_det.restype = ctypes.c_int
    lib.h_ln_bwd_det.argtypes = [vp, i32, vp, i32, i32, vp, i64, vp, i32, vp, vp, pws, vp]
    return lib


@pytest.mark.skipif(not os.path.exists(ge.NVCC), reason="needs nvcc")
def test_det_harness_builds_and_links(tmp_path):
    """No GPU needed: the harness compiles and links against a fresh build, and its HSrc matches the ctypes mirror."""
    lib = _compile_det_harness(tmp_path)
    assert lib.h_sizeof_src() == ctypes.sizeof(tk.HSrc)
    assert lib.h_det_ws_bytes() == 32 << 20


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    global DK
    DK = _compile_det_harness(tmp_path_factory.mktemp("gw_det_harness"))
    return DK


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


def _budget():
    return int(DK.h_det_ws_bytes())


# ---- weight gradient ---------------------------------------------------------------------------------------------------------
def _wgrad_det(dY, a, K, rows, batch, dW, col, db):
    """dW[:, col:col + K] += dY^T A, db += colsum(dY) (db may be None); returns the workspace bytes."""
    ws = ctypes.c_longlong(0)
    h = a.h()
    pw = ctypes.c_void_p(dW.data_ptr() + 4 * col)
    _ok(DK.h_wgrad_det(_p(dY), dY.shape[1], dY.shape[1], ctypes.byref(h), K, rows, batch, pw, dW.shape[1], _p(db), ctypes.byref(ws), _st()))
    return 4 * ws.value


def _wg_case(N, K, d):
    R = WG_ROWS * WG_BATCH
    dY = d.operand(R, N, outlier=False)
    a = stream(d.operand(R, K), WG_ROWS)
    return dY, a


@gpu
@pytest.mark.parametrize("data", tk.EXACT)
@pytest.mark.parametrize("N,K", WG_SHAPES)
def test_wgrad_det_exact(N, K, data):
    """Exact integers: bit for bit the float64 result, written into a column slice (offset 3) of a wider prefilled buffer that
    stays untouched outside it; the bias gradient too."""
    d = Data(7000 + 10 * N + K, **data)
    dY, a = _wg_case(N, K, d)
    g64, b64, _ = tk._wg_ref(WG_ROWS, WG_BATCH, dY, a)
    ldw, col = K + 8, 3
    dW = d.addend(N, ldw)
    db = d.operand(N)
    dW0, db0 = dW.clone(), db.clone()
    ws = _wgrad_det(dY, a, K, WG_ROWS, WG_BATCH, dW, col, db)
    torch.cuda.synchronize()
    got, want = dW[:, col:col + K].double(), dW0[:, col:col + K].double() + g64
    assert torch.equal(got, want), f"{(got != want).sum().item()} of {got.numel()} dW values differ"
    assert torch.equal(db.double(), db0.double() + b64), "db differs"
    outside = torch.ones_like(dW, dtype=torch.bool)
    outside[:, col:col + K] = False
    assert torch.equal(dW[outside].view(torch.int32), dW0[outside].view(torch.int32)), "values outside the slice changed"
    assert 0 < ws <= _budget(), ws


@gpu
@pytest.mark.parametrize("data", tk.FLOAT)
@pytest.mark.parametrize("N,K", WG_SHAPES)
def test_wgrad_det_float(N, K, data):
    """Random floats: within the fp32_simt bars of the atomic kernel (tests/test_gpu_kernels.py)."""
    d = Data(8000 + 10 * N + K, **data)
    dY, a = _wg_case(N, K, d)
    g64, b64, c = tk._wg_ref(WG_ROWS, WG_BATCH, dY, a)
    dW = torch.zeros(N, K, device="cuda")
    db = torch.zeros(N, device="cuda")
    _wgrad_det(dY, a, K, WG_ROWS, WG_BATCH, dW, 0, db)
    torch.cuda.synchronize()
    bf, bel = BARS[SIMT]
    ef, eel = _eps(dW, g64, c)
    efb, eelb = _eps(db, b64, dY.abs().sum(0, dtype=torch.float64))
    print(f"N {N} K {K}: dW eps_F {ef:.2e} eps_el {eel:.2e}  db eps_F {efb:.2e} eps_el {eelb:.2e}")
    assert ef < bf and eel < bel, (ef, eel)
    assert eelb < 1e-6, eelb


@gpu
@pytest.mark.parametrize("N,K,rows", [(64, 2, 12_345), (256, 3, 12_345), (256, 256, 40_001), (1024, 621, 9_999), (1024, 1024, 20_000)])
def test_wgrad_det_repeats_across_launches_and_streams(N, K, rows):
    """Three launches -- two on the current stream, one on another stream -- give identical bits (bias included), and the
    workspace stays within its budget (1024 x 1024: train/run.py's widest weights)."""
    d = Data(9000 + N + K, exact=False)
    dY = d.operand(rows * 2, N)
    a = stream(d.operand(rows * 2, K), rows)
    outs = []
    side = torch.cuda.Stream()
    for s in (torch.cuda.current_stream(), torch.cuda.current_stream(), side):
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            dW = torch.zeros(N, K, device="cuda")
            db = torch.zeros(N, device="cuda")
            ws = _wgrad_det(dY, a, K, rows, 2, dW, 0, db)
        torch.cuda.synchronize()
        assert 0 < ws <= _budget(), (ws, _budget())
        outs.append((dW.view(torch.int32).clone(), db.view(torch.int32).clone()))
    for dW, db in outs[1:]:
        assert torch.equal(dW, outs[0][0]) and torch.equal(db, outs[0][1]), "fixed-order weight gradient is not repeatable"


@gpu
def test_wgrad_det_no_bias_and_zero_rows():
    """db = nullptr leaves nothing else written; no rows leaves dW untouched."""
    d = Data(11, exact=False)
    N, K, rows = 300, 40, 5_000
    dY = d.operand(rows, N)
    a = stream(d.operand(rows, K), rows)
    dW = torch.full((N, K), 5.0, device="cuda")
    _wgrad_det(dY, a, K, rows, 1, dW, 0, None)
    torch.cuda.synchronize()
    ref = 5.0 + dY.double().T @ a.t.double()
    assert float((dW.double() - ref).abs().max() / ref.abs().max()) < 1e-5
    dW.fill_(5.0)
    assert _wgrad_det(dY, a, K, 0, 1, dW, 0, None) == 0
    torch.cuda.synchronize()
    assert torch.all(dW == 5.0)


# ---- LayerNorm backward -------------------------------------------------------------------------------------------------------
def _ln(kernel, dy, z, gamma, dg, dbt):
    """(dz, workspace bytes) of one LayerNorm backward; dgamma / dbeta accumulate into dg / dbt."""
    R, N = z.shape
    dz = torch.full_like(z, float("nan"))
    if kernel == "atomic":
        _ok(tk.HK.h_ln_bwd(_p(dy), N, _p(z), N, N, _p(gamma), R, _p(dz), N, _p(dg), _p(dbt), _st()))
        return dz, 0
    ws = ctypes.c_longlong(0)
    _ok(DK.h_ln_bwd_det(_p(dy), N, _p(z), N, N, _p(gamma), R, _p(dz), N, _p(dg), _p(dbt), ctypes.byref(ws), _st()))
    return dz, 4 * ws.value


@gpu
@pytest.mark.parametrize("s", [-40, 0, 20])
@pytest.mark.parametrize("R", [5, 20_001])
@pytest.mark.parametrize("N", LN_N)
def test_ln_bwd_det_exact(N, R, s):
    """Rows of +-2^10 with as many of each sign normalise to exactly +-1, so that with integer dy (x 2^s) dgamma and dbeta are
    exact integer sums: bit for bit the float64 result, added to prefilled buffers.  dz is per row, the same code as the atomic
    kernel's: bit for bit its dz."""
    g = torch.Generator(device="cuda").manual_seed(N + R)
    sign = torch.ones(R, N, device="cuda")
    sign[:, N // 2:] = -1.0
    z = torch.gather(sign, 1, torch.argsort(torch.rand(R, N, generator=g, device="cuda"), dim=1)) * 1024.0
    dy = torch.randint(-3, 4, (R, N), generator=g, device="cuda").float() * 2.0**s
    gamma = torch.randint(1, 4, (N,), generator=g, device="cuda").float()
    dg0 = torch.randint(-3, 4, (N,), generator=g, device="cuda").float() * 2.0**s
    db0 = torch.randint(-3, 4, (N,), generator=g, device="cuda").float() * 2.0**s
    dg, dbt = dg0.clone(), db0.clone()
    dz, ws = _ln("det", dy, z, gamma, dg, dbt)
    dz_atomic, _ = _ln("atomic", dy, z, gamma, dg0.clone(), db0.clone())
    torch.cuda.synchronize()
    zh = z.double() / 1024.0
    assert torch.equal(dg.double(), dg0.double() + (dy.double() * zh).sum(0)), "dgamma differs"
    assert torch.equal(dbt.double(), db0.double() + dy.double().sum(0)), "dbeta differs"
    assert torch.equal(dz.view(torch.int32), dz_atomic.view(torch.int32)), "dz differs from the atomic kernel's"
    assert 0 < ws <= _budget()


@gpu
@pytest.mark.parametrize("offset", [0.0, 1000.0])
@pytest.mark.parametrize("N", LN_N)
def test_ln_bwd_det_float(N, offset):
    """Random floats against float64 autograd of layer_norm(eps=1e-5), under the bars of the atomic kernel's tests."""
    g = torch.Generator(device="cuda").manual_seed(N)
    R = 30_001
    z = torch.randn(R, N, generator=g, device="cuda") + offset
    dy = torch.randn(R, N, generator=g, device="cuda")
    gamma = torch.rand(N, generator=g, device="cuda") + 0.5
    beta = torch.randn(N, generator=g, device="cuda")
    dg0, db0 = torch.randn(N, generator=g, device="cuda"), torch.randn(N, generator=g, device="cuda")
    dg, dbt = dg0.clone(), db0.clone()
    dz, _ = _ln("det", dy, z, gamma, dg, dbt)
    torch.cuda.synchronize()
    with torch.enable_grad():
        z64 = z.double().requires_grad_()
        g64 = gamma.double().requires_grad_()
        b64 = beta.double().requires_grad_()
        torch.nn.functional.layer_norm(z64, (N,), g64, b64, eps=1e-5).backward(dy.double())
    ez = float((dz.double() - z64.grad).norm() / z64.grad.norm())
    eg = float((dg.double() - dg0.double() - g64.grad).norm() / g64.grad.norm())
    eb = float((dbt.double() - db0.double() - b64.grad).norm() / b64.grad.norm())
    print(f"ln_bwd_det N {N} offset {offset}: dz {ez:.2e} dgamma {eg:.2e} dbeta {eb:.2e}")
    bar = 2e-6 if offset == 0.0 else 2e-4
    assert ez < bar and eg < bar and eb < 2e-6, (ez, eg, eb)


@gpu
@pytest.mark.parametrize("N", LN_N)
def test_ln_bwd_det_repeats_across_launches_and_streams(N):
    """Two launches on the current stream and one on another stream give identical dz, dgamma and dbeta bits."""
    g = torch.Generator(device="cuda").manual_seed(3 * N)
    R = 50_003
    z = torch.randn(R, N, generator=g, device="cuda")
    dy = torch.randn(R, N, generator=g, device="cuda")
    gamma = torch.rand(N, generator=g, device="cuda") + 0.5
    outs = []
    side = torch.cuda.Stream()
    for s in (torch.cuda.current_stream(), torch.cuda.current_stream(), side):
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            dg, dbt = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
            dz, ws = _ln("det", dy, z, gamma, dg, dbt)
        torch.cuda.synchronize()
        assert 0 < ws <= _budget()
        outs.append([t.view(torch.int32).clone() for t in (dz, dg, dbt)])
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0])), "fixed-order LayerNorm backward is not repeatable"
