"""The CUDA primitives of the training step, one at a time, against float64 references that torch computes on the GPU from the
same fp32 inputs (never against another kernel).

The kernels are reached through tests/kernels/gw_kernel_harness.cu, a host-only shim over the library's internal launchers that
the `harness` fixture compiles into a temporary directory and links against the freshly built libgwb200.so.

Every kernel is checked in two ways:
  (a) exact-integer inputs -- values in {-3..3} x 2^s, s in {-40, 0, 20}, sums far below 2^24 units -- are exact in fp16, bf16
      and fp32, so every kernel (whatever its precision) must reproduce the float64 result bit for bit: a dropped or repeated
      row, a sample mix-up, a wrong mask or a wrong power-of-two scale becomes a mismatch whatever the tolerance.  With s = -40 an
      operand that is not scaled up into the fp16 range underflows.
  (b) random floats -- normal data, an outlier column 1e4 above the rest, gradient-sized (1e-8) and raw (1e5) magnitudes --
      are held to per-precision bars on  eps_F = |y - y64|_F / |y64|_F  and  eps_el = max |y - y64| / (|A| |W|^T + |y64|).
      The fp32 bars sit well below what a dropped lo-part product (about 2^-12 relative per product) leaves."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import __graft_entry__ as ge

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "kernels", "gw_kernel_harness.cu")
PKG = os.path.join(ROOT, "graph_weather_b200")

NONE, STREAM, BCAST, GATHER, SEGSUM, GBR, BGATHER = 0, 1, 2, 3, 4, 5, 6  # gw::SrcKind (GBR: relu(gather + broadcast))
SIMT, FP32, BF16 = 0, 1, 2
PREC_NAME = {SIMT: "fp32_simt", FP32: "fp32", BF16: "bf16"}

# Bars (eps_F, eps_el) of the random-float cases.  Worst values measured over every case of this file on an H100 80GB HBM3 (400 W):
#   fp32_simt  row ops 4.3e-7 / 1.3e-6,  weight gradients 6.1e-7 / 2.0e-7
#   fp32       row ops 1.8e-6 / 2.5e-6,  weight gradients 7.3e-6 / 2.4e-7 (eps_F of the two long reductions, measured at 700 W: each
#              wgmma accumulator sums at most 2048 rows, gw_wgrad_tc.cu; the other shapes, <= 8.5e3 rows, stay below 1.1e-6)
#   bf16       row ops 2.4e-3 / 4.9e-3,  weight gradients 4.8e-3 / 1.7e-3
# A dropped lo-part product leaves about 2^-12 = 2.4e-4 relative per product: 24x the fp32 eps_F bar.
BARS = {
    SIMT: (1e-5, 1e-4),
    FP32: (1e-5, 1e-4),
    BF16: (8e-3, 2.0**-7),
}


# ---- the harness ------------------------------------------------------------------------------------------------------------
class HSrc(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("width", ctypes.c_int32), ("ld", ctypes.c_int32), ("col0", ctypes.c_int32),
                ("base", ctypes.c_void_p), ("src_rows", ctypes.c_int32), ("idx", ctypes.c_void_p), ("base2", ctypes.c_void_p),
                ("ld2", ctypes.c_int32), ("bound_mul_i", ctypes.c_void_p), ("ptr", ctypes.c_void_p), ("perm", ctypes.c_void_p)]


class HOp(ctypes.Structure):
    _fields_ = [("rows", ctypes.c_int32), ("batch", ctypes.c_int32), ("a", HSrc * 2), ("W", ctypes.c_void_p), ("K", ctypes.c_int32),
                ("N", ctypes.c_int32), ("ldw", ctypes.c_int32), ("bias", ctypes.c_void_p), ("add", HSrc * 2), ("relu", ctypes.c_int32),
                ("ln_g", ctypes.c_void_p), ("ln_b", ctypes.c_void_p), ("residual", HSrc), ("out", ctypes.c_void_p), ("ldo", ctypes.c_int32),
                ("save_pre", ctypes.c_void_p), ("mask", HSrc)]


class HLayer(ctypes.Structure):  # one forward chain layer (tests/test_gpu_chains.py)
    _fields_ = [("W", ctypes.c_void_p), ("K", ctypes.c_int32), ("N", ctypes.c_int32), ("ldw", ctypes.c_int32), ("bias", ctypes.c_void_p),
                ("add", HSrc * 2), ("relu", ctypes.c_int32), ("ln_g", ctypes.c_void_p), ("ln_b", ctypes.c_void_p), ("residual", HSrc),
                ("out", ctypes.c_void_p), ("ldo", ctypes.c_int32), ("out_cols", ctypes.c_int32), ("feeds_next", ctypes.c_int32),
                ("reuse_a", ctypes.c_int32), ("seg_dst", ctypes.c_void_p), ("seg_out", ctypes.c_void_p), ("seg_ld", ctypes.c_int32),
                ("seg_rows", ctypes.c_int32), ("seg_maxdeg", ctypes.c_int32), ("seg_add", ctypes.c_void_p), ("out_bound", ctypes.c_void_p),
                ("seg_bound", ctypes.c_void_p)]


class HChain(ctypes.Structure):
    _fields_ = [("rows", ctypes.c_int32), ("batch", ctypes.c_int32), ("K0", ctypes.c_int32), ("n_layers", ctypes.c_int32), ("a0", HSrc * 2),
                ("layer", HLayer * 6), ("out_mode", ctypes.c_int32), ("n_out_peers", ctypes.c_int32), ("out_peer", ctypes.c_void_p * 3)]


_vp, _i32, _i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
_SIGNATURES = {
    "h_sizeof_src": [],
    "h_sizeof_op": [],
    "h_sizeof_layer": [],
    "h_sizeof_chain": [],
    "h_chain": [_i32, ctypes.POINTER(HChain), ctypes.POINTER(ctypes.c_int), _vp, _vp],
    "h_wgrad_tc": [_i32, _vp, _i32, _i32, ctypes.POINTER(HSrc), _i32, _i32, _i32, _vp, _i32, _vp, _vp, _vp],
    "h_wgrad_simt": [_vp, _i32, _i32, ctypes.POINTER(HSrc), _i32, _i32, _i32, _vp, _i32, _vp, _vp],
    "h_row_op": [_i32, ctypes.POINTER(HOp), ctypes.POINTER(ctypes.c_int), _vp, _vp],
    "h_ln_bwd": [_vp, _i32, _vp, _i32, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp],
    "h_segsum": [_vp, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _vp, _i32, _vp],
    "h_segsum_chunked": [_vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp],
    "h_batch_reduce": [_vp, _i32, _i64, _i32, _i32, _vp, _i32, _i32, _vp],
    "h_gather_rows": [_vp, _i32, _i32, _vp, _i64, _i32, _i32, _vp, _i32, _i32, _vp],
    "h_segsum_range": [_vp, _i32, _i32, _vp, _vp, _i32, _i32, _i32, _vp, _i32, _i32, _i32, _vp],
    "h_gather_rows_base": [_vp, _i32, _i32, _vp, _i64, _i32, _i32, _vp, _i32, _i32, _i32, _vp],
    "h_permute_rows": [_vp, _i32, _vp, _i64, _i32, _i32, _i32, _vp, _i32, _i32, _vp],
    "h_strided_add": [_vp, _i32, _vp, _i32, _i64, _i32, _vp],
    "h_transpose": [_vp, _i32, _i32, _vp, _vp],
    "h_pad_rows": [_vp, _i32, _i32, _vp, _i32, _i64, _vp, _vp],
    "h_absmax_flat": [_vp, _i64, _vp, _vp],
    "h_csr_expand": [_vp, _i32, _vp, _vp, _vp],
    "h_sort_csr": [_vp, _i32, _i32, _vp, _vp, _vp],
    "h_obs_graph": [_i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, ctypes.c_double, ctypes.c_double, ctypes.c_double, _vp, _i32, _i32, _vp, _vp,
                    _vp, _vp, _vp, _vp],
}


def _compile_harness(out_dir):
    """Builds the package, then the harness against its libgwb200.so (undefined symbols are link errors)."""
    ge.build()
    so = os.path.join(str(out_dir), "libgwharness.so")
    cmd = [ge.NVCC, "-shared", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", HARNESS, "-o", so,
           "-L" + PKG, "-lgwb200", "-lcudart", "-Xlinker", "-rpath," + PKG, "-Xlinker", "--no-undefined"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"harness build failed:\n{r.stdout}{r.stderr}"
    lib = ctypes.CDLL(so)
    for name, args in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = ctypes.c_int, args
    return lib


def test_harness_builds_and_links(tmp_path):
    """No GPU needed: the harness compiles and links against a fresh build, and its structs match their ctypes mirrors."""
    lib = _compile_harness(tmp_path)
    assert lib.h_sizeof_src() == ctypes.sizeof(HSrc)
    assert lib.h_sizeof_op() == ctypes.sizeof(HOp)
    assert lib.h_sizeof_layer() == ctypes.sizeof(HLayer)
    assert lib.h_sizeof_chain() == ctypes.sizeof(HChain)


HK = None  # the harness library of the GPU tests (fixture `hk`)


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    global HK
    HK = _compile_harness(tmp_path_factory.mktemp("gw_kernel_harness"))
    return HK


def gpu(f):
    """A test that runs kernels: needs a GPU and the harness."""
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _a(t):  # address for a pointer field of HOp
    return t.data_ptr() if t is not None else None


def _ok(rc):
    assert rc == 0, f"CUDA error {rc}"


# ---- data --------------------------------------------------------------------------------------------------------------------
class Data:
    """Value generator of one case.  exact: integers in {-3..3} x 2^s (operands) and x 2^(2 s) (values added to products);
    otherwise normal floats of magnitude `mag`, optionally with an outlier column 1e4 above the rest."""

    def __init__(self, seed, exact, s=0, mag=1.0, outlier=False):
        self.g = torch.Generator(device="cuda").manual_seed(seed)
        self.exact, self.s, self.mag, self.outlier = exact, s, mag, outlier

    def _ints(self, shape, e):
        return torch.randint(-3, 4, shape, generator=self.g, device="cuda").float() * 2.0**e

    def operand(self, *shape, outlier=True):  # activations / upstream gradients
        if self.exact:
            return self._ints(shape, self.s)
        t = torch.randn(shape, generator=self.g, device="cuda") * self.mag
        if self.outlier and outlier:
            t[..., shape[-1] // 3] *= 1e4
        return t

    def weight(self, *shape):
        if self.exact:
            return self._ints(shape, self.s)
        return torch.randn(shape, generator=self.g, device="cuda") * 0.06

    def addend(self, *shape):  # bias / addends / residual: on the grid of the products
        if self.exact:
            return self._ints(shape, 2 * self.s)
        return torch.randn(shape, generator=self.g, device="cuda") * (self.mag * 0.5)

    def relu_rows(self, *shape):  # a taped ReLU output: many exact zeros
        return torch.relu(self._ints(shape, 0) if self.exact else torch.randn(shape, generator=self.g, device="cuda"))


EXACT = [pytest.param(dict(exact=True, s=s), id=f"int_s{s}") for s in (-40, 0, 20)]
FLOAT = [pytest.param(dict(exact=False, mag=1.0), id="normal"), pytest.param(dict(exact=False, mag=1.0, outlier=True), id="outlier"),
         pytest.param(dict(exact=False, mag=1e-8), id="grad1e-8"), pytest.param(dict(exact=False, mag=1e5), id="raw1e5")]


class Src:
    """A row source over a 2-d fp32 tensor t [*, ld]; rows64() assembles the [batch * rows, width] float64 rows it stands for.
    SEGSUM: the sum of t's rows over CSR segment i (ptr, optional perm); GBR: relu(t[b, idx[i]] + t2[i]) (t2 [rows, ld2])."""

    def __init__(self, kind, t, width, col0=0, src_rows=0, idx=None, ptr=None, perm=None, t2=None):
        self.kind, self.t, self.width, self.ld, self.col0, self.src_rows, self.idx = kind, t, width, t.shape[1], col0, src_rows, idx
        self.ptr, self.perm, self.t2 = ptr, perm, t2

    def h(self):
        def a(x):
            return x.data_ptr() if x is not None else None

        return HSrc(self.kind, self.width, self.ld, self.col0, self.t.data_ptr(), self.src_rows, a(self.idx), a(self.t2),
                    self.t2.shape[1] if self.t2 is not None else 0, None, a(self.ptr), a(self.perm))  # fmt: skip

    def rows64(self, rows, batch, absolute=False):
        """absolute: the rows of |values| a sum runs over (SEGSUM: the sum of |rows|), for the magnitude term of eps_el."""
        t = self.t[:, self.col0:self.col0 + self.width].double()
        b = torch.arange(batch, device="cuda")[:, None]
        i = torch.arange(rows, device="cuda")[None, :]
        if self.kind == SEGSUM:  # float64 sum over each segment, rows in perm order when perm is set
            t = t.abs() if absolute else t
            ptr = self.ptr.long()
            seg = torch.repeat_interleave(torch.arange(rows, device="cuda"), ptr[1:] - ptr[:-1])
            e = self.perm.long() if self.perm is not None else torch.arange(int(ptr[-1]), device="cuda")
            out = torch.zeros(batch, rows, self.width, dtype=torch.float64, device="cuda")
            for s in range(batch):
                out[s].index_add_(0, seg, t[s * self.src_rows + e])
            return out.reshape(batch * rows, self.width)
        if self.kind == GBR:
            g = t[(b * self.src_rows + self.idx.long()[None, :]).reshape(-1)]
            return torch.relu(g + self.t2[:, :self.width].double()[i.expand(batch, rows).reshape(-1)])
        if self.kind == STREAM:
            r = b * self.src_rows + i
        elif self.kind == BCAST:
            r = i.expand(batch, rows)
        elif self.kind == GATHER:
            r = b * self.src_rows + self.idx.long()[None, :]
        else:
            r = self.idx.long()[None, :].expand(batch, rows)
        return t[r.reshape(-1)]


def stream(t, rows, width=None, col0=0):
    return Src(STREAM, t, t.shape[1] if width is None else width, col0, rows)


def bcast(t, width=None):
    return Src(BCAST, t, t.shape[1] if width is None else width)


def _eps(y, y64, c):
    d = y.double() - y64
    ef = float(d.norm() / y64.norm().clamp_min(1e-300))
    eel = float((d.abs() / (c + y64.abs()).clamp_min(1e-300)).max())
    return ef, eel


# ---- one training row op -----------------------------------------------------------------------------------------------------
class RowOp:
    """A GemmOp of the training step: out = mask(residual + LN(relu(concat(a) W^T + bias + add))) over batch x rows rows."""

    def __init__(self, rows, batch, a, W, K, N, wcol=0, bias=None, add=(), relu=False, ln=None, residual=None, save_pre=False, mask=None,
                 ldo=None):
        self.rows, self.batch, self.a, self.W, self.K, self.N, self.wcol = rows, batch, a, W, K, N, wcol
        self.bias, self.add, self.relu, self.ln, self.residual, self.save_pre, self.mask = bias, add, relu, ln, residual, save_pre, mask
        self.ldo = N if ldo is None else ldo

    def run(self, prec, nofast=False):
        R = self.rows * self.batch
        out = torch.full((R, self.ldo), float("nan"), device="cuda")
        pre = torch.full((R, self.ldo), float("nan"), device="cuda") if self.save_pre else None
        h = HOp()
        h.rows, h.batch = self.rows, self.batch
        for j, s in enumerate(self.a):
            h.a[j] = s.h()
        h.W = self.W.data_ptr() + 4 * self.wcol
        h.K, h.N, h.ldw = self.K, self.N, self.W.shape[1]
        h.bias = _a(self.bias)
        for j, s in enumerate(self.add):
            h.add[j] = s.h()
        h.relu = int(self.relu)
        if self.ln is not None:
            h.ln_g, h.ln_b = _a(self.ln[0]), _a(self.ln[1])
        if self.residual is not None:
            h.residual = self.residual.h()
        h.out, h.ldo, h.save_pre = out.data_ptr(), self.ldo, _a(pre)
        if self.mask is not None:
            h.mask = self.mask.h()
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        lean = ctypes.c_int(-2)
        old = os.environ.pop("GW_TC3_NOFAST", None)
        try:
            if nofast:
                os.environ["GW_TC3_NOFAST"] = "1"
            _ok(HK.h_row_op(prec, ctypes.byref(h), ctypes.byref(lean), _p(status), _st()))
            torch.cuda.synchronize()
        finally:
            os.environ.pop("GW_TC3_NOFAST", None)
            if old is not None:
                os.environ["GW_TC3_NOFAST"] = old
        assert int(status.item()) == 0, f"status word {int(status.item())}"
        return out, pre, lean.value

    def ref(self):
        """float64: (out, pre-LayerNorm value, |A| |W|^T)."""
        A = torch.cat([s.rows64(self.rows, self.batch) for s in self.a], dim=1)
        W = self.W[:, self.wcol:self.wcol + self.K].double()
        y = A @ W.T
        c = torch.cat([s.rows64(self.rows, self.batch, absolute=True) for s in self.a], dim=1).abs() @ W.abs().T
        if self.bias is not None:
            y = y + self.bias.double()
        for s in self.add:
            y = y + s.rows64(self.rows, self.batch)
        if self.relu:
            y = torch.relu(y)
        pre = y
        if self.ln is not None:
            y = torch.nn.functional.layer_norm(y, (self.N,), self.ln[0].double(), self.ln[1].double(), eps=1e-5)
        if self.residual is not None:
            y = y + self.residual.rows64(self.rows, self.batch)
        if self.mask is not None:
            y = torch.where(self.mask.rows64(self.rows, self.batch) > 0, y, torch.zeros_like(y))
        return y, pre, c


H_ROWS = 150  # rows of the per-node tables the edge shapes gather from


def _shape(name, d, rows=300, batch=2):
    """The row ops gw_train.cu builds, on the data of generator d."""
    R = rows * batch
    if name == "hidden":  # hidden layer: K = N = 256, relu (the lean path)
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(256, 256), 256, 256, bias=d.addend(256), relu=True)
    if name == "features102":  # Linear 0 of the node encoder on the 102 raw features (K0 = 128, general path)
        return RowOp(rows, batch, [stream(d.operand(R, 102), rows)], d.weight(256, 102), 102, 256, bias=d.addend(256), relu=True)
    if name == "edge_l1_gather":  # factored edge layer 1: e W1e^T + P[src, :He] + P[dst, He:]  (W a column slice of the 768-wide W1)
        P = d.addend(batch * H_ROWS, 512)
        src = torch.randint(0, H_ROWS, (rows,), generator=d.g, device="cuda", dtype=torch.int32)
        dst = torch.randint(0, H_ROWS, (rows,), generator=d.g, device="cuda", dtype=torch.int32)
        add = (Src(GATHER, P, 256, 0, H_ROWS, src), Src(GATHER, P, 256, 256, H_ROWS, dst))
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(256, 768), 256, 256, wcol=512, bias=d.addend(256), add=add, relu=True)
    if name == "enc_l1_bgather":  # encoder edge layer 1: xg W1s^T + Pm[mesh] (batch-invariant gather) + Pe (broadcast)
        mesh = torch.randint(0, H_ROWS, (rows,), generator=d.g, device="cuda", dtype=torch.int32)
        add = (Src(BGATHER, d.addend(H_ROWS, 256), 256, 0, H_ROWS, mesh), bcast(d.addend(rows, 256)))
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(256, 768), 256, 256, wcol=0, bias=d.addend(256), add=add, relu=True)
    if name == "two_source":  # node MLP layer 1 on [x (broadcast) ; aggregate]: K0 = 512, multiplied in two windows
        a = [bcast(d.operand(rows, 256)), stream(d.operand(R, 256), rows)]
        return RowOp(rows, batch, a, d.weight(256, 512), 512, 256, bias=d.addend(256), relu=True)
    if name in ("ln_res_stream", "ln_res_bcast"):  # last layer of an MLP: LayerNorm (pre-LN value taped) + residual
        res = stream(d.addend(R, 256), rows) if name == "ln_res_stream" else bcast(d.addend(rows, 256))
        g = torch.rand(256, generator=d.g, device="cuda") + 0.5
        b = torch.randn(256, generator=d.g, device="cuda") * 0.1
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(256, 256), 256, 256, bias=d.addend(256), ln=(g, b), residual=res,
                     save_pre=True)
    if name == "out78":  # the forecast's output layer: 78 columns + the first 78 of the 102-wide features (narrow path)
        res = stream(d.addend(R, 102), rows, width=78)
        return RowOp(rows, batch, [stream(d.operand(R, 128), rows)], d.weight(78, 128), 128, 78, bias=d.addend(78), residual=res)
    if name.startswith("dgrad_mask"):  # data gradient through a ReLU: (dY W) masked by the taped activation, W^T [n_in, n_out]
        n = int(name[len("dgrad_mask"):])
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(n, 256), 256, n, mask=stream(d.relu_rows(R, n), rows))
    if name == "dgrad_add256":  # data gradient with the residual path's gradient added, and masked
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(256, 256), 256, 256, add=(stream(d.addend(R, 256), rows),),
                     mask=stream(d.relu_rows(R, 256), rows))
    if name == "dgrad_add102":
        return RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(102, 256), 256, 102, add=(stream(d.addend(R, 102), rows),))
    raise KeyError(name)


SHAPES = ["hidden", "features102", "edge_l1_gather", "enc_l1_bgather", "two_source", "ln_res_stream", "ln_res_bcast", "out78", "dgrad_mask256",
          "dgrad_mask128", "dgrad_mask102", "dgrad_add256", "dgrad_add102"]
# shapes that the launcher must send to the lean path (when GW_TC3_NOFAST is unset); every other one takes the general path
LEAN = {"hidden", "two_source", "out78"}
RUNS = [(SIMT, False), (FP32, False), (FP32, True), (BF16, False), (BF16, True)]


def _check_lean(name, prec, nofast, lean):
    if prec == SIMT:
        return []
    want = 1 if (name in LEAN and not nofast) else 0
    return [] if lean == want else [f"{name} {PREC_NAME[prec]}: lean path {lean}, expected {want}"]


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("name", SHAPES)
def test_row_op_exact(name, data):
    """Exact-integer row ops: every precision and both chain paths reproduce float64 bit for bit (LayerNorm layers: the taped
    pre-LN value bit for bit, the normalised output within 1e-5)."""
    d = Data(1000 + SHAPES.index(name), **data)
    op = _shape(name, d)
    y64, pre64, _ = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, pre, lean = op.run(prec, nofast)
        tag = f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
        fails += _check_lean(name, prec, nofast, lean)
        if op.ln is None:
            bad = (out[:, :op.N].double() != y64).sum().item()
            if bad:
                fails.append(f"{tag}: {bad} of {y64.numel()} values differ")
        else:
            if not torch.equal(pre.double(), pre64):
                fails.append(f"{tag}: pre-LayerNorm values differ")
            ef = float((out.double() - y64).norm() / y64.norm())
            if not ef < 1e-5:
                fails.append(f"{tag}: LayerNorm output eps_F {ef:.2e}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("rows,batch", [(1, 1), (1, 3), (127, 1), (127, 3), (129, 1), (129, 3)])
@pytest.mark.parametrize("name", ["hidden", "dgrad_mask102", "ln_res_bcast"])
def test_row_op_exact_row_counts(name, rows, batch):
    """Row counts around the 128-row tile (and single rows), one or three samples: bit for bit on every path."""
    d = Data(7 + rows + batch, exact=True, s=0)
    op = _shape(name, d, rows, batch)
    y64, pre64, _ = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, pre, lean = op.run(prec, nofast)
        tag = f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
        if not (torch.equal(out[:, :op.N].double(), y64) if op.ln is None else torch.equal(pre.double(), pre64)):
            fails.append(tag)
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("name", SHAPES)
def test_row_op_float(name, data):
    """Random-float row ops under the precision bars (LayerNorm layers: the pre-LN value under both bars, the normalised output
    under the eps_F bar; measured worst 3.0e-7 / 5.5e-7 / 1.9e-3 for fp32_simt / fp32 / bf16)."""
    d = Data(2000 + SHAPES.index(name), **data)
    op = _shape(name, d)
    y64, pre64, c = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, pre, lean = op.run(prec, nofast)
        fails += _check_lean(name, prec, nofast, lean)
        bf, bel = BARS[prec]
        tag = f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
        if op.ln is None:
            ef, eel = _eps(out[:, :op.N], y64, c)
        else:
            ef, eel = _eps(pre, pre64, c)
            efo = float((out.double() - y64).norm() / y64.norm())
            print(f"{tag}: LayerNorm output eps_F {efo:.2e}")
            if not efo < bf:
                fails.append(f"{tag}: LayerNorm output eps_F {efo:.2e}")
        print(f"{tag}: eps_F {ef:.2e} eps_el {eel:.2e}")
        if not (ef < bf and eel < bel):
            fails.append(f"{tag}: eps_F {ef:.2e} eps_el {eel:.2e}")
    assert not fails, fails


# ---- weight gradient ---------------------------------------------------------------------------------------------------------
def _wgrad(kind, dY, a, K, rows, batch, dW, ldw_col, db, status=None):
    """kind 'fp32' / 'bf16': gw_wgrad_tc.cu (split / not); 'simt': the CUDA-core kernel.  dW: [N, ldw] buffer, ldw_col: the
    slice's first column."""
    N = dY.shape[1]
    h = a.h()
    pw = ctypes.c_void_p(dW.data_ptr() + 4 * ldw_col)
    if kind == "simt":
        return HK.h_wgrad_simt(_p(dY), dY.shape[1], N, ctypes.byref(h), K, rows, batch, pw, dW.shape[1], _p(db), _st())
    st = status if status is not None else torch.zeros(1, dtype=torch.int32, device="cuda")
    rc = HK.h_wgrad_tc(1 if kind == "fp32" else 0, _p(dY), dY.shape[1], N, ctypes.byref(h), K, rows, batch, pw, dW.shape[1], _p(db), _p(st), _st())
    if status is None and rc == 0:
        torch.cuda.synchronize()
        assert int(st.item()) == 0, f"status word {int(st.item())}"
    return rc


WG_KINDS = ["fp32", "bf16", "simt"]
# (R as rows x batch, N, K, A kind, A's first column)
WG_SHAPES = {
    "r1": (1, 1, 128, 128, STREAM, 0),
    "r63": (63, 1, 200, 102, STREAM, 0),
    "r64": (64, 1, 256, 256, STREAM, 0),
    "r65": (65, 1, 78, 78, STREAM, 0),
    "idle_ctas": (64 * 133 + 5, 1, 256, 128, STREAM, 0),  # 134 chunks over 132 row ranges: the trailing CTAs get none
    "samples_stream": (77, 3, 128, 256, STREAM, 0),      # 64-row chunks straddle the samples
    "samples_bcast": (77, 3, 200, 102, BCAST, 0),
    "col0": (300, 2, 256, 78, STREAM, 40),               # A is a column window of wider rows
    "n200_k256": (1000, 1, 200, 256, STREAM, 0),         # N > 128: a second o-block
    "many_partials": (500_000, 2, 128, 102, STREAM, 0),  # ~1.0e6 rows
    # the top of gw_wgrad_tc.cu's design range: the decoder's edges at 1 degree, batch 8 (3.63e6 rows); N = 256 leaves 66 row
    # ranges of ~55 000 rows.  Summed in one wgmma accumulator each, fp32 mode measured eps_F 1.9e-4; since each accumulator
    # sums at most 2048 rows into the CTA's fp32 partial, 7.3e-6 (many_partials: 3.2e-5 -> 6.9e-6)
    "dec_edges_1deg_b8": (453_600, 8, 256, 256, STREAM, 0),
}


def _wg_case(name, d):
    rows, batch, N, K, kind, col0 = WG_SHAPES[name]
    dY = d.operand(rows * batch, N, outlier=False)  # (the outlier column is one of A's: a column of dW, not a single sum)
    if kind == STREAM:
        a = Src(STREAM, d.operand(rows * batch, col0 + K + (3 if col0 else 0)), K, col0, rows)
    else:
        a = Src(BCAST, d.operand(rows, K), K)
    return rows, batch, N, K, dY, a


def _wg_ref(rows, batch, dY, a, block=1 << 18):
    """float64 dW, db and |dY|^T |A|.  A streamed A is taken `block` rows at a time, so that float64 copies of dY and A (7.4 GB
    each at 3.63e6 x 256) never exist whole."""
    if a.kind != STREAM:
        A = a.rows64(rows, batch)
        Y = dY.double()
        return Y.T @ A, Y.sum(0), Y.abs().T @ A.abs()
    assert a.src_rows == rows, "row r of a streamed A is row r of t only when samples are rows apart"
    N, R = dY.shape[1], rows * batch
    g = torch.zeros(N, a.width, dtype=torch.float64, device="cuda")
    b, c = torch.zeros(N, dtype=torch.float64, device="cuda"), torch.zeros_like(g)
    for r0 in range(0, R, block):
        A = a.t[r0:r0 + block, a.col0:a.col0 + a.width].double()  # STREAM: row r of A is row r of t
        Y = dY[r0:r0 + block].double()
        g += Y.T @ A
        b += Y.sum(0)
        c += Y.abs().T @ A.abs()
    return g, b, c


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("name", list(WG_SHAPES))
def test_wgrad_exact(name, data):
    """dW += dY^T A and db += colsum(dY), exact integers: bit for bit, also written into a column slice of a wider prefilled
    gradient (ldw = 768, offsets 256 / 512) that must be untouched outside the slice."""
    d = Data(3000 + list(WG_SHAPES).index(name), **data)
    rows, batch, N, K, dY, a = _wg_case(name, d)
    g64, b64, _ = _wg_ref(rows, batch, dY, a)
    fails = []
    for kind in WG_KINDS:
        for col in (256, 512) if name in ("r64", "samples_bcast") else (0,):
            ldw = 768 if col else K
            dW = d.addend(N, ldw)  # prefilled on the results' grids: prefill + gradient stays exact
            db = d.operand(N)
            dW0, db0 = dW.clone(), db.clone()
            _ok(_wgrad(kind, dY, a, K, rows, batch, dW, col, db))
            torch.cuda.synchronize()
            tag = f"{name} {kind} col {col}"
            got = dW[:, col:col + K].double()
            want = dW0[:, col:col + K].double() + g64
            if not torch.equal(got, want):
                fails.append(f"{tag}: {(got != want).sum().item()} of {got.numel()} dW values differ")
            if not torch.equal(db.double(), db0.double() + b64):
                fails.append(f"{tag}: {(db.double() != db0.double() + b64).sum().item()} of {N} db values differ")
            outside = torch.ones_like(dW, dtype=torch.bool)
            outside[:, col:col + K] = False
            if not torch.equal(dW[outside].view(torch.int32), dW0[outside].view(torch.int32)):
                fails.append(f"{tag}: values outside the slice changed")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("name", ["r65", "idle_ctas", "samples_bcast", "col0", "n200_k256", "many_partials", "dec_edges_1deg_b8"])
def test_wgrad_float(name, data):
    d = Data(4000 + list(WG_SHAPES).index(name), **data)
    rows, batch, N, K, dY, a = _wg_case(name, d)
    g64, b64, c = _wg_ref(rows, batch, dY, a)
    fails = []
    for kind in WG_KINDS:
        dW = torch.zeros(N, K, device="cuda")
        db = torch.zeros(N, device="cuda")
        _ok(_wgrad(kind, dY, a, K, rows, batch, dW, 0, db))
        torch.cuda.synchronize()
        bf, bel = BARS[{"fp32": FP32, "bf16": BF16, "simt": SIMT}[kind]]
        ef, eel = _eps(dW, g64, c)
        efb, eelb = _eps(db, b64, dY.abs().sum(0, dtype=torch.float64))
        print(f"{name} {kind}: dW eps_F {ef:.2e} eps_el {eel:.2e}  db eps_F {efb:.2e} eps_el {eelb:.2e}")
        if not (ef < bf and eel < bel):
            fails.append(f"{name} {kind}: dW eps_F {ef:.2e} eps_el {eel:.2e}")
        if not eelb < 1e-6:  # an fp32 column sum on every path (measured worst 8.7e-8)
            fails.append(f"{name} {kind}: db eps_el {eelb:.2e}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("kind", ["fp32", "bf16"])
def test_wgrad_tc_no_bias_zero_and_repeatable(kind):
    """db = nullptr (nothing else written), all-zero dY (exact zeros) and two calls giving bit-identical results."""
    d = Data(5, exact=False)
    rows, batch, N, K = 20_000, 2, 256, 256
    dY = d.operand(rows * batch, N)
    a = stream(d.operand(rows * batch, K), rows)
    dW = torch.full((N, 768), 5.0, device="cuda")
    _ok(_wgrad(kind, dY, a, K, rows, batch, dW, 256, None))
    first = dW.clone()
    dW.fill_(5.0)
    _ok(_wgrad(kind, dY, a, K, rows, batch, dW, 256, None))
    torch.cuda.synchronize()
    assert torch.equal(dW.view(torch.int32), first.view(torch.int32)), "weight gradient is not repeatable"
    assert torch.all(dW[:, :256] == 5.0) and torch.all(dW[:, 512:] == 5.0)
    dW = torch.zeros(N, K, device="cuda")
    db = torch.zeros(N, device="cuda")
    _ok(_wgrad(kind, torch.zeros_like(dY), a, K, rows, batch, dW, 0, db))
    torch.cuda.synchronize()
    assert torch.all(dW == 0) and torch.all(db == 0)


@gpu
def test_wgrad_tc_nan_sets_status():
    """A NaN in dY: the fp32-faithful weight gradient flags status bit 3 (value 8) and the launch still returns success."""
    d = Data(6, exact=False)
    rows, N, K = 1000, 128, 128
    dY = d.operand(rows, N)
    dY[517, 33] = float("nan")
    a = stream(d.operand(rows, K), rows)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    dW = torch.zeros(N, K, device="cuda")
    _ok(_wgrad("fp32", dY, a, K, rows, 1, dW, 0, None, status=status))
    torch.cuda.synchronize()
    assert int(status.item()) & 8, f"status word {int(status.item())}"


# ---- memory-bound primitives --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("offset", [0.0, 1000.0])
@pytest.mark.parametrize("N", [78, 128, 256])
def test_ln_bwd(N, offset):
    """LayerNorm backward against float64 autograd of layer_norm(eps=1e-5); dgamma / dbeta accumulate into prefilled buffers."""
    g = torch.Generator(device="cuda").manual_seed(N)
    R = 3001
    z = torch.randn(R, N, generator=g, device="cuda") + offset
    dy = torch.randn(R, N, generator=g, device="cuda")
    gamma = torch.rand(N, generator=g, device="cuda") + 0.5
    beta = torch.randn(N, generator=g, device="cuda")
    dg0, db0 = torch.randn(N, generator=g, device="cuda"), torch.randn(N, generator=g, device="cuda")
    dg, dbt = dg0.clone(), db0.clone()
    dz = torch.full_like(z, float("nan"))
    _ok(HK.h_ln_bwd(_p(dy), N, _p(z), N, N, _p(gamma), R, _p(dz), N, _p(dg), _p(dbt), _st()))
    torch.cuda.synchronize()
    with torch.enable_grad():
        z64 = z.double().requires_grad_()
        g64 = gamma.double().requires_grad_()
        b64 = beta.double().requires_grad_()
        y = torch.nn.functional.layer_norm(z64, (N,), g64, b64, eps=1e-5)
        y.backward(dy.double())
    ez = float((dz.double() - z64.grad).norm() / z64.grad.norm())
    eg = float((dg.double() - dg0.double() - g64.grad).norm() / g64.grad.norm())
    eb = float((dbt.double() - db0.double() - b64.grad).norm() / b64.grad.norm())
    print(f"ln_bwd N {N} offset {offset}: dz {ez:.2e} dgamma {eg:.2e} dbeta {eb:.2e}")
    # measured worst: dz 7.0e-8 / 8.0e-6, dgamma 3.8e-7 / 4.9e-5 (offset 0 / 1000: fp32 statistics of rows far from zero), dbeta 4.1e-7
    bar = 2e-6 if offset == 0.0 else 2e-4
    assert ez < bar and eg < bar and eb < 2e-6, (ez, eg, eb)


def _csr(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)


def _seq_sum(rows_f32):  # sequential float32 sum, first row first
    if rows_f32.shape[0] == 0:
        return np.zeros(rows_f32.shape[1], np.float32)
    return np.cumsum(rows_f32, axis=0, dtype=np.float32)[-1]


@gpu
@pytest.mark.parametrize("use_perm", [False, True])
def test_segsum(use_perm):
    """Per-segment sums (CSR, optional edge permutation, empty segments, 3 samples): bit for bit a sequential float32 sum."""
    rng = np.random.Generator(np.random.PCG64(11))
    lengths = rng.integers(0, 9, 200)
    lengths[[3, 50, 51, 199]] = 0
    lengths[10] = 700
    ptr = _csr(lengths)
    E, S, B, W = int(ptr[-1]), len(lengths), 3, 128
    base = rng.standard_normal((B * E, 256)).astype(np.float32)
    perm = rng.permutation(E).astype(np.int32) if use_perm else None
    out = torch.full((B * S, W), float("nan"), device="cuda")
    tb = torch.from_numpy(base).cuda()
    tp = torch.from_numpy(ptr).cuda()
    tperm = torch.from_numpy(perm).cuda() if use_perm else None
    _ok(HK.h_segsum(_p(tb), 256, W, _p(tp), _p(tperm), E, S, B, _p(out), W, _st()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for b in range(B):
        for i in range(S):
            e = np.arange(ptr[i], ptr[i + 1])
            e = perm[e] if use_perm else e
            want = _seq_sum(base[b * E + e, :W])
            assert np.array_equal(got[b * S + i], want), f"sample {b} segment {i} (length {lengths[i]})"


@gpu
@pytest.mark.parametrize("use_perm", [False, True])
def test_segsum_chunked(use_perm):
    """The two-level segment sum: each segment is cut into 64-row chunks from its first row, each chunk summed sequentially from
    zero, then the chunk sums added in order -- bit for bit.  Segments of 0, 1, 64, 65 and 5000 rows."""
    rng = np.random.Generator(np.random.PCG64(12))
    lengths = np.array([0, 1, 64, 65, 5000, 3, 0, 128, 129, 63, 2, 1], dtype=np.int64)
    ptr = _csr(lengths)
    E, S, B = int(ptr[-1]), len(lengths), 3
    base = rng.standard_normal((B * E, 256)).astype(np.float32)
    perm = rng.permutation(E).astype(np.int32) if use_perm else None
    out = torch.full((B * S, 256), float("nan"), device="cuda")
    tb = torch.from_numpy(base).cuda()
    tp = torch.from_numpy(ptr).cuda()
    tperm = torch.from_numpy(perm).cuda() if use_perm else None
    _ok(HK.h_segsum_chunked(_p(tb), 256, _p(tp), _p(tperm), E, S, E, B, _p(out), 256, _st()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for b in range(B):
        for i in range(S):
            e = np.arange(ptr[i], ptr[i + 1])
            e = perm[e] if use_perm else e
            parts = [_seq_sum(base[b * E + e[j:j + 64]]) for j in range(0, max(len(e), 1), 64)]
            want = parts[0] if len(parts) == 1 else _seq_sum(np.stack(parts))
            assert np.array_equal(got[b * S + i], want), f"sample {b} segment {i} (length {lengths[i]})"


@gpu
@pytest.mark.parametrize("accumulate", [False, True])
def test_batch_reduce_and_gather_rows(accumulate):
    """out (+)= sum over the samples (batch order), and out (+)= in[sample, idx[row]]: bit for bit."""
    rng = np.random.Generator(np.random.PCG64(13))
    rows, width, B, src_rows = 1001, 102, 3, 257
    x = rng.standard_normal((B * rows, 104)).astype(np.float32)
    o0 = rng.standard_normal((rows, 108)).astype(np.float32)
    out = torch.from_numpy(o0).cuda()
    tx = torch.from_numpy(x).cuda()  # (every device input stays referenced until the kernel has run)
    _ok(HK.h_batch_reduce(_p(tx), 104, rows, width, B, _p(out), 108, int(accumulate), _st()))
    torch.cuda.synchronize()
    want = o0.copy()
    acc = o0[:, :width].copy() if accumulate else np.zeros((rows, width), np.float32)
    for b in range(B):
        acc = acc + x[b * rows:(b + 1) * rows, :width]
    want[:, :width] = acc
    assert np.array_equal(out.cpu().numpy(), want)

    tin = rng.standard_normal((B * src_rows, 132)).astype(np.float32)
    idx = rng.integers(0, src_rows, rows).astype(np.int32)
    g0 = rng.standard_normal((B * rows, 128)).astype(np.float32)
    gout = torch.from_numpy(g0).cuda()
    ttin, tidx = torch.from_numpy(tin).cuda(), torch.from_numpy(idx).cuda()
    _ok(HK.h_gather_rows(_p(ttin), 132, src_rows, _p(tidx), rows, 128, B, _p(gout), 128, int(accumulate), _st()))
    torch.cuda.synchronize()
    src = tin[(np.arange(B)[:, None] * src_rows + idx[None, :]).reshape(-1), :128]
    assert np.array_equal(gout.cpu().numpy(), g0 + src if accumulate else src)


@gpu
@pytest.mark.parametrize("rows,cols", [(256, 768), (78, 128), (256, 102)])
def test_transpose(rows, cols):
    W = torch.randn(rows, cols, device="cuda")
    WT = torch.full((cols, rows), float("nan"), device="cuda")
    _ok(HK.h_transpose(_p(W), rows, cols, _p(WT), _st()))
    torch.cuda.synchronize()
    assert torch.equal(WT, W.T)


@gpu
@pytest.mark.parametrize("with_scale_dev", [False, True])
@pytest.mark.parametrize("with_inv_var", [False, True])
def test_normalized_mse_loss_grad(with_inv_var, with_scale_dev):
    """grad = (*scale_dev) * scale * node_weight[n] * 2 (pred - target) * inv_variance[f] / F   (include/gw_b200.h)."""
    from graph_weather_b200 import _capi

    lib = _capi.load()
    g = torch.Generator(device="cuda").manual_seed(3)
    B, Nn, F = 2, 1003, 78
    pred = torch.randn(B, Nn, F, generator=g, device="cuda")
    target = torch.randn(B, Nn, F, generator=g, device="cuda")
    w = torch.rand(Nn, generator=g, device="cuda")
    iv = torch.rand(F, generator=g, device="cuda") + 0.5 if with_inv_var else None
    sd = torch.tensor([0.37], device="cuda") if with_scale_dev else None
    scale = 1.0 / (B * Nn)
    grad = torch.full_like(pred, float("nan"))
    _capi._check(lib.gw_normalized_mse_loss_grad(_p(pred), _p(target), _p(iv), _p(w), B, Nn, F, _p(sd), ctypes.c_float(scale), _p(grad), _st()))
    torch.cuda.synchronize()
    want = (pred.double() - target.double()) * 2.0 / F * scale * w.double()[None, :, None]
    if with_inv_var:
        want = want * iv.double()
    if with_scale_dev:
        want = want * 0.37
    err = float(((grad.double() - want).abs() / want.abs().clamp_min(1e-30)).max())
    print(f"loss grad: max relative error {err:.2e}")
    assert err < 1e-6, err  # measured worst 2.3e-7
