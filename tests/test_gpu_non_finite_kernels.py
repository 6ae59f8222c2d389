"""-m gpu: NaN, +inf and -inf inputs through the CUDA primitives, one at a time, against float64 torch.

ERA5's sea-surface fields are NaN over land, so non-finite values are ordinary data.  The contract (README, "Non-finite inputs"):
  * the exact-fp32 CUDA-core row op (fp32_simt) and the training step's memory-bound kernels propagate NaN and +-inf as torch
    does: torch.relu keeps a NaN (and -0.0), and a ReLU's backward zeroes the gradient only where the taped activation is <= 0
    (threshold_backward), so a NaN activation passes its gradient through;
  * the tensor-core chains (fp32, bf16) refuse non-finite operands, weights, biases and LayerNorm parameters: status bit 3
    (value 8), return code 0, nothing written outside the stored rows x columns, and the next clean launch is unaffected.

One non-finite value is placed at a time, in an entry the operation reads.  The data are the exact integers of
test_gpu_kernels.py, so every finite result of a row op must match float64 bit for bit (LayerNorm outputs: the pre-LayerNorm value
bit for bit, the normalised value within 1e-5).  The float64 reference is written here with torch's semantics and does not reuse
RowOp.ref, whose mask keeps `mask > 0`."""
import ctypes

import pytest
import torch

import test_gpu_forward_simt as fs
import test_gpu_kernels as tk
from test_gpu_kernels import BCAST, BF16, BGATHER, FP32, GATHER, GBR, SEGSUM, SIMT, STREAM, Data, HChain, HOp, HSrc, _a, _ok, _p, _st

VALUES = {"nan": float("nan"), "inf": float("inf"), "-inf": float("-inf")}
SENTINEL = 1234.5  # finite prefill: a NaN prefill could not show a stray NaN store


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    tk.HK = tk._compile_harness(tmp_path_factory.mktemp("gw_non_finite_harness"))  # (the helpers of test_gpu_kernels call through it)
    return tk.HK


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


def _close_fails(got, want, tag, rel=0.0):
    """NaN where want is NaN, +-inf where want is +-inf (same sign), finite entries equal (rel = 0) or within rel of max |want|."""
    got = got.double()
    fails = []
    if not torch.equal(torch.isnan(got), torch.isnan(want)):
        fails.append(f"{tag}: NaN at {int((torch.isnan(got) != torch.isnan(want)).sum())} entries where float64 torch differs")
    for f in (torch.isposinf, torch.isneginf):
        if not torch.equal(f(got), f(want)):
            fails.append(f"{tag}: {f.__name__[2:]} at {int((f(got) != f(want)).sum())} entries where float64 torch differs")
    fin = torch.isfinite(got) & torch.isfinite(want)
    if bool(fin.any()):
        err = float((got[fin] - want[fin]).abs().max())
        if not err <= rel * float(want[fin].abs().max()):
            fails.append(f"{tag}: finite entries differ by up to {err:.3e}")
    return fails


# ---- the CUDA-core row op ------------------------------------------------------------------------------------------------------
def _ref64(op):
    """float64 (out, pre-LayerNorm value) of a RowOp with torch's semantics: torch.relu, and the mask zeroes where mask <= 0."""
    A = torch.cat([s.rows64(op.rows, op.batch) for s in op.a], dim=1)
    y = A @ op.W[:, op.wcol:op.wcol + op.K].double().T
    if op.bias is not None:
        y = y + op.bias.double()
    for s in op.add:
        y = y + s.rows64(op.rows, op.batch)
    if op.relu:
        y = torch.relu(y)
    pre = y
    if op.ln is not None:
        y = torch.nn.functional.layer_norm(y, (op.N,), op.ln[0].double(), op.ln[1].double(), eps=1e-5)
    if op.residual is not None:
        y = y + op.residual.rows64(op.rows, op.batch)
    if op.mask is not None:
        y = torch.where(op.mask.rows64(op.rows, op.batch) <= 0, torch.zeros_like(y), y)
    return y, pre


def _hop(op, out, pre, ocol):
    h = HOp()
    h.rows, h.batch = op.rows, op.batch
    for j, s in enumerate(op.a):
        h.a[j] = s.h()
    h.W = op.W.data_ptr() + 4 * op.wcol
    h.K, h.N, h.ldw = op.K, op.N, op.W.shape[1]
    h.bias = _a(op.bias)
    for j, s in enumerate(op.add):
        h.add[j] = s.h()
    h.relu = int(op.relu)
    if op.ln is not None:
        h.ln_g, h.ln_b = _a(op.ln[0]), _a(op.ln[1])
    if op.residual is not None:
        h.residual = op.residual.h()
    h.out, h.ldo = out.data_ptr() + 4 * ocol, op.ldo
    h.save_pre = pre.data_ptr() + 4 * ocol if pre is not None else None
    if op.mask is not None:
        h.mask = op.mask.h()
    return h


def _simt_fails(op, tag):
    """Runs op on the CUDA cores into SENTINEL-prefilled buffers (two spare rows) and compares it with _ref64."""
    R, ocol = op.rows * op.batch, getattr(op, "ocol", 0)
    out = torch.full((R + 2, op.ldo), SENTINEL, device="cuda")
    pre = torch.full((R + 2, op.ldo), SENTINEL, device="cuda") if op.save_pre else None
    h = _hop(op, out, pre, ocol)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    _ok(tk.HK.h_row_op(SIMT, ctypes.byref(h), None, _p(status), _st()))
    torch.cuda.synchronize()
    y64, pre64 = _ref64(op)
    fails = [] if int(status.item()) == 0 else [f"{tag}: status word {int(status.item())}"]
    if op.ln is None:
        fails += _close_fails(out[:R, ocol:ocol + op.N], y64, tag)
    else:
        fails += _close_fails(pre[:R, ocol:ocol + op.N], pre64, tag + " pre-LayerNorm")
        fails += _close_fails(out[:R, ocol:ocol + op.N], y64, tag + " LayerNorm output", rel=1e-5)
    for name, buf in (("out", out), ("save_pre", pre)):
        if buf is None:
            continue
        outside = torch.ones_like(buf, dtype=torch.bool)
        outside[:R, ocol:ocol + op.N] = False
        if not bool((buf[outside] == SENTINEL).all()):
            fails.append(f"{tag}: {name} written outside the stored rows / columns")
    return fails


def _pick(g, n):
    return int(torch.randint(0, n, (1,), generator=g))


def _src_entries(s, rows, batch, g):
    """[(tensor, index)] of one entry the row source reads (GBR: one of the gathered table and one of the broadcast table)."""
    b, i, c = _pick(g, batch), _pick(g, rows), s.col0 + _pick(g, s.width)
    if s.kind == STREAM:
        r = b * s.src_rows + i
    elif s.kind == BCAST:
        r = i
    elif s.kind in (GATHER, GBR):
        r = b * s.src_rows + int(s.idx[i])
    elif s.kind == BGATHER:
        r = int(s.idx[i])
    elif s.kind == SEGSUM:  # an edge row that belongs to a segment
        j = _pick(g, int(s.ptr[-1]))
        r = b * s.src_rows + (int(s.perm[j]) if s.perm is not None else j)
    else:
        raise KeyError(s.kind)
    out = [(s.t, (r, c))]
    if s.kind == GBR:
        out.append((s.t2, (i, _pick(g, s.width))))
    return out


KIND_NAME = {STREAM: "stream", BCAST: "bcast", GATHER: "gather", BGATHER: "bgather", SEGSUM: "segsum", GBR: "gbr"}


def _slots(op, g):
    """(slot name, tensor, index) of every input of op that can hold the non-finite value."""
    out = []
    for j, s in enumerate(op.a):
        for k, (t, ix) in enumerate(_src_entries(s, op.rows, op.batch, g)):
            out.append((f"a{j}:{KIND_NAME[s.kind]}{'.t2' if k else ''}", t, ix))
    out.append(("W", op.W, (_pick(g, op.N), op.wcol + _pick(g, op.K))))
    if op.bias is not None:
        out.append(("bias", op.bias, (_pick(g, op.N),)))
    for j, s in enumerate(op.add):
        for t, ix in _src_entries(s, op.rows, op.batch, g):
            out.append((f"add{j}:{KIND_NAME[s.kind]}", t, ix))
    if op.residual is not None:
        for t, ix in _src_entries(op.residual, op.rows, op.batch, g):
            out.append((f"residual:{KIND_NAME[op.residual.kind]}", t, ix))
    if op.mask is not None:  # where the taped activation is 0: the old `mask > 0` and torch's `mask <= 0` disagree on a NaN there
        m = op.mask
        R = op.batch * m.src_rows
        z = (m.t[:R, m.col0:m.col0 + m.width] <= 0).nonzero()
        r, c = z[_pick(g, z.shape[0])].tolist()
        out.append(("mask", m.t, (r, m.col0 + c)))
    return out


SIMT_CASES = [pytest.param("train", n, id=f"train-{n}") for n in tk.SHAPES] + [pytest.param("fwd", n, id=f"fwd-{n}") for n in fs.VARIANTS]


@gpu
@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("where,name", SIMT_CASES)
def test_simt_row_op_non_finite(where, name, value):
    """Every row op the training step (test_gpu_kernels._shape) and the forward (test_gpu_forward_simt.variant, 256 wide) run on
    the CUDA cores, with one NaN / +inf / -inf in each input in turn: NaN and +-inf exactly where float64 torch has them, every
    finite entry bit for bit, nothing stored outside the output rows x columns, status 0."""
    seed = 9000 + (tk.SHAPES.index(name) if where == "train" else 100 + fs.VARIANTS.index(name))
    d = Data(seed, exact=True, s=0)
    ops = [tk._shape(name, d)] if where == "train" else fs.variant(name, d, fs.WIDTHS["w256"])
    g = torch.Generator().manual_seed(seed)
    v = VALUES[value]
    fails = []
    for k, op in enumerate(ops):
        for slot, t, ix in _slots(op, g):
            old = t[ix].clone()
            t[ix] = v
            try:
                fails += _simt_fails(op, f"{name}[{k}] {value} in {slot}")
            finally:
                t[ix] = old
    assert not fails, fails


@gpu
def test_simt_relu_and_mask_semantics():
    """The case of the contract spelled out on one row: relu([nan, -0., -1, 2, inf, -inf]) = [nan, -0., 0, 2, inf, 0] (sign of
    zero included), and a gradient of ones masked by that activation is [1, 0, 0, 1, 1, 0]."""
    v = torch.tensor([float("nan"), -0.0, -1.0, 2.0, float("inf"), float("-inf")], device="cuda")
    n = v.numel()
    eye = torch.eye(n, device="cuda")
    out = torch.full((1, n), SENTINEL, device="cuda")
    op = tk.RowOp(1, 1, [tk.stream(torch.ones(1, 1, device="cuda"), 1)], torch.zeros(n, 1, device="cuda"), 1, n,
                  add=(tk.stream(v[None, :].clone(), 1),), relu=True)  # fmt: skip
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    _ok(tk.HK.h_row_op(SIMT, ctypes.byref(_hop(op, out, None, 0)), None, _p(status), _st()))
    act = torch.relu(v)
    torch.cuda.synchronize()
    assert torch.equal(out[0].view(torch.int32).cpu()[1:], act.view(torch.int32).cpu()[1:]) and bool(torch.isnan(out[0, 0])), out
    grad = torch.full((1, n), SENTINEL, device="cuda")
    op = tk.RowOp(1, 1, [tk.stream(torch.ones(1, n, device="cuda"), 1)], eye, n, n, mask=tk.stream(act[None, :].clone(), 1))
    _ok(tk.HK.h_row_op(SIMT, ctypes.byref(_hop(op, grad, None, 0)), None, _p(status), _st()))
    torch.cuda.synchronize()
    assert grad[0].tolist() == [1.0, 0.0, 0.0, 1.0, 1.0, 0.0], grad


# ---- memory-bound primitives ---------------------------------------------------------------------------------------------------
def _ints(g, *shape):
    return torch.randint(-3, 4, shape, generator=g, device="cuda").float()


@gpu
@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("slot", ["dY", "A"])
def test_wgrad_simt_non_finite(slot, value):
    """dW = dY^T A and db = colsum(dY) on the CUDA cores with one non-finite entry in dY or A: equal to float64, NaN and +-inf
    included (a row of two samples straddles nothing: 77 rows x 3 samples, K = 102, N = 128)."""
    g = torch.Generator(device="cuda").manual_seed(31)
    rows, batch, N, K = 77, 3, 128, 102
    dY, A = _ints(g, rows * batch, N), _ints(g, rows * batch, K)
    (dY if slot == "dY" else A)[100, 17] = VALUES[value]
    dW, db = torch.zeros(N, K, device="cuda"), torch.zeros(N, device="cuda")
    _ok(tk._wgrad("simt", dY, tk.stream(A, rows), K, rows, batch, dW, 0, db))
    torch.cuda.synchronize()
    fails = _close_fails(dW, dY.double().T @ A.double(), "dW") + _close_fails(db, dY.double().sum(0), "db")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("slot", ["dy", "z", "gamma"])
@pytest.mark.parametrize("N", [78, 256])
def test_ln_bwd_non_finite(N, slot, value):
    """LayerNorm backward with one non-finite entry in dy, z or gamma: dz, dgamma and dbeta NaN / +-inf exactly where float64
    autograd has them, finite entries within 2e-6 of max |value| (test_gpu_kernels.test_ln_bwd's bar)."""
    g = torch.Generator(device="cuda").manual_seed(N + 1)
    R = 301
    z, dy = torch.randn(R, N, generator=g, device="cuda"), torch.randn(R, N, generator=g, device="cuda")
    gamma = torch.rand(N, generator=g, device="cuda") + 0.5
    {"dy": dy, "z": z, "gamma": gamma[None, :]}[slot][-1 if slot == "gamma" else 150, N // 3] = VALUES[value]
    dz = torch.full_like(z, SENTINEL)
    dg, dbt = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    _ok(tk.HK.h_ln_bwd(_p(dy), N, _p(z), N, N, _p(gamma), R, _p(dz), N, _p(dg), _p(dbt), _st()))
    torch.cuda.synchronize()
    with torch.enable_grad():
        z64, g64 = z.double().requires_grad_(), gamma.double().requires_grad_()
        b64 = torch.zeros(N, dtype=torch.float64, device="cuda", requires_grad=True)
        torch.nn.functional.layer_norm(z64, (N,), g64, b64, eps=1e-5).backward(dy.double())
    fails = _close_fails(dz, z64.grad, "dz", 2e-6) + _close_fails(dg, g64.grad, "dgamma", 2e-6) + _close_fails(dbt, b64.grad, "dbeta", 2e-6)
    assert not fails, fails


@gpu
@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("use_perm", [False, True])
def test_segsum_non_finite(use_perm, value):
    """Per-segment sums with one non-finite edge row entry (CSR, optional permutation, empty segments, 3 samples): equal to the
    float64 sums, NaN and +-inf included."""
    g = torch.Generator(device="cuda").manual_seed(41)
    lengths = torch.randint(0, 9, (200,), generator=g, device="cuda")
    lengths[[3, 50, 199]] = 0
    ptr = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), lengths.cumsum(0)]).int()
    E, S, B, W = int(ptr[-1]), 200, 3, 128
    base = _ints(g, B * E, 256)
    perm = torch.randperm(E, generator=g, device="cuda").int() if use_perm else None
    j = int(ptr[100]) if int(lengths[100]) else int(ptr[101])  # an edge of a non-empty segment
    base[E + (int(perm[j]) if use_perm else j), 5] = VALUES[value]
    out = torch.full((B * S + 1, W), SENTINEL, device="cuda")
    _ok(tk.HK.h_segsum(_p(base), 256, W, _p(ptr), _p(perm), E, S, B, _p(out), W, _st()))
    torch.cuda.synchronize()
    src = tk.Src(SEGSUM, base, W, 0, E, ptr=ptr, perm=perm)
    fails = _close_fails(out[:B * S], src.rows64(S, B), "segsum")
    assert bool((out[B * S] == SENTINEL).all()), "a row past the output was written"
    assert not fails, fails


@gpu
@pytest.mark.parametrize("value", list(VALUES))
def test_gather_rows_and_batch_reduce_non_finite(value):
    """out = in[sample, idx[row]] and out = sum over the samples, with one non-finite input entry: equal to float64."""
    g = torch.Generator(device="cuda").manual_seed(43)
    rows, B, src_rows = 1001, 3, 257
    tin = _ints(g, B * src_rows, 132)
    idx = torch.randint(0, src_rows, (rows,), generator=g, device="cuda", dtype=torch.int32)
    tin[src_rows + int(idx[500]), 7] = VALUES[value]
    gout = torch.full((B * rows, 128), SENTINEL, device="cuda")
    _ok(tk.HK.h_gather_rows(_p(tin), 132, src_rows, _p(idx), rows, 128, B, _p(gout), 128, 0, _st()))
    x = _ints(g, B * rows, 104)
    x[rows + 321, 11] = VALUES[value]
    rout = torch.full((rows, 108), SENTINEL, device="cuda")
    _ok(tk.HK.h_batch_reduce(_p(x), 104, rows, 102, B, _p(rout), 108, 0, _st()))
    torch.cuda.synchronize()
    gather64 = tk.Src(GATHER, tin, 128, 0, src_rows, idx).rows64(rows, B)
    reduce64 = x[:, :102].double().reshape(B, rows, 102).sum(0)
    fails = _close_fails(gout, gather64, "gather_rows") + _close_fails(rout[:, :102], reduce64, "batch_reduce")
    assert bool((rout[:, 102:] == SENTINEL).all()), "batch_reduce wrote outside its columns"
    assert not fails, fails


# ---- the tensor-core guard -------------------------------------------------------------------------------------------------------
NT = 150  # rows of the tables the gathers read


def _hs(kind, t, src_rows=0, idx=None, t2=None):
    return HSrc(kind, 256, t.shape[1], 0, t.data_ptr(), src_rows, _a(idx), _a(t2), t2.shape[1] if t2 is not None else 0, None, None, None)


class GuardChain:
    """A two-layer inference chain over one stage-0 source kind (or two sources):
         h   = relu(A W0^T + b0 + add)                       (add: a broadcast addend)
         out = LN(h W1^T + b1; gamma, beta) + residual       (residual: per-sample rows)
    stored into the first 256 of 264 columns of a SENTINEL-prefilled buffer with two spare rows.  Exact-integer data."""

    def __init__(self, kind, rows=300, batch=2):
        g = torch.Generator(device="cuda").manual_seed(77 + kind if isinstance(kind, int) else 99)
        R = rows * batch
        self.rows, self.batch, self.kind = rows, batch, kind
        idx = torch.randint(0, NT, (rows,), generator=g, device="cuda", dtype=torch.int32)
        self.t = {}  # every input tensor, by slot name
        if kind == "second":
            self.t["a0"], self.t["a1"] = _ints(g, R, 256), _ints(g, rows, 256)
            self.a0 = [_hs(STREAM, self.t["a0"], rows), _hs(BCAST, self.t["a1"])]
            self.reads = {"a0": (lambda: (R - 1, 3)), "a1": (lambda: (rows // 2, 200))}
        else:
            tab = {STREAM: (R, rows), BCAST: (rows, 0), GATHER: (batch * NT, NT), BGATHER: (NT, NT), GBR: (batch * NT, NT)}[kind]
            self.t["a0"] = _ints(g, tab[0], 256)
            if kind == GBR:
                self.t["a0.t2"] = _ints(g, rows, 256)
            self.a0 = [_hs(kind, self.t["a0"], tab[1], idx if kind in (GATHER, BGATHER, GBR) else None, self.t.get("a0.t2"))]
            r0 = {STREAM: R - 1, BCAST: rows - 1, GATHER: NT + int(idx[7]), BGATHER: int(idx[7]), GBR: NT + int(idx[7])}[kind]
            self.reads = {"a0": (lambda: (r0, 100))}
            if kind == GBR:
                self.reads["a0.t2"] = lambda: (7, 100)
        self.K0 = 512 if kind == "second" else 256
        self.idx = idx
        W0 = torch.zeros(256, self.K0, device="cuda")  # sparse +-1 weights keep the exact integers small
        W0.scatter_add_(1, torch.randint(0, self.K0, (256, 2), generator=g, device="cuda"), _ints(g, 256, 2).sign())
        W1 = torch.zeros(256, 256, device="cuda")
        W1.scatter_add_(1, torch.randint(0, 256, (256, 2), generator=g, device="cuda"), _ints(g, 256, 2).sign())
        self.t.update(W0=W0, W1=W1, b0=_ints(g, 1, 256), b1=_ints(g, 1, 256), add=_ints(g, rows, 256), res=_ints(g, R, 256),
                      gamma=torch.zeros(1, 256, device="cuda"), beta=_ints(g, 1, 256))  # fmt: skip
        self.reads.update(W0=lambda: (5, 3), W1=lambda: (9, 4), b0=lambda: (0, 17),
                          b1=lambda: (0, 18), add=lambda: (3, 40), res=lambda: (R - 2, 41), gamma=lambda: (0, 42), beta=lambda: (0, 43))  # fmt: skip

    def run(self, prec):
        """-> (return code, status word, output buffer)"""
        R = self.rows * self.batch
        out = torch.full((R + 2, 264), SENTINEL, device="cuda")
        h = HChain()
        h.rows, h.batch, h.K0, h.n_layers = self.rows, self.batch, self.K0, 2
        for j, s in enumerate(self.a0):
            h.a0[j] = s
        L0, L1 = h.layer[0], h.layer[1]
        L0.W, L0.K, L0.N, L0.ldw, L0.bias, L0.relu, L0.feeds_next = self.t["W0"].data_ptr(), self.K0, 256, self.K0, self.t["b0"].data_ptr(), 1, 1
        L0.add[0] = _hs(BCAST, self.t["add"])
        L1.W, L1.K, L1.N, L1.ldw, L1.bias = self.t["W1"].data_ptr(), 256, 256, 256, self.t["b1"].data_ptr()
        L1.ln_g, L1.ln_b = self.t["gamma"].data_ptr(), self.t["beta"].data_ptr()
        L1.residual = _hs(STREAM, self.t["res"], self.rows)
        L1.out, L1.ldo, L1.out_cols = out.data_ptr(), 264, 256
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        rc = tk.HK.h_chain(prec, ctypes.byref(h), None, _p(status), _st())
        torch.cuda.synchronize()
        return rc, int(status.item()), out


def _guard_fails(run, inputs, value, tag):
    """run() -> (rc, status, out buffer, stored-region mask).  Clean run, then one non-finite entry in each input in turn (bit 3,
    rc 0, nothing written outside the stored region), then a clean run again (status 0, the first clean output bit for bit)."""
    rc, st, clean, stored = run()
    assert rc == 0 and st == 0, (tag, rc, st)
    assert bool(torch.isfinite(clean[stored]).all())
    fails = []
    for slot, (t, ix) in inputs.items():
        old = t[ix].clone()
        t[ix] = value
        try:
            rc, st, out, _ = run()
        finally:
            t[ix] = old
        if rc != 0 or not st & 8:
            fails.append(f"{tag} {slot}: return code {rc}, status word {st} (expected 0 and bit 3)")
        if not bool((out[~stored] == SENTINEL).all()):
            fails.append(f"{tag} {slot}: written outside the stored rows / columns")
        rc, st, again, _ = run()
        if rc != 0 or st != 0 or not torch.equal(again.view(torch.int32), clean.view(torch.int32)):
            fails.append(f"{tag} {slot}: the clean launch after it gave return code {rc}, status {st}, or different bits")
    return fails


GUARD_KINDS = [pytest.param(k, id=n) for k, n in ((STREAM, "stream"), (BCAST, "bcast"), (GATHER, "gather"), (BGATHER, "bgather"), (GBR, "gbr"),
                                                   ("second", "second"))]  # fmt: skip


@gpu
@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("prec", [FP32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("kind", GUARD_KINDS)
def test_chain_refuses_non_finite(kind, prec, value):
    """An inference chain (h_chain, prepared as gw_api.cu prepares it) with one NaN / +inf / -inf in its stage-0 source, an
    addend, the residual, either weight, either bias, LayerNorm gamma or beta: status bit 3 and return code 0, no store outside
    the output rows x columns, and the next clean launch gives status 0 and the clean output bit for bit."""
    c = GuardChain(kind)
    R = c.rows * c.batch

    def run():
        rc, st, out = c.run(prec)
        stored = torch.zeros_like(out, dtype=torch.bool)
        stored[:R, :256] = True
        return rc, st, out, stored

    inputs = {slot: (c.t[slot], where()) for slot, where in c.reads.items()}
    fails = _guard_fails(run, inputs, VALUES[value], f"{tk.PREC_NAME[prec]} {kind}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("name", ["hidden", "features102", "two_source", "ln_res_stream"])
def test_fp32_row_op_refuses_non_finite(name, value):
    """A training row op on tensor cores in fp32 (h_row_op: stage-0 sources bounded by launch_operand_bound, weight images scaled
    on the device) with one non-finite entry in a stage-0 source or in W: status bit 3, return code 0, no store outside the output
    rows, and the next clean launch unaffected."""
    d = Data(8000 + tk.SHAPES.index(name), exact=True, s=0)
    op = tk._shape(name, d)
    op.ldo = op.N + 8
    R = op.rows * op.batch
    g = torch.Generator().manual_seed(8000 + tk.SHAPES.index(name))

    def run():
        out = torch.full((R + 2, op.ldo), SENTINEL, device="cuda")
        pre = torch.full((R + 2, op.ldo), SENTINEL, device="cuda") if op.save_pre else None
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        rc = tk.HK.h_row_op(FP32, ctypes.byref(_hop(op, out, pre, 0)), None, _p(status), _st())
        torch.cuda.synchronize()
        both = out if pre is None else torch.cat([out, pre], dim=1)
        stored = torch.zeros_like(both, dtype=torch.bool)
        stored[:R, :op.N] = True
        if pre is not None:
            stored[:R, op.ldo:op.ldo + op.N] = True
        return rc, int(status.item()), both, stored

    inputs = {f"a{j}:{KIND_NAME[s.kind]}": _src_entries(s, op.rows, op.batch, g)[0] for j, s in enumerate(op.a)}
    inputs["W"] = (op.W, (_pick(g, op.N), op.wcol + _pick(g, op.K)))
    fails = _guard_fails(run, inputs, VALUES[value], f"fp32 {name}")
    assert not fails, fails
