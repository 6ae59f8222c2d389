"""-m gpu: the exact-fp32 CUDA-core row op (gw_rowop_f32_kernel, and gw_ln_rows_kernel for LayerNorm rows wider than 256) in the
roles csrc/gw_forward.cu gives it in the forward, and the forward's small helpers, one at a time against float64.

This row op computes the weight constants every precision reads (xm0, e_enc, C1_enc, e_lat, e_dec, E1_dec), it is the whole
forward of every model the tensor-core chains do not fit (hidden 64, the 32-wide regional model, 1024-wide models, the per-sample
node decoder), and it is what the tensor-core forward is compared with.  Each variant below rebuilds one GemmOp gw_forward.cu issues on
the CUDA cores, named after its call site, at the widths of the models that run it.  The helpers of tests/test_gpu_kernels.py do
the work (Data, Src, RowOp, the harness); the checks:
  * exact-integer data bit for bit (LayerNorm layers: the pre-LN value bit for bit, the normalised output within 1e-5);
  * random data under the fp32_simt bars of test_gpu_kernels.py;
  * identity weights (K = N, W = I, no bias), so that the output IS the A row the kernel assembled: a segment sum must equal the
    left-to-right float32 sum in perm / ptr order, relu(gather + broadcast) must equal relu(fp32(P[src] + E1)), bit for bit
    (a float64 reference can show a wrong summation order only as a small error);
  * every float outside the stored rows and columns keeps its NaN prefill, bit for bit.
Helpers: launch_pad_rows (widening copy + absmax), launch_absmax_flat (unaligned head, float4 body, tail), launch_csr_expand."""
import ctypes

import pytest
import torch

import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import BGATHER, GATHER, GBR, SEGSUM, SIMT, STREAM, Data, HOp, Src, _a, _eps, _ok, _p, _st, bcast, stream

BAR_F, BAR_EL = tk.BARS[SIMT]
NAN_BITS = 0x7FC00000  # torch.full(..., nan)


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    tk.HK = tk._compile_harness(tmp_path_factory.mktemp("gw_forward_harness"))  # (the helpers of test_gpu_kernels call through it)
    return tk.HK


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


# ---- one forward row op, stored into a column window of a shared NaN-prefilled buffer -----------------------------------------------
class Op(tk.RowOp):
    """A GemmOp of the forward on the CUDA cores; its N outputs go to columns ocol .. ocol + N of [rows * batch, ldo] buffers."""

    def __init__(self, *a, ocol=0, **kw):
        super().__init__(*a, **kw)
        self.ocol = ocol

    def launch(self, out, pre=None):
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
        h.out, h.ldo = out.data_ptr() + 4 * self.ocol, self.ldo
        h.save_pre = pre.data_ptr() + 4 * self.ocol if pre is not None else None
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        _ok(tk.HK.h_row_op(SIMT, ctypes.byref(h), None, _p(status), _st()))


def run(ops):
    """Runs ops (same rows, batch, ldo) into one pair of NaN-prefilled buffers: (out, pre, stored-region mask)."""
    R, ldo = ops[0].rows * ops[0].batch, ops[0].ldo
    out = torch.full((R, ldo), float("nan"), device="cuda")
    pre = torch.full((R, ldo), float("nan"), device="cuda") if any(o.save_pre for o in ops) else None
    stored = torch.zeros(R, ldo, dtype=torch.bool, device="cuda")
    for o in ops:
        o.launch(out, pre if o.save_pre else None)
        stored[:, o.ocol:o.ocol + o.N] = True
    torch.cuda.synchronize()
    return out, pre, stored


def untouched(buf, stored):
    """The entries outside the stored region still hold the NaN prefill, bit for bit."""
    return buf is None or bool((buf.view(torch.int32)[~stored] == NAN_BITS).all())


# ---- graphs ----------------------------------------------------------------------------------------------------------------------
def _csr(d, n, big=0, hi=7):
    """CSR over n segments of 1 .. hi rows, with empty segments (when n > 3) and, when big, one segment of `big` rows."""
    L = torch.randint(1, hi + 1, (n,), generator=d.g, device="cuda")
    if n > 3:
        L[1] = 0
        L[n // 2] = 0
        L[n - 1] = 0
    if big:
        L[n // 3] = big
    return torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), L.cumsum(0)]).int()


def _perm(d, n):
    return torch.randperm(n, generator=d.g, device="cuda").int()


def _idx(d, n, hi):
    return torch.randint(0, hi, (n,), generator=d.g, device="cuda", dtype=torch.int32)


# ---- the forward's CUDA-core row ops -------------------------------------------------------------------------------------------
# widths of the models that run these ops: node = edge = hidden width D, node-decoder hidden hd, input features fin, outputs nout
WIDTHS = {
    "w256": dict(D=256, hd=128, fin=102, nout=78),  # the default model (its constants, and the CUDA-core forward it is checked with)
    "w64": dict(D=64, hd=32, fin=14, nout=10),      # the hidden-64 fixture (10 + 4 features)
    "w32": dict(D=32, hd=32, fin=16, nout=12),      # the regional configuration (12 + 4 features, a LayerNorm'd node decoder)
}
NT = 150  # rows per sample of the tables the gathers read


def _ln(d, n):
    return torch.rand(n, generator=d.g, device="cuda") + 0.5, torch.randn(n, generator=d.g, device="cuda") * 0.1


def variant(name, d, w, rows=None, batch=None):
    """The GemmOps (one, or the two P halves) of one gw_forward.cu call site, on the data of generator d."""
    D, hd, fin, nout = w["D"], w["hd"], w["fin"], w["nout"]
    batch1 = name.startswith("pre_")  # the constants are computed once, batch 1
    rows = rows or 300
    batch = batch or (1 if batch1 else 3)
    R = rows * batch

    def W1():  # the edge MLP's first Linear [He, 2 Dn + De]: columns 0 / Dn / 2 Dn act on x_src / x_dst / e
        return d.weight(D, 3 * D)

    if name in ("pre_node_enc_h3", "enc_node_features"):  # node encoder Linear 0 (h3_nodes: xm0; raw features: the lat/lon rows)
        return [Op(rows, batch, [stream(d.operand(R, fin), rows)], d.weight(D, fin), fin, D, bias=d.addend(D), relu=True)]
    if name in ("pre_edge_enc_k2", "pre_edge_enc_k3"):  # edge encoders on [sin d, cos d] (latent, decoder) / [.., height] (assimilator)
        k = int(name[-1])
        return [Op(rows, batch, [stream(d.operand(R, k), rows)], d.weight(D, k), k, D, bias=d.addend(D), relu=True)]
    if name == "pre_tmpP":  # tmpP = xm0 W1d^T: a column slice of W1 (ldw = 3 Dn)
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], W1(), D, D, wcol=D)]
    if name == "pre_C1_enc":  # C1_enc = e_enc W1e^T + b1 + tmpP[enc_mesh]  (batch-invariant gather)
        add = (Src(BGATHER, d.addend(NT, D), D, 0, NT, _idx(d, rows, NT)),)
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], W1(), D, D, wcol=2 * D, bias=d.addend(D), add=add)]
    if name == "pre_E1_dec":  # E1_dec = e_dec W1e^T + b1
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], W1(), D, D, wcol=2 * D, bias=d.addend(D))]
    if name == "enc_edge_l1":  # encoder edge layer 1: xg W1s^T + C1_enc (broadcast), no bias
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], W1(), D, D, add=(bcast(d.addend(rows, D)),), relu=True)]
    if name == "enc_edge_ln_bcast":  # last edge layer: LayerNorm + the broadcast e_enc residual
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], d.weight(D, D), D, D, bias=d.addend(D), ln=_ln(d, D),
                   residual=bcast(d.addend(rows, D)), save_pre=True)]  # fmt: skip
    if name == "enc_mesh_node_l1":  # mesh node layer 1 on [xm0 (broadcast) ; sum over the lat/lon points of e' in perm order]
        ptr = _csr(d, rows, big=4096 if rows >= 64 else 0)  # (a polar cell collects > 4096 points at 0.25 degree)
        E = int(ptr[-1])
        a = [bcast(d.operand(rows, D)), Src(SEGSUM, d.operand(batch * E, D), D, 0, E, ptr=ptr, perm=_perm(d, E))]
        return [Op(rows, batch, a, d.weight(D, 2 * D), 2 * D, D, bias=d.addend(D), relu=True)]
    if name == "proc_P":  # P = x [W1s ; W1d]^T: the two halves of one [rows, 2 He] buffer
        x, W = stream(d.operand(R, D), rows), W1()
        return [Op(rows, batch, [x], W, D, D, wcol=h * D, ldo=2 * D, ocol=h * D) for h in (0, 1)]
    if name == "proc_edge_l1":  # processor edge layer 1: e W1e^T + b1 + P[src, :He] + P[dst, He:]
        P = d.addend(batch * NT, 2 * D)
        add = (Src(GATHER, P, D, 0, NT, _idx(d, rows, NT)), Src(GATHER, P, D, D, NT, _idx(d, rows, NT)))
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], W1(), D, D, wcol=2 * D, bias=d.addend(D), add=add, relu=True)]
    if name == "proc_node_l1":  # processor node layer 1 on [x ; sum of e' over the node's CSR segment] (no perm)
        ptr = _csr(d, rows)
        E = int(ptr[-1])
        a = [stream(d.operand(R, D), rows), Src(SEGSUM, d.operand(batch * E, D), D, 0, E, ptr=ptr)]
        return [Op(rows, batch, a, d.weight(D, 2 * D), 2 * D, D, bias=d.addend(D), relu=True)]
    if name == "proc_ln_res":  # last node layer: LayerNorm + the per-sample x residual
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], d.weight(D, D), D, D, bias=d.addend(D), ln=_ln(d, D),
                   residual=stream(d.addend(R, D), rows), save_pre=True)]  # fmt: skip
    if name == "dec_Pd":  # decoder Pd = x W1s^T
        return [Op(rows, batch, [stream(d.operand(R, D), rows)], W1(), D, D)]
    if name == "dec_edge_l2":  # decoder edge layer 2 on relu(Pd[dec_src] + E1_dec), the virtual layer 1
        a = [Src(GBR, d.operand(batch * NT, D), D, 0, NT, _idx(d, rows, NT), t2=d.operand(rows, D))]
        return [Op(rows, batch, a, d.weight(D, D), D, D, bias=d.addend(D), relu=True)]
    if name == "dec_node_l1":  # decoder node layer 1: the aggregate half of W1 (columns Dn ..) on the per-point sums
        ptr = _csr(d, rows)
        E = int(ptr[-1])
        a = [Src(SEGSUM, d.operand(batch * E, D), D, 0, E, ptr=ptr)]
        return [Op(rows, batch, a, d.weight(D, 2 * D), D, D, wcol=D, bias=d.addend(D), relu=True)]
    if name in ("dec_out", "dec_out_ln"):  # node decoder output layer + start-feature residual (start_ld = in_dim > out_dim),
        # written into rows of in_dim floats (a rollout's next input); the regional node decoder has a LayerNorm
        res = stream(d.addend(R, fin), rows, width=nout)
        ln = _ln(d, nout) if name == "dec_out_ln" else None
        return [Op(rows, batch, [stream(d.operand(R, hd), rows)], d.weight(nout, hd), hd, nout, bias=d.addend(nout), ln=ln, residual=res,
                   ldo=fin, save_pre=ln is not None)]  # fmt: skip
    raise KeyError(name)


VARIANTS = ["pre_node_enc_h3", "pre_edge_enc_k2", "pre_edge_enc_k3", "pre_tmpP", "pre_C1_enc", "pre_E1_dec", "enc_node_features",
            "enc_edge_l1", "enc_edge_ln_bcast", "enc_mesh_node_l1", "proc_P", "proc_edge_l1", "proc_node_l1", "proc_ln_res", "dec_Pd",
            "dec_edge_l2", "dec_node_l1", "dec_out", "dec_out_ln"]  # fmt: skip


def _wide(name, d, rows=200, batch=2):
    """Rows wider than one 256-column block: LayerNorm'd rows of N outputs (gw_ln_rows_kernel finishes them), and the 597 outputs
    of an ERA5 decoder over 621-wide start rows (three column blocks, no LayerNorm)."""
    R = rows * batch
    if name.startswith("ln_rows"):
        N = int(name[len("ln_rows"):])
        res = Src(STREAM, d.addend(R, N + 3), N, 2, rows)
        return [Op(rows, batch, [stream(d.operand(R, 64), rows)], d.weight(N, 64), 64, N, bias=d.addend(N), ln=_ln(d, N), residual=res,
                   ldo=N + 5, save_pre=True)]  # fmt: skip
    res = stream(d.addend(R, 621), rows, width=597)
    return [Op(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(597, 256), 256, 597, bias=d.addend(597), residual=res, ldo=621)]


WIDE = ["ln_rows300", "ln_rows597", "ln_rows1024", "out597"]


def _build(name, d, wname, rows=None, batch=None):
    return _wide(name, d, **({} if rows is None else dict(rows=rows, batch=batch))) if wname == "wide" else variant(name, d, WIDTHS[wname], rows, batch)


def _exact_fails(ops, tag):
    out, pre, stored = run(ops)
    fails = []
    for o in ops:
        y64, pre64, _ = o.ref()
        got = out[:, o.ocol:o.ocol + o.N].double()
        if o.ln is None:
            bad = int((got != y64).sum())
            if bad:
                fails.append(f"{tag}: {bad} of {y64.numel()} values differ")
        else:
            if not torch.equal(pre[:, o.ocol:o.ocol + o.N].double(), pre64):
                fails.append(f"{tag}: pre-LayerNorm values differ")
            ef = float((got - y64).norm() / y64.norm())
            if not ef < 1e-5:
                fails.append(f"{tag}: LayerNorm output eps_F {ef:.2e}")
    if not (untouched(out, stored) and untouched(pre, stored)):
        fails.append(f"{tag}: entries outside the stored rows / columns were written")
    return fails


CASES = [pytest.param(n, w, id=f"{n}-{w}") for w in WIDTHS for n in VARIANTS] + [pytest.param(n, "wide", id=n) for n in WIDE]


@gpu
@pytest.mark.parametrize("data", tk.EXACT)
@pytest.mark.parametrize("name,wname", CASES)
def test_forward_row_op_exact(name, wname, data):
    d = Data(100 + VARIANTS.index(name) if name in VARIANTS else 200 + WIDE.index(name), **data)
    ops = _build(name, d, wname)
    fails = _exact_fails(ops, f"{name} {wname}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("rows,batch", [(r, b) for r in (1, 63, 64, 65, 129) for b in (1, 3)])
@pytest.mark.parametrize("name", ["enc_mesh_node_l1", "proc_P", "proc_edge_l1", "proc_node_l1", "proc_ln_res", "dec_edge_l2", "dec_out_ln"])
def test_forward_row_op_row_counts(name, rows, batch):
    """Row counts around the 64-row tile, one or three samples (64-row tiles straddle the samples): bit for bit."""
    d = Data(rows * 10 + batch, exact=True, s=0)
    fails = _exact_fails(variant(name, d, WIDTHS["w256"], rows, batch), f"{name} rows {rows} batch {batch}")
    assert not fails, fails


# Worst measured over every case on an H100 80GB HBM3: eps_F 1.1e-6, eps_el 1.0e-6, LayerNorm output eps_F 3.0e-7 (bars 1e-5 / 1e-4).
@gpu
@pytest.mark.parametrize("data", tk.FLOAT)
@pytest.mark.parametrize("name,wname", CASES)
def test_forward_row_op_float(name, wname, data):
    d = Data(300 + VARIANTS.index(name) if name in VARIANTS else 400 + WIDE.index(name), **data)
    ops = _build(name, d, wname)
    out, pre, stored = run(ops)
    fails = []
    for o in ops:
        y64, pre64, c = o.ref()
        got = out[:, o.ocol:o.ocol + o.N]
        if o.ln is None:
            ef, eel = _eps(got, y64, c)
        else:
            ef, eel = _eps(pre[:, o.ocol:o.ocol + o.N], pre64, c)
            efo = float((got.double() - y64).norm() / y64.norm())
            print(f"{name} {wname}: LayerNorm output eps_F {efo:.2e}")
            if not efo < BAR_F:
                fails.append(f"LayerNorm output eps_F {efo:.2e}")
        print(f"{name} {wname} col {o.ocol}: eps_F {ef:.2e} eps_el {eel:.2e}")
        if not (ef < BAR_F and eel < BAR_EL):
            fails.append(f"col {o.ocol}: eps_F {ef:.2e} eps_el {eel:.2e}")
    if not (untouched(out, stored) and untouched(pre, stored)):
        fails.append("entries outside the stored rows / columns were written")
    assert not fails, fails


# ---- the assembled A rows, bit for bit -----------------------------------------------------------------------------------------
def _seq_segsum(base, width, ptr, perm, src_rows, rows, batch):
    """Per segment, the float32 sum of its rows left to right (in perm order when set), one row position at a time."""
    L = (ptr[1:] - ptr[:-1]).long()
    e_all = perm.long() if perm is not None else torch.arange(int(ptr[-1]), device="cuda")
    t = base[:, :width].reshape(batch, src_rows, width)
    acc = torch.zeros(batch, rows, width, device="cuda")
    for j in range(int(L.max()) if rows else 0):
        seg = torch.nonzero(L > j).squeeze(1)
        acc[:, seg] = acc[:, seg] + t[:, e_all[ptr[seg].long() + j]]
    return acc.reshape(batch * rows, width)


@gpu
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("wname", list(WIDTHS))
@pytest.mark.parametrize("kind", ["segsum_perm", "segsum", "gbr"])
def test_assembled_rows_identity(kind, wname, batch):
    """W = I (K = N, no bias): the output is the A row the kernel assembled.  Segment sums (empty segments, 1-7 rows, one of 4096
    rows) must equal the sequential float32 sum in perm / ptr order; relu(gather + broadcast) must equal relu(fp32(P[src] + E1))."""
    D = WIDTHS[wname]["D"]
    d = Data(500 + batch, exact=False, mag=1.0)
    rows = 300
    eye = torch.eye(D, device="cuda")
    if kind == "gbr":
        P, E1, idx = d.operand(batch * NT, D), d.operand(rows, D), _idx(d, rows, NT)
        a = Src(GBR, P, D, 0, NT, idx, t2=E1)
        want = torch.relu(P.view(batch, NT, D)[:, idx.long()] + E1[None]).reshape(batch * rows, D)
    else:
        ptr = _csr(d, rows, big=4096 if kind == "segsum_perm" else 0)
        E = int(ptr[-1])
        perm = _perm(d, E) if kind == "segsum_perm" else None
        base = d.operand(batch * E, D + 4)  # (rows of a wider stride: the source reads the first D columns)
        a = Src(SEGSUM, base, D, 0, E, ptr=ptr, perm=perm)
        want = _seq_segsum(base, D, ptr, perm, E, rows, batch)
    out, _, stored = run([Op(rows, batch, [a], eye, D, D)])
    got = out[:, :D]
    assert torch.equal(got, want), f"{int((got != want).sum())} of {want.numel()} assembled values differ"
    assert untouched(out, stored)


# ---- the forward's small helpers -----------------------------------------------------------------------------------------------
def _aligned_view(t, off, n):
    """n floats starting `off` floats past a 16-byte boundary of t's storage."""
    assert t.data_ptr() % 16 == 0
    return t[off:off + n]


@gpu
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
@pytest.mark.parametrize("width,ld_dst", [(102, 128), (14, 64)])
def test_pad_rows(width, ld_dst, shift):
    """The widening copy of raw feature rows (K0-wide, zero padded) and its absmax, from rows that start at misaligned offsets."""
    g = torch.Generator(device="cuda").manual_seed(width + shift)
    rows = 3001
    buf = torch.randn(rows * width + 8, generator=g, device="cuda") * 7
    src = _aligned_view(buf, shift, rows * width)
    dst = torch.full((rows, ld_dst), float("nan"), device="cuda")
    amax = torch.zeros(1, device="cuda")
    _ok(tk.HK.h_pad_rows(_p(src), width, width, _p(dst), ld_dst, rows, _p(amax), _st()))
    torch.cuda.synchronize()
    assert torch.equal(dst[:, :width], src.view(rows, width))
    assert bool((dst[:, width:].view(torch.int32) == 0).all()), "padding is not +0"
    assert float(amax) == float(src.abs().max())


@gpu
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
@pytest.mark.parametrize("where", [0, 0.37, 1.0])
def test_pad_rows_non_finite_bound(where, bad):
    """One NaN / inf anywhere among the inputs: the bound is +inf (the chain flags it as a non-finite operand)."""
    rows, width = 2000, 102
    src = torch.randn(rows, width, device="cuda")
    k = min(int(where * rows * width), rows * width - 1)
    src.view(-1)[k] = bad
    dst = torch.empty(rows, 128, device="cuda")
    amax = torch.zeros(1, device="cuda")
    _ok(tk.HK.h_pad_rows(_p(src), width, width, _p(dst), 128, rows, _p(amax), _st()))
    torch.cuda.synchronize()
    assert float(amax) == float("inf")


def _regions(off, n):
    """(head, body, tail) index ranges of launch_absmax_flat over n floats starting `off` floats past a 16-byte boundary."""
    head = min(n, (4 - off) % 4)
    nv = (n - head) // 4
    return {"head": range(0, head), "body": range(head, head + 4 * nv), "tail": range(head + 4 * nv, n)}


ABSMAX_N = list(range(1, 10)) + [1_000_003]  # (large n: every thread strides over the float4 body)


@gpu
@pytest.mark.parametrize("n", ABSMAX_N)
@pytest.mark.parametrize("off", [0, 1, 2, 3])
def test_absmax_flat(off, n):
    """max |x| over a contiguous array whose base is 0-3 floats past 16-byte alignment, with the largest value placed in the
    unaligned head, the float4 body and the tail in turn; a NaN in each region makes the bound +inf."""
    g = torch.Generator(device="cuda").manual_seed(off * 100 + n % 97)
    buf = torch.randn(n + 8, generator=g, device="cuda")
    for region, ix in _regions(off, n).items():
        if not len(ix):
            continue
        for pos in sorted({ix[0], ix[len(ix) // 2], ix[-1]}):
            for v, want in ((-(2.0**100), 2.0**100), (float("nan"), float("inf"))):
                t = buf.clone()
                p = _aligned_view(t, off, n)
                p[pos] = v
                amax = torch.zeros(1, device="cuda")
                _ok(tk.HK.h_absmax_flat(_p(p), n, _p(amax), _st()))
                torch.cuda.synchronize()
                assert float(amax) == want, f"{region} position {pos}: {float(amax)} (expected {want})"
    p = _aligned_view(buf, off, n)
    amax = torch.zeros(1, device="cuda")
    _ok(tk.HK.h_absmax_flat(_p(p), n, _p(amax), _st()))
    torch.cuda.synchronize()
    assert float(amax) == float(p.abs().max())


@gpu
@pytest.mark.parametrize("case", ["small", "no_empty", "strided"])
def test_csr_expand(case):
    """dst[j] = i over the whole CSR and {longest, shortest} segment (they pick the fused-sum path and scale magnitude bounds);
    n above 1184 x 256 segments: every thread of the capped grid strides."""
    g = torch.Generator(device="cuda").manual_seed(len(case))
    n = {"small": 7, "no_empty": 1000, "strided": 1184 * 256 + 777}[case]
    L = torch.randint(0 if case != "no_empty" else 2, 8, (n,), generator=g, device="cuda")
    if case == "strided":
        L[-1] = 11  # the longest segment is the last one, met by a striding thread
    if case == "small":
        L[3] = 0
    ptr = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), L.cumsum(0)]).int()
    E = int(ptr[-1])
    dst = torch.full((E + 4,), -7, dtype=torch.int32, device="cuda")
    stats = torch.tensor([0, 2**31 - 1], dtype=torch.int32, device="cuda")
    _ok(tk.HK.h_csr_expand(_p(ptr), n, _p(dst), _p(stats), _st()))
    stats2 = torch.tensor([0, 2**31 - 1], dtype=torch.int32, device="cuda")
    _ok(tk.HK.h_csr_expand(_p(ptr), n, None, _p(stats2), _st()))  # statistics only
    torch.cuda.synchronize()
    want = torch.repeat_interleave(torch.arange(n, device="cuda", dtype=torch.int32), L)
    assert torch.equal(dst[:E], want)
    assert bool((dst[E:] == -7).all())
    assert stats.tolist() == [int(L.max()), int(L.min())] == stats2.tolist()
