"""The forward's tensor-core chains (gw_chain_tc3_kernel), one at a time, against float64 references that torch computes on the GPU
from the same fp32 inputs, layer by layer (never against another kernel).

Every chain gw_forward.cu builds for the forecast is rebuilt here through h_chain (tests/kernels/gw_kernel_harness.cu), prepared as
inference prepares it: weight images and LayerNorm bounds through the library's tc_weights and tc_ln_bound, stage-0 bounds from
the inputs' absmax, the carry pass after fused per-target sums.  Each runs in fp32 (fp16 hi/lo split) and bf16, on the lean path and under GW_TC3_NOFAST (the general path), and must:
  (a) exact-integer data -- integers of at most 3 significant bits (both precisions) or 16 (fp32 only, so the lo parts are not
      zero) times 2^s, sparse +-1 weights, LayerNorm gamma = 0 so that a LayerNorm'd row is exactly beta + residual -- reproduce
      float64 bit for bit: every output, every per-target sum, carry and per-target constant.  s = -40 underflows any fp16
      operand that is not scaled up, s = 20 overflows any that is not scaled down;
  (b) random floats (normal, an outlier column, 1e-3 / 1e-6 / 1e5 magnitudes) stay under per-precision bars on eps_F and eps_el
      (test_gpu_kernels._eps) for every stored tensor and every per-target sum;
and in every case: the status word stays 0, every out_bound / seg_bound the chain writes bounds its tensor, memory outside the
stored rows x columns keeps its NaN prefill bit for bit, and the lean flag is the one gw_forward.cu relies on."""
import ctypes
import os

import pytest
import torch

from test_gpu_kernels import BCAST, BF16, FP32, GATHER, PREC_NAME, STREAM, HChain, HSrc, _compile_harness, _eps, _st

GBR = 5  # SRC_GATHER_BCAST_RELU: relu(P[idx] + E1)
H_ROWS = 150  # rows of the per-node tables the edge chains gather from
# Bars (eps_F, eps_el) of the random-float cases; worst values measured over every case of this file on an H100 80GB HBM3 (400 W):
#   fp32  4.4e-6 / 4.9e-5     bf16  6.4e-3 / 5.2e-3
# A dropped lo-part product leaves about 2^-12 = 2.4e-4 relative per product: 24x the fp32 eps_F bar.  Unscaled small operands
# (fp16 lo parts subnormal) measured 1.8e-5 .. 5.2e-5 eps_F at max|A| = 1e-3 and 1e-6.
BARS = {FP32: (1e-5, 1e-4), BF16: (2e-2, 2e-2)}
RUNS = [(FP32, False), (FP32, True), (BF16, False), (BF16, True)]

HK = None


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    global HK
    HK = _compile_harness(tmp_path_factory.mktemp("gw_chain_harness"))
    return HK


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


# ---- data ------------------------------------------------------------------------------------------------------------------------
class Gen:
    """Values of one case.  exact: integers in [-R, R] x 2^s everywhere except the weights (sparse: two +-1 per output row, so
    that values stay small integers through six layers) and gamma (0); otherwise normal floats of magnitude `mag` (weights
    N(0, 0.06), gamma in [0.5, 1.5), beta N(0, 0.1)), optionally with an outlier column 1e4 above the rest."""

    def __init__(self, seed, exact, s=0, wide=False, mag=1.0, outlier=False):
        self.g = torch.Generator(device="cuda").manual_seed(seed)
        self.exact, self.s, self.R, self.mag, self.outlier = exact, s, (2**15 if wide else 3), mag, outlier

    def _ints(self, shape):
        return torch.randint(-self.R, self.R + 1, shape, generator=self.g, device="cuda").float() * 2.0**self.s

    def operand(self, *shape):
        if self.exact:
            return self._ints(shape)
        t = torch.randn(shape, generator=self.g, device="cuda") * self.mag
        if self.outlier:
            t[..., shape[-1] // 3] *= 1e4
        return t

    def addend(self, *shape):
        return self._ints(shape) if self.exact else torch.randn(shape, generator=self.g, device="cuda") * (self.mag * 0.5)

    def weight(self, N, K):
        if not self.exact:
            return torch.randn(N, K, generator=self.g, device="cuda") * 0.06
        W = torch.zeros(N, K, device="cuda")
        cols = torch.randint(0, K, (N, 2), generator=self.g, device="cuda")
        sign = torch.randint(0, 2, (N, 2), generator=self.g, device="cuda").float() * 2 - 1
        W.scatter_add_(1, cols, sign)
        return W

    def ln(self, N):
        if self.exact:
            return torch.zeros(N, device="cuda"), self._ints((N,))
        return (torch.rand(N, generator=self.g, device="cuda") + 0.5, torch.randn(N, generator=self.g, device="cuda") * 0.1)

    def index(self, n, hi):
        return torch.randint(0, hi, (n,), generator=self.g, device="cuda", dtype=torch.int32)

    def targets(self, n_rows, maxdeg, empty):
        """seg_dst of n_rows rows sorted by target, runs of 1..maxdeg rows (at least one of maxdeg), and (empty) targets
        without rows between them and after the last one."""
        draws = torch.randint(0, 9 if empty else 8, (n_rows + 1,), generator=self.g, device="cuda").tolist()
        lengths = []
        for k in draws:
            if sum(lengths) >= n_rows:
                break
            lengths.append(0 if k == 8 else min(k + 1, maxdeg))
        if maxdeg not in lengths and n_rows >= maxdeg:
            lengths[len(lengths) // 2] = maxdeg
        dst, t = [], 0
        for k in lengths:
            dst += [t] * k
            t += 1
        dst = dst[:n_rows]
        n_targets = dst[-1] + 1 + (2 if empty else 0)
        return torch.tensor(dst, dtype=torch.int32, device="cuda"), n_targets


class S:
    """A row source over a 2-d fp32 tensor; rows64() assembles the float64 rows it stands for."""

    def __init__(self, kind, t, width=None, col0=0, src_rows=0, idx=None, t2=None, mul_i=None):
        self.kind, self.t, self.width, self.col0, self.src_rows, self.idx = kind, t, t.shape[1] if width is None else width, col0, src_rows, idx
        self.t2, self.mul_i = t2, mul_i

    def h(self):
        return HSrc(self.kind, self.width, self.t.shape[1], self.col0, self.t.data_ptr(), self.src_rows,
                    self.idx.data_ptr() if self.idx is not None else None, self.t2.data_ptr() if self.t2 is not None else None,
                    self.t2.shape[1] if self.t2 is not None else 0, self.mul_i.data_ptr() if self.mul_i is not None else None)

    def rows64(self, rows, batch):
        t = self.t[:, self.col0:self.col0 + self.width].double()
        b = torch.arange(batch, device="cuda")[:, None]
        i = torch.arange(rows, device="cuda")[None, :]
        if self.kind == STREAM:
            r = b * self.src_rows + i
        elif self.kind == BCAST:
            r = i.expand(batch, rows)
        elif self.kind in (GATHER, GBR):
            r = b * self.src_rows + self.idx.long()[None, :]
        else:
            r = self.idx.long()[None, :].expand(batch, rows)
        v = t[r.reshape(-1)]
        if self.kind == GBR:
            v = torch.relu(v + self.t2[:, :self.width].double().repeat(batch, 1))
        return v


class Lay:
    """One layer: out = residual + LN(relu(A W[:, wcol:wcol + K]^T + bias + add)).  out = (buffer, first column, columns);
    bound: name of the out_bound float it sets (layers naming the same one share it); seg = (seg_dst, targets, maxdeg, seg_add)."""

    def __init__(self, W, K, wcol=0, bias=None, add=(), relu=False, ln=None, res=None, out=None, feeds=False, reuse=False, bound=None,
                 seg=None):
        self.W, self.K, self.N, self.wcol, self.bias, self.add, self.relu, self.ln, self.res = W, K, W.shape[0], wcol, bias, add, relu, ln, res
        self.out, self.feeds, self.reuse, self.bound, self.seg = out, feeds, reuse, bound, seg


class Chain:
    def __init__(self, rows, batch, K0, a0, layers, bufs, peers=()):
        self.rows, self.batch, self.K0, self.a0, self.layers, self.bufs, self.peers = rows, batch, K0, a0, layers, bufs, tuple(peers)

    def seg_layer(self):
        return next((L for L in self.layers if L.seg is not None), None)

    def without_seg(self):
        """gw_forward.cu's unfused variant (general path): the layer's rows are stored instead of summed (buffer "e_rows" when the
        fused layer stores none)."""
        layers, bufs = [], dict(self.bufs)
        for L in self.layers:
            if L.seg is not None:
                out = L.out
                if out is None:
                    out, bufs["e_rows"] = ("e_rows", 0, L.N), L.N
                L = Lay(L.W, L.K, L.wcol, L.bias, L.add, L.relu, L.ln, L.res, out, L.feeds, L.reuse, L.bound, None)
            layers.append(L)
        return Chain(self.rows, self.batch, self.K0, self.a0, layers, bufs, self.peers)

    def run(self, prec, nofast=False):
        """-> (return code, lean flag, {buffer: tensor}, {bound name: float}, status word)"""
        R = self.rows * self.batch
        bufs = {k: torch.full((R, ld), float("nan"), device="cuda") for k, ld in self.bufs.items()}
        for k in self.peers[1:]:
            bufs[k] = torch.full((R, self.bufs[self.peers[0]]), float("nan"), device="cuda")
        bounds = {}
        h = HChain()
        h.rows, h.batch, h.K0, h.n_layers = self.rows, self.batch, self.K0, len(self.layers)
        for j, s in enumerate(self.a0):
            h.a0[j] = s.h()
        seg = self.seg_layer()
        if seg is not None:
            dst, nt, _, _ = seg.seg
            n_rows_per_target = torch.bincount(dst.long(), minlength=nt)
            fill = 0.0 if bool((n_rows_per_target == 0).any()) else float("nan")  # gw_forward.cu memsets the sums when a target has no rows
            bufs["seg"] = torch.full((self.batch * nt, seg.N), fill, device="cuda")
        for l, L in enumerate(self.layers):
            y = h.layer[l]
            y.W, y.K, y.N, y.ldw = L.W.data_ptr() + 4 * L.wcol, L.K, L.N, L.W.shape[1]
            y.bias = L.bias.data_ptr() if L.bias is not None else None
            for j, s in enumerate(L.add):
                y.add[j] = s.h()
            y.relu = int(L.relu)
            if L.ln is not None:
                y.ln_g, y.ln_b = L.ln[0].data_ptr(), L.ln[1].data_ptr()
            if L.res is not None:
                y.residual = L.res.h()
            if L.out is not None:
                b = bufs[L.out[0]]
                y.out, y.ldo, y.out_cols = b.data_ptr() + 4 * L.out[1], b.shape[1], L.out[2]
            y.feeds_next, y.reuse_a = int(L.feeds), int(L.reuse)
            if L.bound is not None:
                bounds.setdefault(L.bound, torch.zeros(1, device="cuda"))
                y.out_bound = bounds[L.bound].data_ptr()
            if L.seg is not None:
                dst, nt, maxdeg, sadd = L.seg
                y.seg_dst, y.seg_out, y.seg_ld, y.seg_rows, y.seg_maxdeg = dst.data_ptr(), bufs["seg"].data_ptr(), L.N, nt, maxdeg
                y.seg_add = sadd.data_ptr() if sadd is not None else None
                bounds["seg"] = torch.zeros(1, device="cuda")
                y.seg_bound = bounds["seg"].data_ptr()
        if self.peers:
            last = self.layers[-1].out
            h.out_mode, h.n_out_peers = 2, len(self.peers)
            for j, k in enumerate(self.peers):
                h.out_peer[j] = bufs[k].data_ptr() + 4 * last[1]
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        lean = ctypes.c_int(-2)
        old = os.environ.pop("GW_TC3_NOFAST", None)
        try:
            if nofast:
                os.environ["GW_TC3_NOFAST"] = "1"
            rc = HK.h_chain(prec, ctypes.byref(h), ctypes.byref(lean), ctypes.c_void_p(status.data_ptr()), _st())
            torch.cuda.synchronize()
        finally:
            os.environ.pop("GW_TC3_NOFAST", None)
            if old is not None:
                os.environ["GW_TC3_NOFAST"] = old
        return rc, lean.value, bufs, {k: float(v.item()) for k, v in bounds.items()}, int(status.item())

    def ref(self):
        """float64 {buffer: expected values, NaN where nothing is stored} and {buffer: |A| |W|^T + |addends| scale of each value}"""
        R = self.rows * self.batch
        want = {k: torch.full((R, ld), float("nan"), dtype=torch.float64, device="cuda") for k, ld in self.bufs.items()}
        scale = {k: torch.zeros((R, ld), dtype=torch.float64, device="cuda") for k, ld in self.bufs.items()}
        A = torch.cat([s.rows64(self.rows, self.batch) for s in self.a0], dim=1)
        cur, feed = A, None
        for l, L in enumerate(self.layers):
            if l > 0 and not L.reuse:
                cur = feed
            W = L.W[:, L.wcol:L.wcol + L.K].double()
            y = cur[:, :L.K] @ W.T
            c = cur[:, :L.K].abs() @ W.abs().T
            if L.bias is not None:
                y, c = y + L.bias.double(), c + L.bias.double().abs()
            for s in L.add:
                t = s.rows64(self.rows, self.batch)
                y, c = y + t, c + t.abs()
            if L.relu:
                y = torch.relu(y)
            if L.ln is not None:
                g, b = L.ln[0].double(), L.ln[1].double()
                sigma = torch.sqrt(y.var(dim=1, unbiased=False, keepdim=True) + 1e-5)
                y = torch.nn.functional.layer_norm(y, (L.N,), g, b, eps=1e-5)
                c = g.abs() * c / sigma + b.abs()  # an error of the pre-LayerNorm row reaches the output divided by its deviation
            if L.res is not None:
                t = L.res.rows64(self.rows, self.batch)
                y, c = y + t, c + t.abs()
            if L.out is not None:
                k, c0, n = L.out
                want[k][:, c0:c0 + n], scale[k][:, c0:c0 + n] = y[:, :n], c[:, :n]
            if L.seg is not None:
                dst, nt, _, sadd = L.seg
                idx = (torch.arange(self.batch, device="cuda")[:, None] * nt + dst.long()[None, :]).reshape(-1)
                ssum = torch.zeros(self.batch * nt, L.N, dtype=torch.float64, device="cuda").index_add_(0, idx, y)
                sc = torch.zeros_like(ssum).index_add_(0, idx, c)
                if sadd is not None:
                    has = (torch.bincount(dst.long(), minlength=nt) > 0).double()[:, None].repeat(self.batch, 1)
                    ssum, sc = ssum + has * sadd.double().repeat(self.batch, 1), sc + has * sadd.double().abs().repeat(self.batch, 1)
                want["seg"], scale["seg"] = ssum, sc
            feed = y
        for k in self.peers[1:]:
            want[k], scale[k] = want[self.peers[0]], scale[self.peers[0]]
        return want, scale


# ---- the catalogue: the chains gw_forward.cu builds -------------------------------------------------------------------------------
# name -> does the launcher send it to the lean path (GW_TC3_NOFAST unset)?
LEAN = {"enc_grid": 1, "enc_mesh": 1, "proc_p": 1, "proc_edge": 1, "proc_edge_last": 1, "proc_node": 1, "dec_p": 1, "dec_edge": 1,
        "dec_edge_res": 1, "dec_node": 1, "dec_node_misaligned": 0, "dec_node5": 1, "dec_out_odd": 0, "dec_node_n24": 0, "dec_node_n150": 0,
        "dec_node_peers": 0}
CHAINS = list(LEAN)
SEG_CHAINS = ["proc_edge", "proc_edge_last", "dec_edge", "dec_edge_res"]


def _chain(name, g, rows=300, batch=2, maxdeg=8, empty=True):
    R = rows * batch

    def mlp_tail(first):  # two more 256-wide layers of an MLP after `first`; the last one is returned bare
        return [first, Lay(g.weight(256, 256), 256, bias=g.addend(256), relu=True, feeds=True), Lay(g.weight(256, 256), 256, bias=g.addend(256))]

    def w768(*slices):  # [256, 768] first-layer weight whose column slices (offsets) are full weights of their own
        W = g.weight(256, 768)
        for c in slices:
            W[:, c:c + 256] = g.weight(256, 256)
        return W

    if name == "enc_grid":  # node encoder on 102 raw features (rows widened to 128) -> encoder block's edge MLP (+ C1, e_enc)
        x = torch.zeros(R, 128, device="cuda")
        x[:, :102] = g.operand(R, 102)
        L = [Lay(g.weight(256, 102), 102, bias=g.addend(256), relu=True, feeds=True),
             Lay(g.weight(256, 256), 256, bias=g.addend(256), relu=True, feeds=True),
             Lay(g.weight(256, 256), 256, bias=g.addend(256), ln=g.ln(256), feeds=True),
             Lay(g.weight(256, 256), 256, add=(S(BCAST, g.addend(rows, 256)),), relu=True, feeds=True),
             Lay(g.weight(256, 256), 256, bias=g.addend(256), relu=True, feeds=True),
             Lay(g.weight(256, 256), 256, bias=g.addend(256), ln=g.ln(256), res=S(BCAST, g.addend(rows, 256)), out=("e", 0, 256), bound="e")]
        return Chain(rows, batch, 128, [S(STREAM, x, src_rows=rows)], L, {"e": 256})
    if name == "enc_mesh":  # [xm0 (broadcast) | sum of incoming e' (bound x the longest segment)] -> node MLP + LN + xm0
        xm0 = g.operand(rows, 256)
        deg = torch.tensor([7], dtype=torch.int32, device="cuda")
        a0 = [S(BCAST, xm0), S(STREAM, g.operand(R, 256), src_rows=rows, mul_i=deg)]
        L = [Lay(g.weight(256, 512), 512, bias=g.addend(256), relu=True, feeds=True),
             Lay(g.weight(256, 256), 256, bias=g.addend(256), relu=True, feeds=True),
             Lay(g.weight(256, 256), 256, bias=g.addend(256), ln=g.ln(256), res=S(BCAST, xm0), out=("x", 0, 256), bound="x")]
        return Chain(rows, batch, 512, a0, L, {"x": 256})
    if name in ("proc_p", "dec_p"):  # P = x [W1s ; W1d]^T: two products of one operand into the halves of P, sharing one bound
        a0 = [S(STREAM, g.operand(R, 256), src_rows=rows)]
        if name == "dec_p":
            return Chain(rows, batch, 256, a0, [Lay(g.weight(256, 256), 256, out=("P", 0, 256), bound="P")], {"P": 256})
        W = w768(0)
        W1d = g.weight(256, 256) * 2.0**-10  # the second half is far smaller: its bound alone does not bound P
        L = [Lay(W, 256, out=("P", 0, 256), bound="P"), Lay(W1d, 256, out=("P", 256, 256), bound="P", reuse=True)]
        return Chain(rows, batch, 256, a0, L, {"P": 512})
    if name in ("proc_edge", "proc_edge_last"):  # W1e e + b1 + P[src, :256] + P[dst, 256:] -> 2 layers + LN + e -> e' (+ per-node sums)
        dst, nt = g.targets(rows, maxdeg, empty)
        P = g.addend(batch * H_ROWS, 512)
        e = S(STREAM, g.operand(R, 256), src_rows=rows)
        add = (S(GATHER, P, 256, 0, H_ROWS, g.index(rows, H_ROWS)), S(GATHER, P, 256, 256, H_ROWS, g.index(rows, H_ROWS)))
        first = Lay(w768(512), 256, wcol=512, bias=g.addend(256), add=add, relu=True, feeds=True)
        L = mlp_tail(first)
        L[2].ln, L[2].res, L[2].seg = g.ln(256), e, (dst, nt, maxdeg, None)
        if name == "proc_edge":
            L[2].out, L[2].bound = ("e", 0, 256), "e"
        return Chain(rows, batch, 256, [e], L, {"e": 256} if name == "proc_edge" else {})
    if name == "proc_node":  # [x | agg] -> node MLP + LN + x -> x', which is also the operand of the next block's two P products
        x = g.operand(R, 256)
        a0 = [S(STREAM, x, src_rows=rows), S(STREAM, g.operand(R, 256), src_rows=rows)]
        L = mlp_tail(Lay(g.weight(256, 512), 512, bias=g.addend(256), relu=True, feeds=True))
        L[2].ln, L[2].res, L[2].out, L[2].bound, L[2].feeds = g.ln(256), S(STREAM, x, src_rows=rows), ("x", 0, 256), "x", True
        W = w768(0, 256)
        L += [Lay(W, 256, out=("P", 0, 256), bound="P"), Lay(W, 256, wcol=256, out=("P", 256, 256), bound="P", reuse=True)]
        return Chain(rows, batch, 512, a0, L, {"x": 256, "P": 512})
    if name in ("dec_edge", "dec_edge_res"):  # relu(P[src] + E1) -> 2 layers + LN (+ e_dec, or + S_dec per target) -> per-point sums
        dst, nt = g.targets(rows, maxdeg, empty)
        a0 = [S(GBR, g.addend(batch * H_ROWS, 256), src_rows=H_ROWS, idx=g.index(rows, H_ROWS), t2=g.addend(rows, 256))]
        L = [Lay(g.weight(256, 256), 256, bias=g.addend(256), relu=True, feeds=True), Lay(g.weight(256, 256), 256, bias=g.addend(256), ln=g.ln(256))]
        if name == "dec_edge":
            L[1].seg = (dst, nt, maxdeg, g.addend(nt, 256))
        else:
            L[1].res, L[1].seg = S(BCAST, g.addend(rows, 256)), (dst, nt, maxdeg, None)
        return Chain(rows, batch, 256, a0, L, {})
    if name.startswith("dec_node"):  # aggregate -> node MLP + LN -> node decoder (256 -> 128 -> 128 -> out) + start features
        out_dim = {"dec_node_n24": 24, "dec_node_n150": 150}.get(name, 78)
        a0 = [S(STREAM, g.operand(R, 256), src_rows=rows)]
        L = mlp_tail(Lay(g.weight(256, 256), 256, bias=g.addend(256), relu=True, feeds=True))
        L[2].ln, L[2].feeds = g.ln(256), True
        L += [Lay(g.weight(128, 256), 256, bias=g.addend(128), relu=True, feeds=True), Lay(g.weight(128, 128), 128, bias=g.addend(128), relu=True)]
        if name == "dec_node5":  # the 5 + 1 split: the hidden rows leave the chain
            L[4].out, L[4].bound = ("h", 0, 128), "h"
            return Chain(rows, batch, 256, a0, L, {"h": 128})
        L[4].feeds = True
        last = Lay(g.weight(out_dim, 128), 128, bias=g.addend(out_dim))
        if out_dim == 78:  # rollout-style rows: the forecast lands in the first 78 of 102 columns, beside a residual of 102-wide rows
            last.res = S(STREAM, g.addend(R, 102), 78, src_rows=rows)
            last.out = ("o", 1 if name == "dec_node_misaligned" else 0, 78)
            bufs = {"o": 102}
        else:
            last.out, bufs = ("o", 0, out_dim), {"o": out_dim}
        L.append(last)
        return Chain(rows, batch, 256, a0, L, bufs, peers=("o", "o_p1", "o_p2") if name == "dec_node_peers" else ())
    if name == "dec_out_odd":  # the split's output chain with an odd width (77 of 102-wide rows): general path
        last = Lay(g.weight(77, 128), 128, bias=g.addend(77), res=S(STREAM, g.addend(R, 102), 77, src_rows=rows), out=("o", 0, 77))
        return Chain(rows, batch, 128, [S(STREAM, g.operand(R, 128), src_rows=rows)], [last], {"o": 77})
    raise KeyError(name)


# ---- checks ---------------------------------------------------------------------------------------------------------------------
def _untouched_ok(got, want):
    """every entry the chain must not store still holds the NaN prefill, bit for bit"""
    keep = torch.isnan(want)
    nan = torch.full_like(got, float("nan"))
    return torch.equal(got[keep].view(torch.int32), nan[keep].view(torch.int32))


def _check(chain, name, prec, nofast, exact, results=None):
    """Runs one configuration; returns (failure messages, {tensor: (eps_F, eps_el)})."""
    tag = f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
    rc, lean, bufs, bounds, status = chain.run(prec, nofast)
    fails = []
    if nofast and chain.seg_layer() is not None:  # the fused per-target sums exist on the lean path only
        if rc != 1:
            fails.append(f"{tag}: return code {rc}, expected cudaErrorInvalidValue")
        chain = chain.without_seg()
        rc, lean, bufs, bounds, status = chain.run(prec, nofast)
    if rc != 0:
        return [f"{tag}: return code {rc}"], {}
    want_lean = 0 if nofast else LEAN[name]
    if lean != want_lean:
        fails.append(f"{tag}: lean path {lean}, expected {want_lean}")
    if status != 0:
        fails.append(f"{tag}: status word {status}")
    want, scale = chain.ref()
    errs = {}
    for k, w in want.items():
        got = bufs[k]
        if not _untouched_ok(got, w):
            fails.append(f"{tag}: {k}: memory outside the stored values changed")
        m = ~torch.isnan(w)
        if k == "seg":
            m = torch.ones_like(w, dtype=torch.bool)
        gm, wm = got[m].double(), w[m]
        if exact:
            bad = int((gm != wm).sum().item())
            if bad:
                fails.append(f"{tag}: {k}: {bad} of {wm.numel()} values differ")
        else:
            errs[k] = _eps(gm, wm, scale[k][m])
        bname = "seg" if k == "seg" else k
        if bname in bounds and wm.numel() and not bounds[bname] >= float(gm.abs().max()):
            fails.append(f"{tag}: {k}: bound {bounds[bname]:.4g} below max |value| {float(gm.abs().max()):.4g}")
    return fails, errs


EXACT = [pytest.param(dict(exact=True, s=s), id=f"int_s{s}") for s in (-40, 0, 20)] + \
        [pytest.param(dict(exact=True, s=s, wide=True), id=f"wide_s{s}") for s in (-40, 0)]
FLOAT = [pytest.param(dict(exact=False, mag=1.0), id="normal"), pytest.param(dict(exact=False, mag=1.0, outlier=True), id="outlier"),
         pytest.param(dict(exact=False, mag=1e-3), id="mag1e-3"), pytest.param(dict(exact=False, mag=1e-6), id="mag1e-6"),
         pytest.param(dict(exact=False, mag=1e5), id="raw1e5")]


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("name", CHAINS)
def test_chain_exact(name, data):
    """Exact-integer chains: bit for bit on both precisions and both paths (16-bit operands: fp32 only -- they are not exact in
    bf16), every stored value, per-target sum and bound."""
    g = Gen(100 + CHAINS.index(name), **data)
    chain = _chain(name, g)
    fails = []
    for prec, nofast in RUNS:
        if data.get("wide") and prec == BF16:
            continue
        f, _ = _check(chain, name, prec, nofast, exact=True)
        fails += f
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("name", CHAINS)
def test_chain_float(name, data):
    """Random-float chains under the precision bars; two launches give identical bits."""
    g = Gen(200 + CHAINS.index(name), **data)
    chain = _chain(name, g)
    fails = []
    for prec, nofast in RUNS:
        tag = f"{name} {PREC_NAME[prec]}{' nofast' if nofast else ''}"
        f, errs = _check(chain, name, prec, nofast, exact=False)
        fails += f
        bf, bel = BARS[prec]
        for k, (ef, eel) in errs.items():
            print(f"{tag} {k}: eps_F {ef:.2e} eps_el {eel:.2e}")
            if not (ef < bf and eel < bel):
                fails.append(f"{tag} {k}: eps_F {ef:.2e} eps_el {eel:.2e}")
    first = chain.run(FP32)[2]
    again = chain.run(FP32)[2]
    for k in first:
        if not torch.equal(first[k].view(torch.int32), again[k].view(torch.int32)):
            fails.append(f"{name}: {k} differs between two launches")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("rows,batch", [(1, 1), (127, 1), (128, 1), (129, 1), (1, 3), (129, 3), (200, 3)])
@pytest.mark.parametrize("name", ["enc_grid", "proc_p", "proc_edge", "proc_node", "dec_edge", "dec_node", "dec_node_n150", "dec_out_odd"])
def test_chain_row_counts(name, rows, batch):
    """Row counts around the 128-row tile and single rows, one or three samples (tiles are ordered batch-major): bit for bit."""
    g = Gen(7 + rows + batch, exact=True, s=0)
    chain = _chain(name, g, rows, batch)
    fails = []
    for prec, nofast in RUNS:
        fails += _check(chain, name, prec, nofast, exact=True)[0]
    assert not fails, fails


@gpu
@pytest.mark.parametrize("name", ["enc_grid", "proc_edge", "dec_edge", "dec_node"])
def test_chain_persistent_tiles(name):
    """More than 132 x 128 rows: every CTA loops over several tiles (and, for the sums, several tiles' carry rows)."""
    g = Gen(31, exact=True, s=0)
    chain = _chain(name, g, rows=132 * 128 + 777, batch=2)
    fails = []
    for prec, nofast in [(FP32, False), (BF16, False), (FP32, True)]:
        fails += _check(chain, name, prec, nofast, exact=True)[0]
    assert not fails, fails


@gpu
@pytest.mark.parametrize("empty", [False, True])
@pytest.mark.parametrize("maxdeg", [7, 8])
@pytest.mark.parametrize("name", SEG_CHAINS)
def test_chain_target_sums(name, maxdeg, empty):
    """Fused per-target sums over many run shapes: runs of 1 to maxdeg rows starting on either row of a thread, crossing 16-row
    groups (carry rows) and tiles, targets with no rows (their memset zeros stay), single-row targets with the per-target
    constant.  Exact integers, bit for bit, at 16-bit (fp32) and 3-bit (bf16) operands."""
    fails = []
    for wide, runs in ((True, [(FP32, False)]), (False, [(BF16, False)])):
        g = Gen(41 + maxdeg + 2 * empty + 4 * SEG_CHAINS.index(name), exact=True, s=0, wide=wide)
        chain = _chain(name, g, rows=1000, batch=3, maxdeg=maxdeg, empty=empty)
        for prec, nofast in runs:
            fails += _check(chain, name, prec, nofast, exact=True)[0]
    assert not fails, fails
