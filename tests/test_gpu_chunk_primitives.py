"""-m gpu: the row movement of the bounded-memory training step (gw_train.cu: build_chunks, enc_fwd / enc_bwd / enc_node_bwd,
dec_fwd / dec_bwd), one launcher at a time, bit for bit against numpy.

  * launch_permute_rows gathers each encoder chunk's features and attributes through enc_perm and scatters the feature gradient,
    the decoder chunk's output rows and the per-slot sums back: gather and scatter, one and three samples, a strict subset of a
    permutation, widths 2 / 78 / 102 / 621 with strides wider than the rows, below and above one grid-stride pass.  A scatter
    leaves every row and column it does not address bit-identical (NaN prefill included).
  * launch_strided_add adds the residual's share of dOut (78 columns) into dFeatures (102 wide): numpy's float32 add.
  * launch_segsum with ptr_base (the chunk's CSR slice of the full table, over the chunk's own rows) and with accumulate (dPd
    summed over decoder chunks in chunk order: previous value + this call's sequential float32 sum).
  * launch_gather_rows with idx_base (the decoder chunk's d_agg_g holds the chunk's points only).
  * rows == 0: success, nothing written.
The chunk's rows sit at the front of buffers as large as the whole table, as they do in the step, so that a launcher reading
through the wrong offset reads other data instead of leaving the buffer.  The helpers of tests/test_gpu_kernels.py do the work."""
import ctypes

import numpy as np
import pytest
import torch

import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import _csr, _ok, _p, _seq_sum, _st

GRID_THREADS = 132 * 8 * 256  # one grid-stride pass of launch_permute_rows / launch_gather_rows (GRID_SMS x 8 blocks x 256)


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    tk.HK = tk._compile_harness(tmp_path_factory.mktemp("gw_chunk_harness"))  # (the helpers of test_gpu_kernels call through it)
    return tk.HK


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _at(t, elems):  # device address `elems` elements into t (a slice of a table, as the step passes p->enc_ptr.p + r.s0)
    return ctypes.c_void_p(t.data_ptr() + t.element_size() * elems)


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _prefill(rng, rows, ld, width, nan_rows=True):
    """Random rows with every column >= width NaN, and every third row NaN (nan_rows: for a launcher that adds to what it
    finds, whose NaN + x has no defined payload, they stay finite): what a launcher does not address must keep its bits."""
    a = rng.standard_normal((rows, ld)).astype(np.float32)
    if nan_rows:
        a[::3] = np.nan
    a[:, width:] = np.nan
    return a


def _assert_bits(got, want, what):
    bad = _bits(got) != _bits(want)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} floats differ, first at {np.argwhere(bad)[0].tolist()}"


# ---- launch_permute_rows ------------------------------------------------------------------------------------------------------
def _permute_case(width, batch, size):
    """rows and other_rows (> rows) of a case: rows * batch * width below one grid-stride pass, or about 2.5 passes."""
    if size == "small":
        rows = max(1, min(300, (GRID_THREADS // 4) // (batch * width)))
    else:
        rows = (5 * GRID_THREADS) // (2 * batch * width) + 1
    return rows, rows + rows // 3 + 5


@gpu
@pytest.mark.parametrize("size", ["small", "large"])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("width", [2, 78, 102, 621])
def test_permute_rows(width, batch, size):
    rows, other = _permute_case(width, batch, size)
    assert (rows * batch * width < GRID_THREADS) == (size == "small")
    rng = np.random.Generator(np.random.PCG64(width * 10 + batch + (size == "large")))
    idx = rng.permutation(other)[:rows].astype(np.int32)  # a strict subset of a permutation of other_rows
    ld_far, ld_near = width + 3, width + 5
    tidx = _dev(idx)
    far_rows = (np.arange(batch)[:, None] * other + idx[None, :]).reshape(-1)  # row (b, idx[j]) of the other_rows side

    # gather: out row (b, j) = in row (b, idx[j])
    src = rng.standard_normal((batch * other, ld_far)).astype(np.float32)
    out0 = _prefill(rng, batch * rows, ld_near, width)
    out = _dev(out0)
    tsrc = _dev(src)
    _ok(tk.HK.h_permute_rows(_p(tsrc), ld_far, _p(tidx), rows, other, width, batch, _p(out), ld_near, 0, _st()))
    torch.cuda.synchronize()
    want = out0.copy()
    want[:, :width] = src[far_rows, :width]
    _assert_bits(out.cpu().numpy(), want, f"gather rows {rows} batch {batch} width {width}")

    # scatter: out row (b, idx[j]) = in row (b, j); the other rows of out and its columns >= width keep their bits
    src = rng.standard_normal((batch * rows, ld_near)).astype(np.float32)
    out0 = _prefill(rng, batch * other, ld_far, width)
    out = _dev(out0)
    tsrc = _dev(src)
    _ok(tk.HK.h_permute_rows(_p(tsrc), ld_near, _p(tidx), rows, other, width, batch, _p(out), ld_far, 1, _st()))
    torch.cuda.synchronize()
    want = out0.copy()
    want[far_rows, :width] = src[:, :width]
    _assert_bits(out.cpu().numpy(), want, f"scatter rows {rows} batch {batch} width {width}")


# ---- launch_strided_add -------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("rows", [37, 2 * 4001])
def test_strided_add(rows):
    """dFeatures[:, :78] += dOut (the residual's share of the output gradient): rows of 78 into rows of 102, float32 adds; the
    24 auxiliary columns keep their bits.  8002 rows x 78 columns are several grid-stride passes."""
    rng = np.random.Generator(np.random.PCG64(rows))
    src = rng.standard_normal((rows, 78)).astype(np.float32)
    dst0 = rng.standard_normal((rows, 102)).astype(np.float32)
    dst0[:, 78:] = np.nan
    dst0[::5, 80] = 3.0
    tsrc, dst = _dev(src), _dev(dst0)
    _ok(tk.HK.h_strided_add(_p(tsrc), 78, _p(dst), 102, rows, 78, _st()))
    torch.cuda.synchronize()
    want = dst0.copy()
    want[:, :78] = dst0[:, :78] + src
    _assert_bits(dst.cpu().numpy(), want, f"strided add, {rows} rows")


# ---- launch_segsum over a CSR slice (ptr_base) --------------------------------------------------------------------------------
def _full_table(rng):
    """Segment lengths of a full CSR table: mostly short, some empty, one of 700 rows."""
    lengths = rng.integers(0, 9, 120)
    lengths[[20, 41, 42, 43, 99]] = 0
    lengths[60] = 700
    return lengths


@gpu
@pytest.mark.parametrize("use_perm", [False, True])
def test_segsum_ptr_base(use_perm):
    """Slots s0 .. s1 - 1 of a full table as enc_fwd / enc_bwd sum a chunk: ptr = the table's entries from s0 (a device offset
    into the full table), ptr_base = ptr[s0], the rows of the chunk only (src_rows = the chunk's row count, three samples);
    optionally a chunk-local permutation.  Each slot's sum is the sequential float32 sum of its rows, bit for bit."""
    rng = np.random.Generator(np.random.PCG64(21 + use_perm))
    lengths = _full_table(rng)
    ptr = _csr(lengths)
    s0, s1 = 17, 104  # from the middle: empty slots on both sides, the 700-row slot inside
    r0, r1 = int(ptr[s0]), int(ptr[s1])
    n, ns, E, B, W, ld, ldo = r1 - r0, s1 - s0, int(ptr[-1]), 3, 256, 260, 264
    assert r0 > 0 and r1 < E and (lengths[s0:s1] == 0).any()
    # the chunk's B x n rows lead a buffer as large as the whole table's
    base = rng.standard_normal((B * E, ld)).astype(np.float32)
    perm = rng.permutation(n).astype(np.int32) if use_perm else None
    out0 = _prefill(rng, B * ns, ldo, W)
    out = _dev(out0)
    tb, tp = _dev(base), _dev(ptr)
    tperm = _dev(np.concatenate([perm, rng.integers(0, n, E - n).astype(np.int32)])) if use_perm else None  # (chunk's part first)
    _ok(tk.HK.h_segsum_range(_p(tb), ld, W, _at(tp, s0), _p(tperm), n, ns, B, _p(out), ldo, r0, 0, _st()))
    torch.cuda.synchronize()
    want = out0.copy()
    for b in range(B):
        for i in range(ns):
            j = np.arange(ptr[s0 + i], ptr[s0 + i + 1]) - r0
            j = perm[j] if use_perm else j
            want[b * ns + i, :W] = _seq_sum(base[b * n + j, :W])
    _assert_bits(out.cpu().numpy(), want, f"segsum slots {s0}..{s1} ptr_base {r0}")


# ---- launch_segsum accumulated over calls -------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("width", [256, 128])
@pytest.mark.parametrize("n_calls", [2, 3])
@pytest.mark.parametrize("use_perm", [False, True])
def test_segsum_accumulate(use_perm, n_calls, width):
    """Per-segment sums split over row ranges, as dec_bwd sums dPd over decoder chunks: the first call writes, the later ones add.
    Without perm the rows are in segment order (one call boundary inside the 700-row segment) and each call's CSR over all
    segments counts its own rows; with perm (dec_cperm) rows come in any segment order and each call gets the stable segment
    sort of its own rows.  out = (out of the previous call) + (this
    call's sequential float32 sum), bit for bit; a segment a call does not reach gets + 0."""
    rng = np.random.Generator(np.random.PCG64(31 + 2 * n_calls + use_perm + width))
    lengths = _full_table(rng)
    S, E, B = len(lengths), int(_csr(lengths)[-1]), 3
    seg = np.repeat(np.arange(S), lengths)  # the segment of each row
    if use_perm:
        seg = rng.permutation(seg)
    cuts = np.sort(rng.choice(np.arange(1, E), n_calls - 1, replace=False))
    if not use_perm:  # one cut inside the 700-row segment
        start = int(_csr(lengths)[60])
        cuts[0] = start + 333
        cuts = np.sort(cuts)
    bounds = [0, *cuts.tolist(), E]
    ld, ldo = width + 4, width + 8
    out0 = _prefill(rng, B * S, ldo, width)
    out = _dev(out0)
    want = out0.copy()
    keep = []
    for c in range(n_calls):
        e0, e1 = bounds[c], bounds[c + 1]
        ne = e1 - e0
        s = seg[e0:e1]
        order = np.argsort(s, kind="stable").astype(np.int32)  # chunk-local rows, grouped by segment
        cptr = _csr(np.bincount(s, minlength=S))
        rows = rng.standard_normal((B * ne, ld)).astype(np.float32)
        tb, tp = _dev(rows), _dev(cptr)
        tperm = _dev(order) if use_perm else None
        keep += [tb, tp, tperm]
        _ok(tk.HK.h_segsum_range(_p(tb), ld, width, _p(tp), _p(tperm), ne, S, B, _p(out), ldo, 0, int(c > 0), _st()))
        for b in range(B):
            for i in range(S):
                j = order[cptr[i]:cptr[i + 1]] if use_perm else np.arange(cptr[i], cptr[i + 1])
                part = _seq_sum(rows[b * ne + j, :width])
                want[b * S + i, :width] = part if c == 0 else want[b * S + i, :width] + part
    torch.cuda.synchronize()
    _assert_bits(out.cpu().numpy(), want, f"segsum accumulated over {n_calls} calls")


# ---- launch_gather_rows from a range of targets (idx_base) --------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("accumulate", [False, True])
def test_gather_rows_idx_base(accumulate):
    """dec_bwd's d_ep (+)= d_agg_g[dst - r0]: the table holds targets r0 .. r0 + n - 1 only (three samples), the edges' dst
    is a device offset into the full dst array.  Bit for bit; columns >= width keep their bits."""
    rng = np.random.Generator(np.random.PCG64(41 + accumulate))
    n_pts, r0, n, B, W, ld_in, ld_out = 3000, 1211, 503, 3, 256, 260, 264
    dst = np.sort(rng.integers(0, n_pts, 9000)).astype(np.int32)  # edges grouped by target, as the decoder's are
    e0, e1 = int(np.searchsorted(dst, r0)), int(np.searchsorted(dst, r0 + n))
    ne = e1 - e0
    # the chunk's table leads a buffer with room for every target of the full range
    table = rng.standard_normal((B * n + n_pts, ld_in)).astype(np.float32)
    out0 = _prefill(rng, B * ne, ld_out, W, nan_rows=not accumulate)
    out = _dev(out0)
    tt, td = _dev(table), _dev(dst)
    _ok(tk.HK.h_gather_rows_base(_p(tt), ld_in, n, _at(td, e0), ne, W, B, _p(out), ld_out, int(accumulate), r0, _st()))
    torch.cuda.synchronize()
    rows = (np.arange(B)[:, None] * n + (dst[e0:e1] - r0)[None, :]).reshape(-1)
    want = out0.copy()
    want[:, :W] = out0[:, :W] + table[rows, :W] if accumulate else table[rows, :W]
    _assert_bits(out.cpu().numpy(), want, f"gather rows idx_base {r0}")


# ---- empty calls -------------------------------------------------------------------------------------------------------------
@gpu
def test_empty_calls_write_nothing():
    """rows == 0 (a chunk without points, a sample-less call): every launcher returns success and every float keeps its bits."""
    rng = np.random.Generator(np.random.PCG64(51))
    buf0 = _prefill(rng, 64, 264, 256)
    src = _dev(rng.standard_normal((64, 264)).astype(np.float32))
    idx = _dev(np.arange(64, dtype=np.int32))
    ptr = _dev(np.zeros(65, np.int32))
    out = _dev(buf0)
    hk = tk.HK
    _ok(hk.h_permute_rows(_p(src), 264, _p(idx), 0, 64, 102, 2, _p(out), 264, 0, _st()))
    _ok(hk.h_permute_rows(_p(src), 264, _p(idx), 0, 64, 102, 2, _p(out), 264, 1, _st()))
    _ok(hk.h_strided_add(_p(src), 264, _p(out), 264, 0, 78, _st()))
    _ok(hk.h_segsum_range(_p(src), 264, 256, _p(ptr), None, 0, 0, 2, _p(out), 264, 5, 0, _st()))
    _ok(hk.h_segsum_range(_p(src), 264, 256, _p(ptr), None, 0, 0, 2, _p(out), 264, 0, 1, _st()))
    _ok(hk.h_gather_rows_base(_p(src), 264, 0, _p(idx), 0, 256, 2, _p(out), 264, 0, 7, _st()))
    _ok(hk.h_gather_rows_base(_p(src), 264, 0, _p(idx), 0, 256, 2, _p(out), 264, 1, 7, _st()))
    torch.cuda.synchronize()
    _assert_bits(out.cpu().numpy(), buf0, "empty calls")
