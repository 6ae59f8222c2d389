"""-m gpu: the assimilator's narrow row ops of the tensor-core training step, one at a time against float64 (the helpers and bars
of tests/test_gpu_kernels.py).  GraphWeatherAssimilator's 2 observation values make two shapes the forecaster never has:
  * obs_k2    node_encoder Linear 0 on the observation rows: K = 2 (stage 0 rounded up to K0 = 64), N = 256, ReLU, batch 2;
  * dgrad_n2  the data gradient into the observation values: dY [R, 256] . W0 (W^T [2, 256]), N = 2 (one column block of 2);
and its edge encoder reads the 3 observation-graph attributes:
  * edge_k3   edge_encoder Linear 0: K = 3, N = 256, ReLU, batch-shared rows (batch 1).
tc_row_op_chain / tc_column_block accept each of them and run it on the chain kernel's general path (no lean block)."""
import pytest
import torch

import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import FLOAT, RUNS, SIMT, Data, _eps, stream

EXACT = [pytest.param(dict(exact=True, s=s), id=f"int_s{s}") for s in (-40, 0, 20)]
SHAPES = ["obs_k2", "dgrad_n2", "edge_k3"]


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    lib = tk._compile_harness(tmp_path_factory.mktemp("gw_narrow_harness"))
    tk.HK = lib  # (the helpers of test_gpu_kernels call through it)
    return lib


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


def _narrow(name, d, rows=300, batch=2):
    R = rows * batch
    if name == "obs_k2":
        return tk.RowOp(rows, batch, [stream(d.operand(R, 2), rows)], d.weight(256, 2), 2, 256, bias=d.addend(256), relu=True)
    if name == "dgrad_n2":
        return tk.RowOp(rows, batch, [stream(d.operand(R, 256), rows)], d.weight(2, 256), 256, 2)
    if name == "edge_k3":
        return tk.RowOp(rows, 1, [stream(d.operand(rows, 3), rows)], d.weight(256, 3), 3, 256, bias=d.addend(256), relu=True)
    raise KeyError(name)


def _general_path(prec, lean):
    return lean == -1 if prec == SIMT else lean == 0


@gpu
@pytest.mark.parametrize("data", EXACT)
@pytest.mark.parametrize("name", SHAPES)
def test_narrow_row_op_exact(name, data):
    """Exact integers: every precision, both chain settings, reproduce float64 bit for bit."""
    d = Data(9100 + SHAPES.index(name), **data)
    op = _narrow(name, d)
    y64, _, _ = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, _, lean = op.run(prec, nofast)
        tag = f"{name} {tk.PREC_NAME[prec]}{' nofast' if nofast else ''}"
        if not _general_path(prec, lean):
            fails.append(f"{tag}: lean mask {lean}")
        bad = out.double() != y64
        if bad.any():
            fails.append(f"{tag}: {int(bad.sum())} of {y64.numel()} values differ")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("data", FLOAT)
@pytest.mark.parametrize("name", SHAPES)
def test_narrow_row_op_float(name, data):
    d = Data(9200 + SHAPES.index(name), **data)
    op = _narrow(name, d)
    y64, _, c = op.ref()
    fails = []
    for prec, nofast in RUNS:
        out, _, lean = op.run(prec, nofast)
        tag = f"{name} {tk.PREC_NAME[prec]}{' nofast' if nofast else ''}"
        bf, bel = tk.BARS[prec]
        ef, eel = _eps(out, y64, c)
        print(f"{tag}: eps_F {ef:.2e} (bar {bf:.0e}) eps_el {eel:.2e} (bar {bel:.1e}) lean {lean}")
        if not (ef < bf and eel < bel and _general_path(prec, lean)):
            fails.append(f"{tag}: eps_F {ef:.2e} eps_el {eel:.2e} lean {lean}")
    assert not fails, fails


@gpu
@pytest.mark.parametrize("rows,batch", [(1, 1), (63, 2), (129, 3)])
def test_narrow_row_op_row_counts(rows, batch):
    d = Data(93 + rows + batch, exact=True, s=0)
    fails = []
    for name in ("obs_k2", "dgrad_n2"):
        op = _narrow(name, d, rows, batch)
        y64, _, _ = op.ref()
        for prec, nofast in RUNS:
            out, _, _ = op.run(prec, nofast)
            if not torch.equal(out.double(), y64):
                fails.append(f"{name} {tk.PREC_NAME[prec]}{' nofast' if nofast else ''}")
    assert not fails, fails
