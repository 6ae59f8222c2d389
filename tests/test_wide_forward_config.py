"""No GPU: which trunks take precision "fp32" / "bf16".  The 256-wide trunk with 2 hidden layers runs the fused chains; a trunk at
least 256 wide with one width above 256 (train/run.py's 1024-wide model) runs the layer-by-layer tensor-core forward, with any
number of hidden layers.  Everything else, and every tensor-core train_precision on a wide trunk, is still refused."""
import ctypes
import os

import pytest

import __graft_entry__ as ge
import graph_weather_b200 as gwb
from graph_weather_b200.regional import RegionalForecasterConfig

LL = [(float(a), float(b)) for a in range(-80, 90, 40) for b in range(0, 360, 60)]
WIDE = dict(node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024, hidden_dim_decoder=1024,
            feature_dim=605, aux_dim=40, num_blocks=2)  # fmt: skip


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kw", [WIDE, dict(WIDE, edge_dim=256, hidden_dim_processor_edge=512),
                                dict(WIDE, hidden_layers_processor_node=3, hidden_layers_processor_edge=1)],
                         ids=["run_py", "mixed", "hidden_layers"])  # fmt: skip
def test_wide_trunks_construct(prec, kw):
    gwb.GraphWeatherForecaster(LL, precision=prec, **kw)
    gwb.GraphWeatherForecaster(LL, precision=prec, constraint_type="additive", **kw)
    gwb.GraphWeatherAssimilator(output_lat_lons=LL, precision=prec, **{k: v for k, v in kw.items() if k not in ("feature_dim", "aux_dim")})
    RegionalForecasterConfig(precision=prec, **{k: v for k, v in kw.items() if k != "aux_dim"}).build()
    trunk = dict(node_dim=kw["node_dim"], edge_dim=kw["edge_dim"], hidden_dim_processor_node=kw["hidden_dim_processor_node"],
                 hidden_dim_processor_edge=kw["hidden_dim_processor_edge"])  # fmt: skip
    gwb.Processor(input_dim=kw["node_dim"], edge_dim=kw["edge_dim"], num_blocks=2, precision=prec,
                  **{k: v for k, v in trunk.items() if k not in ("node_dim", "edge_dim")})  # fmt: skip


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("kw", [dict(hidden_layers_processor_node=3), dict(node_dim=128), dict(WIDE, edge_dim=128),
                                dict(WIDE, hidden_dim_processor_node=200)],
                         ids=["256_three_layers", "narrow", "wide_but_one_narrow", "wide_but_hidden_narrow"])  # fmt: skip
def test_other_trunks_still_raise(prec, kw):
    with pytest.raises(ValueError, match="precision"):
        gwb.GraphWeatherForecaster(LL, precision=prec, **kw)


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_training_on_wide_trunks_still_raises(tp):
    with pytest.raises(ValueError, match="train_precision"):
        gwb.GraphWeatherForecaster(LL, precision="fp32", train_precision=tp, **WIDE)


def test_auto_keeps_simt_for_wide_trunks():
    from graph_weather_b200.models import resolve_precision

    dims = dict(node_dim=1024, edge_dim=1024, hidden_node=1024, hidden_edge=1024, hidden_layers_node=2, hidden_layers_edge=2)
    assert resolve_precision("auto", dims, None) == "fp32_simt"


@pytest.mark.skipif(not os.path.exists(ge.NVCC), reason="needs nvcc")
def test_wide_forward_harness_builds_and_links(tmp_path):
    """The kernel tests' harness (tests/kernels/gw_wide_forward_harness.cu) compiles and links against a fresh build, and its HOp
    matches the ctypes mirror."""
    import test_gpu_kernels as tk
    from test_gpu_wide_forward import compile_wide_harness

    lib = compile_wide_harness(tmp_path)
    assert lib.h_sizeof_op() == ctypes.sizeof(tk.HOp)
