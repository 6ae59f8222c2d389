"""Training configurations wider than 256 without a GPU: the reference's ERA5 models construct with the train precisions that
cover them (train/run_fulll.py: 597 + 24 features on the default 256-wide trunk, every precision; train/run.py: 1024-wide node /
edge / hidden / decoder widths, exact fp32 only), and the wide LayerNorm backward builds for sm_90a without register spills."""
import os
import re
import subprocess

import pytest

import __graft_entry__ as ge

LL = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]
WIDE = dict(feature_dim=605, aux_dim=40, node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024,
            hidden_dim_decoder=1024, num_blocks=2)  # fmt: skip


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_run_fulll_config_constructs_with_every_train_precision(tp):
    from graph_weather_b200 import GraphWeatherForecaster

    m = GraphWeatherForecaster(LL, feature_dim=597, num_blocks=6, train_precision=tp)
    assert m.train_precision == tp and m.output_dim == 597


def test_1024_wide_config_trains_in_exact_fp32_only():
    from graph_weather_b200 import GraphWeatherForecaster

    assert GraphWeatherForecaster(LL, train_precision="fp32_simt", **WIDE).train_precision == "fp32_simt"
    for tp in ("fp32", "bf16"):  # tensor-core training is built for the 256-wide trunk
        with pytest.raises(ValueError, match="train_precision"):
            GraphWeatherForecaster(LL, train_precision=tp, **WIDE)


@pytest.mark.skipif(not os.path.exists(ge.NVCC), reason="needs nvcc")
def test_wide_layernorm_backward_does_not_spill(tmp_path):
    out = tmp_path / "gw_simt.o"
    r = subprocess.run([ge.NVCC, *ge.FLAGS, "-Xptxas", "-v", "-c", os.path.join(ge.CSRC, "gw_simt.cu"), "-o", str(out)], capture_output=True,
                       text=True)  # fmt: skip
    assert r.returncode == 0, r.stderr[-4000:]
    seen = 0
    for b in re.split(r"ptxas info\s+: Compiling entry function", r.stdout + r.stderr):
        name = b.split("'")[1] if "'" in b else ""
        if "gw_ln_bwd_wide_kernel" not in name:
            continue
        seen += 1
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", (name, b[:400])
    assert seen == 2  # J = 16 (N <= 512) and J = 32 (N <= 1024)
