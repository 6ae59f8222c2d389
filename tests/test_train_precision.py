"""`train_precision` of GraphWeatherForecaster without a GPU: the default, validation at construction, the Config field, the
save_pretrained / from_pretrained round trip, and a clean sm_90a build of the training kernels (no register spills)."""
import json
import os
import re
import subprocess

import pytest
import torch

import __graft_entry__ as ge

LL = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]


def test_default_is_exact_fp32():
    from graph_weather_b200 import GraphWeatherForecaster

    m = GraphWeatherForecaster(LL, num_blocks=1)
    assert m.train_precision == "fp32_simt"


@pytest.mark.parametrize("tp", ["fp32", "bf16", "fp32_simt"])
def test_accepted_values(tp):
    from graph_weather_b200 import GraphWeatherForecaster

    assert GraphWeatherForecaster(LL, num_blocks=1, train_precision=tp).train_precision == tp


def test_unknown_value_raises():
    from graph_weather_b200 import GraphWeatherForecaster

    with pytest.raises(ValueError, match="train_precision"):
        GraphWeatherForecaster(LL, num_blocks=1, train_precision="fp16")


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_values_need_the_chain_dims(tp):
    from graph_weather_b200 import GraphWeatherForecaster

    with pytest.raises(ValueError, match="train_precision"):
        GraphWeatherForecaster(LL, num_blocks=1, hidden_dim_processor_edge=64, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        GraphWeatherForecaster(LL, num_blocks=1, hidden_layers_processor_node=3, train_precision=tp)
    # the exact-fp32 training path covers other sizes
    GraphWeatherForecaster(LL, num_blocks=1, hidden_dim_processor_edge=64, train_precision="fp32_simt")


def test_config_carries_the_value():
    from graph_weather_b200.models import GraphWeatherForecasterConfig

    assert GraphWeatherForecasterConfig(lat_lons=LL).train_precision == "fp32_simt"
    m = GraphWeatherForecasterConfig(lat_lons=LL, num_blocks=1, train_precision="bf16").build()
    assert m.train_precision == "bf16"


def test_hub_round_trip_keeps_it(tmp_path):
    from graph_weather_b200 import GraphWeatherForecaster

    m = GraphWeatherForecaster(LL, num_blocks=1, train_precision="bf16")
    m.save_pretrained(tmp_path / "m")
    assert json.load(open(tmp_path / "m" / "config.json"))["train_precision"] == "bf16"
    m2 = GraphWeatherForecaster.from_pretrained(tmp_path / "m")
    assert m2.train_precision == "bf16"
    assert all(torch.equal(v, m2.state_dict()[k]) for k, v in m.state_dict().items())


def _ptxas_report(src, tmp_path):
    out = tmp_path / (os.path.basename(src) + ".o")
    r = subprocess.run([ge.NVCC, *ge.FLAGS, "-Xptxas", "-v", "-c", os.path.join(ge.CSRC, src), "-o", str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout + r.stderr


@pytest.mark.skipif(not os.path.exists(ge.NVCC), reason="needs nvcc")
def test_build_and_no_spills_in_the_training_kernels(tmp_path):
    ge.build()
    import graph_weather_b200  # noqa: F401

    # every instance of the weight-gradient kernel keeps its accumulator and staging registers without spilling, and ptxas keeps
    # its wgmma asynchronous (the chain kernel's training epilogue parts are run-time flags of its existing general path)
    for src, kernel in (("gw_wgrad_tc.cu", "gw_wgrad_tc_kernel"),):
        rep = _ptxas_report(src, tmp_path)
        blocks = re.split(r"ptxas info\s+: Compiling entry function", rep)
        seen = 0
        for b in blocks:
            name = b.split("'")[1] if "'" in b else ""
            if kernel not in name:
                continue
            seen += 1
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
            assert m and m.group(1) == "0" and m.group(2) == "0", (name, b[:400])
            assert "serialized" not in b, (name, "wgmma serialised")
        assert seen == 8, (src, seen)  # {fp16 split, bf16} x NW in {64, 128, 192, 256}
