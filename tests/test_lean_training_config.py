"""The bounded-memory training step without a GPU: its C ABI additions are declared and bound, `use_checkpointing` travels from
the config to the forecaster and selects a training-only plan for training alone, and the kernels the chunks use build for
sm_90a without register spills."""
import os
import re
import subprocess

import pytest

import __graft_entry__ as ge

LL = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]


def test_abi_symbols_are_declared_and_bound():
    from graph_weather_b200 import _capi

    declared = _capi.header_symbols()
    for name in ("gw_plan_create_train", "gw_train_peak_bytes"):
        assert name in declared and name in _capi._SIGNATURES
    with open(_capi.HEADER_PATH) as f:
        assert "#define GW_ABI_VERSION 2" in f.read()


@pytest.mark.parametrize("flag", [False, True])
def test_config_round_trip(flag):
    from graph_weather_b200 import GraphWeatherForecasterConfig

    model = GraphWeatherForecasterConfig(lat_lons=LL, num_blocks=2, use_checkpointing=flag).build()
    assert model.use_checkpointing is flag
    assert model._training_engine().train_only is flag
    assert model._engine.train_only is False  # inference keeps its plan


@pytest.mark.skipif(not os.path.exists(ge.NVCC), reason="needs nvcc")
def test_chunk_kernels_do_not_spill(tmp_path):
    out = tmp_path / "gw_simt.o"
    r = subprocess.run([ge.NVCC, *ge.FLAGS, "-Xptxas", "-v", "-c", os.path.join(ge.CSRC, "gw_simt.cu"), "-o", str(out)], capture_output=True,
                       text=True)  # fmt: skip
    assert r.returncode == 0, r.stderr[-4000:]
    seen = set()
    for b in re.split(r"ptxas info\s+: Compiling entry function", r.stdout + r.stderr):
        name = b.split("'")[1] if "'" in b else ""
        for k in ("gw_segsum_kernel", "gw_gather_rows_kernel", "gw_permute_rows_kernel"):
            if k in name:
                seen.add(k)
                m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
                assert m and m.group(1) == "0" and m.group(2) == "0", (name, b[:400])
    assert len(seen) == 3
