"""The C-ABI shared library loads and exports every symbol include/gw_b200.h declares (no compute without a GPU),
and the host-side modules keep the reference's state_dict contract."""
import os

import pytest
import torch

import __graft_entry__ as ge
from graph_weather_b200 import _capi


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def test_library_exports_header_symbols():
    lib = _capi.load()
    syms = _capi.header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), s
    assert lib.gw_abi_version() == 1
    assert [lib.gw_timing_tag_name(i).decode() for i in range(lib.gw_timing_num_tags())][:3] == ["const", "enc_grid", "enc_mesh"]


def test_no_cpu_path():
    """The product path must fail loudly instead of computing on the host."""
    from graph_weather_b200 import GraphWeatherForecaster

    ll = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]
    m = GraphWeatherForecaster(ll)
    with pytest.raises(RuntimeError, match="no CPU"):
        m(torch.randn(1, len(ll), 102))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            _capi.Plan("cuda:0", n_in=1, n_out=1, n_mesh=1, n_lat_edges=1, n_dec_edges=1, in_dim=1, enc_edge_attr_dim=2, out_dim=1,
                       residual_dim=0, node_dim=8, edge_dim=8, hidden_node=8, hidden_edge=8, hidden_layers_node=2,
                       hidden_layers_edge=2, hidden_dec=8, hidden_layers_dec=2, num_blocks=1, precision=0, max_batch=1)  # fmt: skip


def test_state_dict_contract_matches_oracle_shapes():
    from graph_weather_b200 import GraphWeatherAssimilator, GraphWeatherForecaster
    from oracle import weights

    ll = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]
    m = GraphWeatherForecaster(ll)
    sd = m.state_dict()
    shapes = weights.forecaster_shapes()
    assert list(sd.keys()) == list(shapes.keys())
    assert all(tuple(sd[k].shape) == tuple(shapes[k]) for k in sd)
    a = GraphWeatherAssimilator(output_lat_lons=ll, analysis_dim=24)
    shapes = weights.forecaster_shapes(assimilator=True, output_dim=24)
    assert list(a.state_dict().keys()) == list(shapes.keys())
    # the key the survey quotes as part of the drop-in contract
    assert tuple(sd["processor.graph_processor.blocks.3.edge_model.edge_mlp.model.0.weight"].shape) == (256, 768)


def test_same_seed_same_init_as_reference(golden_dir):
    """torch.manual_seed(42); GraphWeatherForecaster(ll) initialises every parameter exactly as the reference does: the keys,
    shapes, a seeded sample of 16 values per tensor and the float64 sums of each tensor and of its magnitudes, recorded from the
    reference's own constructor by tests/golden/make_golden.py."""
    import json

    import numpy as np

    from graph_weather_b200 import GraphWeatherForecaster

    z = np.load(os.path.join(golden_dir, "reference_init_seed42.npz"))
    cfg = json.loads(str(z["config"]))
    ll = [(float(a), float(b)) for a in range(-90, 90, cfg["grid_step"]) for b in range(0, 360, cfg["grid_step"])]
    torch.manual_seed(cfg["seed"])
    mine = GraphWeatherForecaster(ll).state_dict()
    assert list(mine.keys()) == cfg["keys"]
    rng = np.random.default_rng(0)
    for i, k in enumerate(cfg["keys"]):
        assert list(mine[k].shape) == cfg["shapes"][i], k
        v = mine[k].detach().cpu().numpy().ravel().astype(np.float32)
        idx = np.sort(rng.choice(v.size, min(v.size, 16), replace=False))
        assert np.array_equal(v[idx], z["samples"][i][: idx.size]), k
        assert np.sum(v, dtype=np.float64) == z["sums"][i][0] and np.sum(np.abs(v), dtype=np.float64) == z["sums"][i][1], k


def test_graphcast_wrapper_contract():
    from graph_weather_b200 import GraphCast, GraphCastConfig
    from oracle import weights

    ll = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]
    m = GraphCast(ll, efficient_batching=True)
    shapes = weights.forecaster_shapes(feature_dim=78, aux_dim=0, hidden_dim_decoder=256)
    assert list(m.state_dict().keys()) == list(shapes.keys())
    GraphCastConfig.balanced_checkpointing(m)
    assert (m._checkpoint_encoder, m._checkpoint_processor_segments, m._checkpoint_decoder) == (True, -1, True)
    GraphCastConfig.full_checkpointing(m)
    assert m._checkpoint_model and not m._checkpoint_encoder


def test_perm32_feature_order_contract():
    """The weight packing (csrc/gw_pack.cu, perm32_f) and the chain kernel (csrc/gw_tc3.cu) agree on this map: inside every group
    of 32 features, packed position a = 8g + 2c + e holds logical feature f(a) = 8c + 2g + e.  It must be a permutation, and the
    eight accumulator columns the wgmma fragment gives lane t in a 32-column step -- 8g + 2(t % 4) + e, g < 4, e < 2 -- must be eight
    consecutive logical features starting at 8 (t % 4), which is what makes the 128-byte row segments of the epilogue legal."""

    def f(a):
        return (a & ~31) | (8 * ((a >> 1) & 3) + 2 * ((a >> 3) & 3) + (a & 1))

    assert sorted(f(a) for a in range(256)) == list(range(256))
    for group in (0, 32, 224):
        for c in range(4):
            cols = [group + 8 * g + 2 * c + e for g in range(4) for e in range(2)]
            assert [f(x) for x in cols] == [group + 8 * c + i for i in range(8)]
    src = open(os.path.join(ge.ROOT, "graph_weather_b200", "csrc", "gw_pack.cu")).read()
    assert "(8 * ((a >> 1) & 3) + 2 * ((a >> 3) & 3) + (a & 1))" in src  # the formula the test restates
