"""Vectorised graph builder (product) == loop-for-loop restatement of the reference construction == reference-made fixture."""
import os

import numpy as np
import pytest

from graph_weather_b200 import graphs
from oracle import restate


def _grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


def _quarter_degree():
    """The ERA5 0.25-degree grid as bench.py builds it: 721 x 1440 points, lat = -90 + 0.25 i (both poles), lon = 0.25 j."""
    lat = -90.0 + 0.25 * np.arange(721)
    lon = 0.25 * np.arange(1440)
    return np.stack(np.meshgrid(lat, lon, indexing="ij"), axis=-1).reshape(-1, 2)


# 10 and 30 degrees; 1 degree (64 800 points); 0.25 degrees (1 038 240 points, up to 9 142 in one mesh cell, 7.27 M decoder edges:
# the loops take about 2 minutes there)
@pytest.mark.parametrize("step", [10, 30, 1, 0.25])
def test_vectorised_equals_loops(step):
    ll = _quarter_degree() if step == 0.25 else _grid(step)
    g = restate.build_forecaster_graphs(ll)
    e = graphs.build_encoder_graph(ll)
    m = graphs.build_mesh_graph()
    d = graphs.build_decoder_graph(ll)
    assert np.array_equal(e.edge_index, g["enc_edge_index"].numpy())
    assert np.array_equal(m.edge_index, g["lat_edge_index"].numpy())
    assert np.array_equal(d.edge_index, g["dec_edge_index"].numpy())
    for a, b in ((e.edge_attr, g["enc_edge_attr"]), (m.edge_attr, g["lat_edge_attr"]), (d.edge_attr, g["dec_edge_attr"])):
        assert np.abs(a - b.numpy()).max() <= 2e-7  # numpy-vectorised vs libm scalar sin/cos: at most an fp32 ulp
    assert m.edge_index.shape == (2, 41162) and m.num_h3 == 5882  # tests/test_model.py:30-31


def test_against_reference_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "forecaster_10deg_b2.npz"))
    ll = _grid(10)
    e = graphs.build_encoder_graph(ll)
    m = graphs.build_mesh_graph()
    d = graphs.build_decoder_graph(ll)
    assert np.array_equal(e.edge_index, z["enc_edge_index"])
    assert np.abs(e.edge_attr - z["enc_edge_attr"]).max() <= 2e-7
    assert np.array_equal(m.edge_index.sum(axis=1), z["lat_edge_index_sum"])
    assert np.abs(m.edge_attr[::53] - z["lat_edge_attr_sub"]).max() <= 2e-7
    assert np.array_equal(d.edge_index[:, ::7], z["dec_edge_index_sub"])
    assert np.abs(d.edge_attr[::7] - z["dec_edge_attr_sub"]).max() <= 2e-7


def test_target_sorted_views():
    m = graphs.build_mesh_graph()
    assert np.all(np.diff(m.dst) >= 0)
    deg = np.diff(m.ptr)
    assert set(deg.tolist()) == {6, 7}
    assert np.array_equal(m.edge_index[1][m.perm], m.dst) and np.array_equal(m.edge_index[0][m.perm], m.src)
    ll = _grid(10)
    e = graphs.build_encoder_graph(ll)
    assert e.ptr[-1] == len(ll) and np.array_equal(np.sort(e.perm), np.arange(len(ll)))
    assert np.all(np.diff(e.mesh_local[e.perm]) >= 0)
    d = graphs.build_decoder_graph(ll)
    assert d.ptr[-1] == d.src.size and set(np.diff(d.ptr).tolist()) <= {6, 7}
    # reference replication offsets assume the highest node id appears in an edge (SURVEY 8(c) caveat)
    assert e.edge_index.max() == len(ll) + 5882 - 1


def test_replicate_matches_reference_formula():
    ei = np.array([[0, 1, 2], [3, 4, 4]])
    r = graphs.replicate_edge_index(ei, 3)
    assert r.shape == (2, 9) and r[1, -1] == 4 + 2 * 4 + 2


def test_validate_lat_lons():
    graphs.validate_lat_lons([(0.0, 0.0), (90.0, 360.0)])
    with pytest.raises(ValueError):
        graphs.validate_lat_lons([(91.0, 0.0)])
