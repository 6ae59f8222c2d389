"""RegionalForecaster.forward_regions' union graph (regional._RegionBatch), on the host: the B regions' graphs side by side, each offset
by the regions before it, padded with inert rows to a capacity.  No GPU."""
import numpy as np
import pytest

from graph_weather_b200.dynamic_graph_builder import DynamicGraphBuilder
from graph_weather_b200.regional import _RegionBatch, _RegionGraphs, _pow2


def _box(lat0, lon0, k, step=0.5):
    return [(lat0 + step * a, lon0 + step * b) for a in range(k) for b in range(k)]


A = _box(45.0, 0.0, 8)
CASES = {
    "overlapping": [A, _box(46.0, 1.0, 8)],
    "same_region_twice": [A, list(A)],
    "different_n": [_box(30.0, -20.0, 5), A, _box(-10.0, 120.0, 11)],
    "one_point": [[(52.0, 4.0)], A],
}


def _union(regions, slack=(0, 1, 0)):
    b = DynamicGraphBuilder(resolution=2)
    gs = [_RegionGraphs(b, r) for r in regions]
    n, m, e = (sum(getattr(g, a) for g in gs) for a in ("n_obs", "n_mesh", "n_lat_edges"))
    cap = dict(n_in=_pow2(n + slack[0]), n_mesh=_pow2(m + slack[1]), n_lat_edges=_pow2(max(1, e + slack[2])))
    cap.update(n_out=cap["n_in"], n_dec_edges=cap["n_in"])
    return gs, _RegionBatch(gs, cap)


@pytest.mark.parametrize("case", list(CASES))
def test_union_is_the_regions_offset(case):
    """Every array of the real part equals the regions' own arrays, offset by the preceding regions' points, cells and edges."""
    gs, u = _union(CASES[case])
    po, co, eo = u.point_offsets, u.cell_offsets, u.edge_offsets
    for i, g in enumerate(gs):
        p0, p1, c0, c1, e0, e1 = po[i], po[i + 1], co[i], co[i + 1], eo[i], eo[i + 1]
        np.testing.assert_array_equal(u.mesh_local[p0:p1], g.mesh_local + c0)
        np.testing.assert_array_equal(u.enc_perm[p0:p1], g.enc_perm + p0)
        np.testing.assert_array_equal(u.enc_ptr[c0:c1 + 1], g.enc_ptr + p0)
        np.testing.assert_array_equal(u.enc_attr[p0:p1], g.enc_attr)
        np.testing.assert_array_equal(u.lat_src[e0:e1], g.lat_src + c0)
        np.testing.assert_array_equal(u.lat_dst[e0:e1], g.lat_dst + c0)
        np.testing.assert_array_equal(u.lat_ptr[c0:c1 + 1], g.lat_ptr + e0)
        np.testing.assert_array_equal(u.lat_attr[e0:e1], g.lat_attr)
        np.testing.assert_array_equal(u.dec_src[p0:p1], g.dec_src + c0)
        np.testing.assert_array_equal(u.dec_ptr[p0:p1 + 1], g.dec_ptr + p0)
        np.testing.assert_array_equal(u.h3_indices[c0:c1], g.h3_indices)
    P, C, E = u.cap["n_in"], u.cap["n_mesh"], u.cap["n_lat_edges"]
    assert u.mesh_local.shape == (P,) and u.enc_perm.shape == (P,) and u.enc_ptr.shape == (C + 1,) and u.enc_attr.shape == (P, 2)
    assert u.lat_src.shape == (E,) and u.lat_ptr.shape == (C + 1,) and u.lat_attr.shape == (E, 2) and u.dec_ptr.shape == (P + 1,)
    assert all(a.dtype == np.int32 for a in (u.mesh_local, u.enc_perm, u.enc_ptr, u.lat_src, u.lat_dst, u.lat_ptr, u.dec_ptr))
    # the CSR forms are well formed over the whole capacity
    assert u.enc_ptr[-1] == P and u.lat_ptr[-1] == E and (np.diff(u.enc_ptr) >= 0).all() and (np.diff(u.lat_ptr) >= 0).all()
    assert (np.diff(u.lat_dst) >= 0).all() and sorted(u.enc_perm.tolist()) == list(range(P))
    assert (np.diff(u.mesh_local[u.enc_perm]) >= 0).all()


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("slack", [(0, 1, 0), (37, 9, 100)], ids=["tight", "padded"])
def test_padding_is_inert(case, slack):
    """No padding edge touches a real row; every real row's in-edges are exactly its region's; padding attributes are zero."""
    gs, u = _union(CASES[case], slack)
    n, m, e = u.n_real, u.m_real, u.e_real
    # padding points feed (and are decoded from) padding cells only; real points feed real cells
    assert (u.mesh_local[n:] >= m).all() and (u.mesh_local[:n] < m).all()
    assert not u.enc_attr[n:].any() and not u.lat_attr[e:].any()
    # padding latent edges are self loops on padding cells
    assert (u.lat_src[e:] == u.lat_dst[e:]).all() and (u.lat_src[e:] >= m).all()
    # real cells: their in-edges (latent, encoder) are exactly their region's edges
    for i, g in enumerate(gs):
        c0, c1 = u.cell_offsets[i], u.cell_offsets[i + 1]
        for c in range(c0, c1):
            src = u.lat_src[u.lat_ptr[c]:u.lat_ptr[c + 1]]
            want = g.lat_src[g.lat_ptr[c - c0]:g.lat_ptr[c - c0 + 1]] + c0
            np.testing.assert_array_equal(src, want)
            pts = u.enc_perm[u.enc_ptr[c]:u.enc_ptr[c + 1]]
            np.testing.assert_array_equal(pts, g.enc_perm[g.enc_ptr[c - c0]:g.enc_ptr[c - c0 + 1]] + u.point_offsets[i])
    # padding cells collect no real point and no real edge
    assert (u.enc_perm[u.enc_ptr[m]:] >= n).all() and (u.lat_ptr[m] == e)


def test_table_gradient_groups_rows_by_cell():
    """Rows of a cell shared by several regions are grouped under that cell, in region order; other cells get empty segments."""
    gs, u = _union(CASES["overlapping"])
    H = 5882
    ptr = u.cell_ptr(H)
    assert ptr[-1] == u.m_real
    for cell in np.unique(u.h3_indices):
        rows = u.by_cell[ptr[cell]:ptr[cell + 1]]
        assert (u.h3_indices[rows] == cell).all() and (np.diff(rows) > 0).all()
        assert len(rows) == sum(int((g.h3_indices == cell).sum()) for g in gs)
    shared = set(gs[0].h3_indices.tolist()) & set(gs[1].h3_indices.tolist())
    assert shared  # the boxes overlap: some cells appear twice


def test_capacity_must_hold_the_union():
    gs, u = _union(CASES["different_n"])
    small = dict(u.cap, n_mesh=u.m_real)  # no room for a padding cell
    with pytest.raises(ValueError, match="capacity"):
        _RegionBatch(gs, small)


def test_forward_regions_has_no_host_path():
    import torch

    from graph_weather_b200.regional import RegionalForecasterConfig

    m = RegionalForecasterConfig(feature_dim=9, aux_dim=0, num_blocks=1).build()
    with pytest.raises(RuntimeError, match="no CPU"):
        m.forward_regions([torch.randn(len(A), 9)], [A])
