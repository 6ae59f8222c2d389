"""-m gpu: csrc/gw_graph.cu against the host graph construction, one kernel at a time.

  * launch_obs_graph (the assimilator's per-call observation graph: point location on the H3 lattice, [sin d, cos d, height],
    a stable radix sort by mesh slot, CSR) against graphs.build_encoder_graph on the same float32 inputs, at resolutions 0-3 (even
    and Class III lattices): slot, perm and ptr exactly, the height exactly, sin d / cos d within one float32 ulp (libdevice and
    numpy transcendentals may differ in the last bit).  Points: 10^6 uniform ones, every cell centre and the 12 pentagons, the
    icosahedron vertices and face-edge midpoints, the poles, longitudes beyond +-180, one point repeated 1000 times (ties keep
    observation order), and points pushed toward the boundary between every pair of neighbouring cells.
  * observations at non-finite coordinates: status bit 4 (value 16), slot 0, zero attributes, the other observations unchanged.
  * launch_sort_csr (the training step's by-source CSR): perm = stable argsort, ptr = cumulative bincount."""
import math
import re

import numpy as np
import pytest
import torch

import test_gpu_kernels as tk  # (tests/ is on sys.path: pytest imports its modules by basename)
from test_gpu_kernels import _ok, _p, _st
from graph_weather_b200 import graphs, h3lite


@pytest.fixture(scope="module")
def hk(tmp_path_factory):
    tk.HK = tk._compile_harness(tmp_path_factory.mktemp("gw_graph_harness"))
    return tk.HK


def gpu(f):
    return pytest.mark.gpu(pytest.mark.usefixtures("hk")(f))


_TABLES = {}


def _tables(res):
    """h3lite.device_tables(res) on the GPU, with cell_slot = H - 1 - rank (what gw_plan_set_h3_tables uploads)."""
    if res not in _TABLES:
        tab = h3lite.device_tables(res)
        H = int(tab["n_cells"])
        dev = dict(
            frames=torch.from_numpy(np.ascontiguousarray(tab["frames"], np.float64)).cuda(),
            cell_of=torch.from_numpy(np.ascontiguousarray(tab["cell_of"], np.int32)).cuda(),
            slot=torch.from_numpy((H - 1 - tab["rank"]).astype(np.int32)).cuda(),
            lat=torch.from_numpy(np.ascontiguousarray(tab["cell_lat"], np.float64)).cuda(),
            lng=torch.from_numpy(np.ascontiguousarray(tab["cell_lng"], np.float64)).cuda(),
        )
        _TABLES[res] = (tab, dev)
    return _TABLES[res]


def device_graph(res, llh):
    """llh float32 [n, 3] -> (slot, perm, ptr, attr, status) from launch_obs_graph."""
    tab, dev = _tables(res)
    H, n = int(tab["n_cells"]), llh.shape[0]
    x = torch.from_numpy(np.ascontiguousarray(llh, np.float32)).cuda()
    slot = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    perm = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ptr = torch.full((H + 1,), -1, dtype=torch.int32, device="cuda")
    attr = torch.full((n, 3), float("nan"), device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    _ok(tk.HK.h_obs_graph(res, H, int(tab["lattice_n"]), _p(dev["frames"]), _p(dev["cell_of"]), _p(dev["slot"]), _p(dev["lat"]), _p(dev["lng"]),
                          float(tab["scale"]), float(tab["rot_cos"]), float(tab["rot_sin"]), _p(x), n, H, _p(slot), _p(perm), _p(ptr), _p(attr),
                          _p(status), _st()))  # fmt: skip
    torch.cuda.synchronize()
    return slot.cpu().numpy(), perm.cpu().numpy(), ptr.cpu().numpy(), attr.cpu().numpy(), int(status.item())


def host_graph(res, llh):
    ll = llh.astype(np.float64)  # (the model hands the host construction the float32 observations as float64)
    return graphs.build_encoder_graph(ll[:, :2], res, heights=ll[:, 2])


def _ulps(a, b):
    """|a - b| in float32 ulps (same-sign values)."""
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _latlng_deg(v):
    lat, lng = h3lite._vec_to_geo(v)
    return np.degrees(lat), np.degrees(lng)


def _points(kind, res):
    """float32 [n, 3] observations (lat deg, lon deg, height)."""
    rng = np.random.Generator(np.random.PCG64(res * 10 + len(kind)))
    t = h3lite.table(res)
    if kind == "uniform":
        n = 1_000_000
        lat = np.degrees(np.arcsin(rng.uniform(-1, 1, n)))
        lng = rng.uniform(-180, 540, n)
    elif kind == "centres":  # every cell centre, then the 12 pentagons again
        lat, lng = _latlng_deg(t.center)
        pent = np.nonzero(t.is_pentagon)[0]
        lat, lng = np.concatenate([lat, lat[pent]]), np.concatenate([lng, lng[pent]])
    elif kind == "icosahedron":  # the 12 vertices (the pentagon centres of resolution 0) and the 30 face-edge midpoints
        t0 = h3lite.table(0)
        vert = t0.center[t0.is_pentagon]
        dots = vert @ vert.T
        i, j = np.nonzero(np.triu(dots > 0.4, 1))  # neighbouring vertices: cos 63.4 deg = 0.447
        assert i.size == 30
        mid = vert[i] + vert[j]
        v = np.concatenate([vert, mid / np.linalg.norm(mid, axis=1, keepdims=True)])
        lat, lng = _latlng_deg(v)
    elif kind == "poles_and_meridians":  # both poles at many longitudes; longitudes -180, 180, 360, 540 at many latitudes
        lons = np.arange(-180.0, 541.0, 15.0)
        lats = np.linspace(-89.5, 89.5, 37)
        L4 = np.array([-180.0, 180.0, 360.0, 540.0])
        lat = np.concatenate([np.full(lons.size, 90.0), np.full(lons.size, -90.0), np.repeat(lats, 4)])
        lng = np.concatenate([lons, lons, np.tile(L4, lats.size)])
    elif kind == "repeated":  # one point 1000 times between others: ties must stay in observation order
        lat = rng.uniform(-90, 90, 3000)
        lng = rng.uniform(-180, 180, 3000)
        lat[1000:2000], lng[1000:2000] = 12.345, 67.89
    else:  # "boundaries": the midpoint of every pair of neighbouring cells, pushed slightly toward either cell
        a = np.repeat(np.arange(t.num), 6)
        b = t.nbr.reshape(-1)
        keep = (b >= 0) & (a < b)
        ca, cb = t.center[a[keep]], t.center[b[keep]]
        mid = ca + cb
        pts = []
        for s in (-1e-7, 1e-7, -1e-10, 1e-10):
            v = mid + s * (ca - cb)
            pts.append(v / np.linalg.norm(v, axis=1, keepdims=True))
        lat, lng = _latlng_deg(np.concatenate(pts))
    h = rng.uniform(0, 9000, lat.size)
    return np.stack([lat, lng, h], 1).astype(np.float32)


def _decision_margin(res, llh):
    """Per point, the smallest of the gaps `locate` decides on: best minus second-best face dot product, the distance of q, r, s
    from their rounding boundaries, and the gaps between the rounding errors it compares (float64 restatement of
    h3lite._ResTable.locate / _plane_to_lattice)."""
    c, ex, ey = h3lite._faces()
    v = h3lite._geo_to_vec(np.radians(llh[:, 0].astype(np.float64)), np.radians(llh[:, 1].astype(np.float64)))
    dots = v @ c.T
    top2 = np.sort(dots, axis=1)[:, -2:]
    m_face = top2[:, 1] - top2[:, 0]
    face = np.argmax(dots, axis=1)
    cf = c[face]
    q3 = v / np.sum(v * cf, axis=-1, keepdims=True) - cf
    x, y = np.sum(q3 * ex[face], axis=-1), np.sum(q3 * ey[face], axis=-1)
    s = (h3lite._SQRT7**res) / h3lite._RES0_U_GNOMONIC
    x, y = x * s, y * s
    if res % 2 == 1:
        cr, sr = math.cos(h3lite._M_AP7_ROT_RADS), math.sin(h3lite._M_AP7_ROT_RADS)
        x, y = cr * x + sr * y, -sr * x + cr * y
    b = y / h3lite._SIN60
    a = x + 0.5 * b
    q, r = a - b, b
    s3 = -q - r
    errs = [np.abs(np.rint(u) - u) for u in (q, r, s3)]
    m_round = np.min([np.abs(e - 0.5) for e in errs], axis=0)
    m_cmp = np.min([np.abs(errs[0] - errs[1]), np.abs(errs[0] - errs[2]), np.abs(errs[1] - errs[2])], axis=0)
    return np.minimum(m_face, np.minimum(m_round, m_cmp))


def _nudged_slots(res, llh, idx, eps=1e-8):
    """Host slots of the points idx nudged by +-eps radians in latitude and in longitude (and not at all): [len(idx), 5]."""
    t = h3lite.table(res)
    H = t.num
    lat = np.radians(llh[idx, 0].astype(np.float64))
    lng = np.radians(llh[idx, 1].astype(np.float64))
    out = []
    for dl, dg in ((0, 0), (eps, 0), (-eps, 0), (0, eps), (0, -eps)):
        out.append(H - 1 - t.rank[t.locate(np.clip(lat + dl, -np.pi / 2, np.pi / 2), lng + dg)])
    return np.stack(out, 1)


def _csr_of(slot, H):
    perm = np.argsort(slot, kind="stable").astype(np.int32)
    ptr = np.zeros(H + 1, np.int32)
    np.cumsum(np.bincount(slot, minlength=H), out=ptr[1:])
    return perm, ptr


KINDS = ["uniform", "centres", "icosahedron", "poles_and_meridians", "repeated", "boundaries"]


@gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("res", [0, 1, 2, 3])
def test_obs_graph_vs_host(res, kind):
    llh = _points(kind, res)
    H = h3lite.get_num_cells(res)
    slot, perm, ptr, attr, status = device_graph(res, llh)
    g = host_graph(res, llh)
    assert status == 0, f"status word {status}"
    margin = _decision_margin(res, llh)
    close = np.nonzero(margin <= 1e-9)[0]
    print(f"res {res} {kind}: {llh.shape[0]} points, {close.size} within a decision margin of 1e-9")
    far = margin > 1e-9
    bad = np.nonzero(far & (slot != g.mesh_local))[0]
    assert bad.size == 0, f"{bad.size} points in a different cell, e.g. {llh[bad[:5]].tolist()}"
    if close.size:
        alt = _nudged_slots(res, llh, close)
        ok = (alt == slot[close, None]).any(axis=1)
        assert ok.all(), f"{int((~ok).sum())} near-boundary points in none of the cells on either side, e.g. {llh[close[~ok][:5]].tolist()}"
    if kind == "uniform":  # (the special points may sit on a boundary: the margin check above covers them)
        assert np.array_equal(slot, g.mesh_local), f"{int((slot != g.mesh_local).sum())} cells differ"
    # the CSR follows the device's own slots: perm = stable order by slot (ties in observation order), ptr = cumulative counts
    want_perm, want_ptr = _csr_of(slot, H)
    assert np.array_equal(perm, want_perm) and np.array_equal(ptr, want_ptr)
    if np.array_equal(slot, g.mesh_local):
        assert np.array_equal(perm, g.perm) and np.array_equal(ptr, g.ptr)
    same = slot == g.mesh_local
    assert np.array_equal(attr[:, 2], g.edge_attr[:, 2]), "heights differ"
    u = _ulps(attr[same, :2], g.edge_attr[same, :2])
    assert int(u.max(initial=0)) <= 1, f"sin d / cos d differ by up to {int(u.max())} float32 ulps"


BAD = {"nan_lat": (0, float("nan")), "nan_lon": (1, float("nan")), "inf_lat": (0, float("inf")), "neg_inf_lat": (0, -float("inf")),
       "inf_lon": (1, float("inf")), "neg_inf_lon": (1, -float("inf"))}  # fmt: skip


@gpu
@pytest.mark.parametrize("bad", list(BAD))
def test_obs_graph_non_finite_coordinates(bad):
    """An observation at a non-finite latitude or longitude cannot be located: status bit 4 (value 16), slot 0, zero attributes,
    every slot in range, and the finite observations' slots and the CSR as if that observation sat in slot 0.  (Every face dot
    product of such a point is NaN; on the H100 its NaN lattice coordinates convert to an integer outside the lattice table, so
    h3_locate returns -1.  A conversion to 0 would instead give the valid cell at lattice point (0, 0) of face 0.)"""
    res = 2
    H = h3lite.get_num_cells(res)
    rng = np.random.Generator(np.random.PCG64(5))
    n = 5000
    llh = np.stack([rng.uniform(-90, 90, n), rng.uniform(-180, 180, n), rng.uniform(0, 9000, n)], 1).astype(np.float32)
    col, v = BAD[bad]
    rows = np.array([0, 1234, n - 1])
    llh[rows, col] = v
    slot, perm, ptr, attr, status = device_graph(res, llh)
    assert status & 16, f"status word {status}"
    assert ((slot >= 0) & (slot < H)).all()
    assert (slot[rows] == 0).all() and (attr[rows] == 0).all()
    fin = np.setdiff1d(np.arange(n), rows)
    g = host_graph(res, llh[fin])
    assert np.array_equal(slot[fin], g.mesh_local)
    want = slot.copy()
    want[fin] = g.mesh_local
    want_perm, want_ptr = _csr_of(want, H)
    assert np.array_equal(perm, want_perm) and np.array_equal(ptr, want_ptr)
    assert _ulps(attr[fin, :2], g.edge_attr[:, :2]).max() <= 1 and np.array_equal(attr[fin, 2], g.edge_attr[:, 2])
    # the same points, all finite: no status
    llh[rows, col] = 10.0
    assert device_graph(res, llh)[4] == 0


@gpu
@pytest.mark.parametrize("precision", ["fp32_simt", "fp32"])
def test_assimilator_refuses_non_finite_observation(precision, monkeypatch):
    """GraphWeatherAssimilator with one NaN observation on the GPU raises (device status 16); the next call, with finite
    observations, succeeds and matches the host-built graph."""
    from graph_weather_b200 import GraphWeatherAssimilator
    from oracle import weights

    monkeypatch.setenv("GW_B200_CHECK", "1")  # synchronise and read the status word after every forward
    out_ll = [(float(a), float(b)) for a in range(-90, 90, 10) for b in range(0, 360, 10)]
    sd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=24), 17)
    rng = np.random.Generator(np.random.PCG64(18))
    n = 2000
    obs = np.stack([rng.uniform(-90, 90, n), rng.uniform(-180, 180, n), rng.uniform(0, 9000, n)], 1).astype(np.float32)
    x = weights.make_features(2, n, 2, 17).cuda()
    model = GraphWeatherAssimilator(output_lat_lons=out_ll, analysis_dim=24, precision=precision).cuda()
    model.load_state_dict(sd)
    bad = obs.copy()
    bad[777, 0] = np.nan
    with pytest.raises(RuntimeError) as e:
        model(x, torch.from_numpy(bad).cuda())
    m = re.search(r"device status (\d+)", str(e.value))
    assert m and int(m.group(1)) & 16, str(e.value)
    dev = model(x, torch.from_numpy(obs).cuda()).clone()
    host = model(x, torch.from_numpy(obs))
    err = float((dev - host).abs().max())
    assert err < 1e-5, err  # (tests/test_gpu_parity.py::test_observation_graph_built_on_the_device)


# ---- launch_sort_csr --------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [1, 1000, 3_100_000])
@pytest.mark.parametrize("n_slots", [1, 2, 5882, 8192, 8193])
def test_sort_csr(n_slots, n):
    """perm = np.argsort(src, kind="stable"), ptr = the cumulative bincount over n_slots (empty slots included); 3.1e6 rows is the
    decoder's edge count at 0.25 degree."""
    rng = np.random.Generator(np.random.PCG64(n_slots + n))
    used = rng.choice(n_slots, size=max(1, (2 * n_slots) // 3), replace=False)  # a third of the slots stay empty
    src = used[rng.integers(0, used.size, n)].astype(np.int32)
    if n > 1:
        src[-1] = n_slots - 1  # the top key: every bit of the sort's key range
    ts = torch.from_numpy(src).cuda()
    perm = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ptr = torch.full((n_slots + 1,), -1, dtype=torch.int32, device="cuda")
    _ok(tk.HK.h_sort_csr(_p(ts), n, n_slots, _p(perm), _p(ptr), _st()))
    torch.cuda.synchronize()
    want_perm, want_ptr = _csr_of(src, n_slots)
    assert np.array_equal(perm.cpu().numpy(), want_perm)
    assert np.array_equal(ptr.cpu().numpy(), want_ptr)
