"""The training step on a point set whose mesh cells collect hundreds of points, against the fp64 autograd oracle.

On the 10-degree grid and on a few hundred random observations most H3 mesh cells receive 0-2 points, so every encoder segment sum
and every per-source decoder sum of the backward (dPm, dPd) adds at most a few dozen rows; on a real grid a polar cell collects
thousands.  Here the forecaster trains on the 10-degree grid followed by a 6 x 6.2 degree patch at 0.1-degree spacing at mid-latitude
(4368 points): a few mesh cells each hold 400-1000 points and a mesh node is the source of up to 3502 decoder edges, and the
loss's cos(lat) weights keep the patch's rows in the loss.  Batch 2.
  * the case itself: the longest segments, the oracle's replicated graphs offset each sample by the node count, and the points
    tile NormalizedMSELoss's latitude weights;
  * every train precision, taped and bounded, against the oracle with the bars of tests/test_gpu_training.py,
    tests/test_gpu_train_precision.py and tests/test_gpu_lean_training.py;
  * the bounded step at chunk sizes 1, 37, 500 and all points (at 37 every dense mesh slot is an encoder chunk larger than the
    budget, and decoder chunks cut through the patch) against the taped step: the forward bit for bit, the gradients within 1e-5
    in fp32_simt (bf16: measured bars, as in the 1-degree comparison);
  * GraphWeatherAssimilator on 2000 observations in five tight clusters, taped and bounded, against its oracle."""
import collections

import numpy as np
import pytest
import torch

import __graft_entry__ as ge
import test_gpu_assimilator_training as ta  # (tests/ is on sys.path: pytest imports its modules by basename)
from training_oracle import ILL_CONDITIONED, check_bf16_bars, check_fp32_bars, forecaster_oracle_step, grid, rel_norm, train_step


def dense_points():
    """The 10-degree grid, then 60 x 62 points 0.1 degree apart from (45.05N, 10E).  NormalizedMSELoss gives node k the weight of
    unique latitude k // (nodes / unique latitudes), so the node count must be a multiple of the unique latitudes' (18 + 60 = 78:
    62 columns, not 60); the patch's nodes then take the weights of latitudes 30 .. 80 degrees, most of them 45 .. 51."""
    return grid(10) + [(round(45.05 + 0.1 * i, 2), round(10.0 + 0.1 * j, 1)) for i in range(60) for j in range(62)]


def _longest(index_row):
    return max(collections.Counter(index_row.tolist()).values())


def test_the_case_has_dense_cells():
    """No GPU needed.  The longest encoder segment (points of one mesh cell) and the longest per-source decoder segment (edges
    out of one mesh node) hold >= 300 rows, and the oracle's _replicate offset (max index + 1) is the node count of both graphs
    (see tests/test_gpu_parity.py::test_irregular_points_against_oracle: otherwise the oracle's samples >= 1 are misaligned)."""
    from oracle import restate

    ll = dense_points()
    g = restate.build_forecaster_graphs(ll)
    n_nodes = len(ll) + g["num_h3"]
    enc, dec = g["enc_edge_index"], g["dec_edge_index"]
    enc_seg, dec_seg = _longest(enc[1]), _longest(dec[0])
    print(f"{len(ll)} points, {g['num_h3']} mesh nodes: longest encoder segment {enc_seg}, longest decoder per-source segment {dec_seg}")
    assert enc_seg >= 300 and dec_seg >= 300
    assert int(enc.max()) + 1 == n_nodes and int(dec.max()) + 1 == n_nodes
    assert len(ll) % len({lat for lat, _ in ll}) == 0


@pytest.fixture(scope="module")
def _built():
    ge.build()


@pytest.fixture(scope="module")
def case(_built):
    """(lat_lons, state_dict, features, target, variances), seeded."""
    from oracle import weights

    ll = dense_points()
    sd = weights.make_state_dict(weights.forecaster_shapes(), 23)
    x = weights.make_features(2, len(ll), 102, 23)
    rng = np.random.Generator(np.random.PCG64(23))
    target = torch.from_numpy(rng.standard_normal((2, len(ll), 78)).astype(np.float32))
    var = rng.uniform(0.5, 2.0, 78).astype(np.float32).tolist()
    return ll, sd, x, target, var


@pytest.fixture(scope="module")
def oracle_steps(case):
    """The oracle step on the case in fp32 and in fp64 (the slow part: computed once per module)."""
    ll, sd, x, target, var = case
    return [forecaster_oracle_step(sd, ll, x, target, var, dt) for dt in (torch.float32, torch.float64)]


def _step(case, tp, lean, loss_fn=None):
    """One training step of a fresh forecaster under NormalizedMSELoss (or loss_fn): (out, loss, d features, {name: grad})."""
    from graph_weather_b200 import GraphWeatherForecaster, NormalizedMSELoss

    ll, sd, x, target, var = case
    model = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=lean).cuda().train()
    model.load_state_dict(sd)
    res = train_step(model, loss_fn or NormalizedMSELoss(var, ll, normalize=True), x, target)
    assert model._train_engine.plan.train_only == lean and model._train_engine.resolved_precision == tp
    return res


def _check(tp, lean, ours, ref32, ref64):
    """The bars of the 10-degree case, but with fp32 mode's 2e-3 floor for fp32_simt too: one decoder node-MLP unit within
    rounding of zero takes the other side of its ReLU than in fp64 (measured on an H100 80GB HBM3, 700 W: 2.3e-4 max-relative
    error on decoder.graph_processor.blocks.0.node_model.node_mlp.model.2 against the fp32 oracle's 8.4e-8, the same in the taped
    and the bounded step, whose forwards are bit-identical; every other parameter within 10x the oracle's error + 2e-5)."""
    tag = f"dense cells {tp} {'bounded' if lean else 'taped'}"
    if tp == "bf16":  # tests/test_gpu_train_precision.py (taped), tests/test_gpu_lean_training.py (bounded)
        check_bf16_bars(ours, ref32, ref64, n_params=215, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=None if lean else 0.999,
                        tag=tag)  # fmt: skip
    else:  # tests/test_gpu_training.py (fp32_simt taped: the median too), tests/test_gpu_train_precision.py, tests/test_gpu_lean_training.py
        check_fp32_bars(ours, ref32, ref64, n_params=215, floor=2e-3, feat_floor=False, median=tp == "fp32_simt" and not lean, ill=None,
                        skip_zero=False, norm_bar=None, tag=tag)  # fmt: skip


@pytest.mark.gpu
@pytest.mark.training
@pytest.mark.parametrize("lean", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_gradients_match_the_oracle(case, oracle_steps, monkeypatch, tp, lean):
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    _check(tp, lean, _step(case, tp, lean), *oracle_steps)


# 1: every encoder chunk one mesh slot, every decoder chunk one point; 37: every dense slot a chunk of its own, larger than the
# budget, and decoder chunks that cut through the patch; 500; one chunk for everything
CHUNKS = ["1", "37", "500", str(len(dense_points()))]


@pytest.mark.gpu
@pytest.mark.training
@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_bounded_step_equals_the_taped_step(case, monkeypatch, tp, chunk):
    """Under torch's MSELoss, which weights every point alike: NormalizedMSELoss gives the first 56 points cos(-90 deg) ~ 6e-17
    (its weights follow the position of a point), so whatever the first decoder chunks add to dPd would not show.
    Gradients: fp32_simt within 1e-5 of the taped step (measured <= 3.6e-6).  bf16 as in tests/test_gpu_lean_training.py::
    test_one_degree_against_the_taped_step: where decoder chunks cut a mesh node's edges (chunks 37 and 500), dPd differs from
    the taped step's in its last bits, which flips the bf16 rounding of single operands upstream, and the tensors summed over the
    whole graph magnify it.  Measured on an H100 80GB HBM3 (700 W) at chunks 37 and 500: encoder.h3_nodes 4.7e-3,
    encoder.node_encoder.model.0.weight 4.4e-3, worst other parameter 1.4e-3 (the encoder block's edge layer 0, whose mesh
    half sums the dense cells' rows), features 2.1e-5; <= 3.7e-6 at chunks 1 and 4368, whose per-source sums add the taped
    step's rows in its order."""
    mse = torch.nn.functional.mse_loss
    out_t, loss_t, gx_t, g_t = _step(case, tp, False, mse)
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", chunk)
    out_l, loss_l, gx_l, g_l = _step(case, tp, True, mse)
    assert torch.equal(out_l, out_t)
    assert loss_l == loss_t
    errs = sorted(((rel_norm(g_l[k], g), k) for k, g in g_t.items() if float(g.norm()) > 0), reverse=True)
    ef = rel_norm(gx_l, gx_t)
    print(f"dense cells {tp} chunk {chunk}: worst norm-relative gradient differences to the taped step {errs[:3]}; features {ef:.2e}")
    for e, k in errs:
        bar = 1e-5 if tp == "fp32_simt" else (1e-2 if k.startswith(ILL_CONDITIONED) else 3e-3)
        assert e <= bar, (k, e)
    assert ef <= (1e-5 if tp == "fp32_simt" else 1e-4), ef


# ---- GraphWeatherAssimilator: observations in a few cells ---------------------------------------------------------------------
CLUSTERS = [(50.3, 10.4), (-31.0, 141.2), (4.6, 251.7), (68.2, 300.5), (-58.9, 61.3)]


def clustered_obs(per_cluster, seed):
    """per_cluster observations uniform within +-0.6 degree of each centre of CLUSTERS (lat, lon, height in [0, 1))."""
    rng = np.random.Generator(np.random.PCG64(seed))
    rows = [np.stack([rng.uniform(a - 0.6, a + 0.6, per_cluster), rng.uniform(b - 0.6, b + 0.6, per_cluster), rng.uniform(0, 1, per_cluster)], 1)
            for a, b in CLUSTERS]  # fmt: skip
    return torch.from_numpy(np.concatenate(rows).astype(np.float32))


@pytest.fixture(scope="module")
def assim_case(_built):
    from oracle import restate, weights

    out_ll = ta._out_grid()
    sd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=ta.ANALYSIS_DIM), 41)
    setup = (out_ll, sd, restate.build_assimilator_graphs(out_ll))
    obs = clustered_obs(400, 91)
    x = weights.make_features(1, obs.shape[0], 2, 91)
    target = torch.randn(1, len(out_ll), ta.ANALYSIS_DIM, generator=torch.Generator().manual_seed(91))
    return (setup, x, obs, target, *ta._oracle(sd, setup[2], x, obs, target))


@pytest.mark.gpu
@pytest.mark.training
@pytest.mark.parametrize("lean", [False, True], ids=["taped", "bounded"])
@pytest.mark.parametrize("tp", ["fp32_simt", "bf16"])
def test_assimilator_on_clustered_observations(assim_case, monkeypatch, tp, lean):
    from oracle import restate

    setup, x, obs, target, ref32, ref64 = assim_case
    ei, _ = restate.assimilator_input_graph(obs, setup[2]["base_h3_grid"])
    seg = _longest(ei[1])
    print(f"{obs.shape[0]} observations: longest encoder segment {seg}")
    assert seg >= 300
    monkeypatch.setenv("GW_B200_TRAIN_CHUNK", "37")
    model = ta._model(setup, tp, lean)
    res = ta._step(model, x, obs, target)
    assert model._train_engine.plan.train_only == lean
    if tp == "bf16":
        # Below tests/test_gpu_assimilator_training.py's bf16 bars (0.99 / 0.98, features 0.98): a mesh node that sums 400
        # messages holds values far above the rest, and bf16's error follows them.  Measured on an H100 80GB HBM3 (700 W), taped:
        # features 0.9702, worst parameter 0.9831 (processor block 6, edge layer 0), next 0.9892; fp32_simt on the same case
        # stays within the fp32 bars (features 2.5e-5 max-relative against the fp32 oracle's 4.7e-4).
        check_bf16_bars(res, ref32, ref64, n_params=214, cos_bar=0.97, ill_cos_bar=0.97, feat_cos=0.95, total_cos=None, tag="clustered obs")
    else:
        ta._check(tp, res, ref32, ref64, "clustered obs")

