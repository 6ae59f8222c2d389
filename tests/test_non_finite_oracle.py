"""The non-finite model cases of tests/test_gpu_non_finite_models.py, and a CPU check that each is worth comparing against.

Each case puts one NaN, +inf or -inf into one input of sample 1 of a seeded 10-degree, batch-2 case (GraphWeatherForecaster,
GraphCast), or into one observation value of the assimilator's batch-1 case.  The GPU tests compare the NaN / inf pattern of the
library's outputs with the CPU oracle's (the reference arithmetic, oracle/restate.py).  That comparison proves something only if
the oracle's pattern is neither empty nor everything: the poisoned sample must be partly NaN, and the other sample must stay
finite.  This file checks that for every case, without a GPU."""
import numpy as np
import pytest
import torch

from training_oracle import assimilator_oracle_step, forecaster_oracle_step, grid

POINT = 345  # the lat/lon point (of 648 on the 10-degree grid) whose features are poisoned
VALUES = {"nan": float("nan"), "inf": float("inf"), "-inf": float("-inf")}
# (value, feature column): column 5 lies inside the 78 columns the decoder adds back (the residual), column 90 is an auxiliary
# feature that reaches the output only through the encoder
FORECASTER_CASES = [("nan", 5), ("nan", 90), ("inf", 5), ("-inf", 5), ("inf", 90), ("-inf", 90)]
ASSIM_DIM, N_OBS, OBS = 24, 300, 123  # the assimilator case: analysis width, observation count, the poisoned observation

_CACHE = {}


def _cached(key, build):
    if key not in _CACHE:
        with torch.enable_grad():  # (the oracle steps differentiate, also when called from an inference test)
            _CACHE[key] = build()
    return _CACHE[key]


def forecaster_base(model="forecaster"):
    """(lat_lons, state_dict, features, target, variances) of the seeded 10-degree, batch-2 case: the forecaster's default
    shapes (78 + 24 features), or GraphCast's (78 features, a 256-wide decoder)."""

    def build():
        from oracle import weights

        ll = grid(10)
        kw = dict(feature_dim=78, aux_dim=0, hidden_dim_decoder=256) if model == "graphcast" else {}
        F, A = 78, (0 if model == "graphcast" else 24)
        sd = weights.make_state_dict(weights.forecaster_shapes(**kw), 21)
        x = weights.make_features(2, len(ll), F + A, 21)
        rng = np.random.Generator(np.random.PCG64(21))
        target = torch.from_numpy(rng.standard_normal((2, len(ll), F)).astype(np.float32))
        var = rng.uniform(0.5, 2.0, F).astype(np.float32).tolist()
        return ll, sd, x, target, var

    return _cached(("base", model), build)


def poisoned(x, value, col):
    """x with VALUES[value] at sample 1, point POINT, feature column col."""
    xp = x.clone()
    xp[1, POINT, col] = VALUES[value]
    return xp


def forecaster_oracle(model, value, col):
    """The fp32 oracle step on the poisoned features: (out, loss, d features, {name: grad})."""

    def build():
        ll, sd, x, target, var = forecaster_base(model)
        return forecaster_oracle_step(sd, ll, poisoned(x, value, col), target, var, torch.float32)

    return _cached(("oracle", model, value, col), build)


def _out_grid():
    return [(float(lat), float(lon)) for lat in range(-90, 90, 5) for lon in range(0, 360, 5)]


def assimilator_base():
    """(output lat/lons, state_dict, static graphs, observation values [1, N_OBS, 2], lat/lon/heights [N_OBS, 3], target): the
    README's assimilator (5-degree output grid, analysis width 24) on N_OBS seeded observations, batch 1."""

    def build():
        from oracle import restate, weights

        out_ll = _out_grid()
        sd = weights.make_state_dict(weights.forecaster_shapes(assimilator=True, output_dim=ASSIM_DIM), 41)
        rng = np.random.Generator(np.random.PCG64(51))
        obs = torch.from_numpy(np.stack([rng.uniform(-90, 90, N_OBS), rng.uniform(0, 360, N_OBS), rng.uniform(0, 1, N_OBS)], 1).astype(np.float32))
        x = weights.make_features(1, N_OBS, 2, 51)
        target = torch.randn(1, len(out_ll), ASSIM_DIM, generator=torch.Generator().manual_seed(51))
        return out_ll, sd, restate.build_assimilator_graphs(out_ll), x, obs, target

    return _cached(("assim",), build)


def assimilator_poisoned():
    x = assimilator_base()[3].clone()
    x[0, OBS, 0] = float("nan")
    return x


def assimilator_oracle():
    def build():
        out_ll, sd, g, _, obs, target = assimilator_base()
        return assimilator_oracle_step(sd, g, assimilator_poisoned(), obs, target, torch.float32)

    return _cached(("assim oracle",), build)


def _partly_nan(t):
    n = torch.isnan(t)
    return bool(n.any()) and not bool(n.all())


@pytest.mark.parametrize("value,col", FORECASTER_CASES)
def test_forecaster_case_is_informative(value, col):
    out, loss, gx, _ = forecaster_oracle("forecaster", value, col)
    assert _partly_nan(out[1]), "the poisoned sample's forecast must be partly NaN"
    assert bool(torch.isfinite(out[0]).all()), "the clean sample's forecast must stay finite"
    assert _partly_nan(gx[1]) and bool(torch.isfinite(gx[0]).all()), "the feature gradient must be partly NaN in sample 1 only"
    assert not np.isfinite(loss)


def test_graphcast_case_is_informative():
    out, _, gx, _ = forecaster_oracle("graphcast", "nan", 5)
    assert _partly_nan(out[1]) and bool(torch.isfinite(out[0]).all())
    assert _partly_nan(gx[1]) and bool(torch.isfinite(gx[0]).all())


def test_assimilator_case_is_informative():
    out, _, gx, _ = assimilator_oracle()
    assert _partly_nan(out), "one NaN observation value must make part of the analysis NaN"
    assert _partly_nan(gx)
