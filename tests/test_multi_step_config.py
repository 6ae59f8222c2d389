"""multi_step() on the CPU: what needs no device."""
import pytest


def test_assimilator_has_no_multi_step():
    """The assimilator's observation graph belongs to its training plan, not to a forward: several of its forwards cannot stay
    differentiable at once, so its window refuses to open."""
    from graph_weather_b200 import GraphWeatherAssimilator

    lat_lons = [(float(lat), float(lon)) for lat in range(-90, 90, 30) for lon in range(0, 360, 30)]
    model = GraphWeatherAssimilator(output_lat_lons=lat_lons, num_blocks=1)
    with pytest.raises(NotImplementedError, match="multi_step"):
        with model.multi_step():
            pass


def test_window_nests_and_closes():
    """The window is a counter on the module: it nests, and leaving it (also by an exception) restores the state outside."""
    from graph_weather_b200 import GraphWeatherForecaster

    lat_lons = [(float(lat), float(lon)) for lat in range(-90, 90, 30) for lon in range(0, 360, 30)]
    model = GraphWeatherForecaster(lat_lons, num_blocks=1)
    assert not model.__dict__.get("_multi_step", 0)
    with model.multi_step():
        with model.multi_step() as m:
            assert m is model and model.__dict__["_multi_step"] == 2
        assert model.__dict__["_multi_step"] == 1
    with pytest.raises(ValueError):
        with model.multi_step():
            raise ValueError("inside")
    assert model.__dict__["_multi_step"] == 0
