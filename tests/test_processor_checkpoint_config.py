"""Processor segments on the CPU: the checkpoint controls that set them, and the binding that hands them to the library."""
import ctypes

import pytest

import __graft_entry__ as ge


def _grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


def _wrappers():
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator, GraphWeatherForecaster
    from graph_weather_b200.regional import RegionalForecasterConfig

    ll = _grid(30)
    return [GraphWeatherForecaster(ll, num_blocks=2), GraphWeatherAssimilator(output_lat_lons=ll, num_blocks=2),
            GraphCast(ll, num_processor_blocks=2), RegionalForecasterConfig(num_blocks=2).build()]  # fmt: skip


def test_default_is_no_segments_on_every_wrapper():
    for model in _wrappers():
        assert model.processor.checkpoint_segments == 0, type(model).__name__
        assert model._processor_segments() == 0, type(model).__name__


@pytest.mark.parametrize("bad", [-2, -10])
def test_values_below_minus_one_are_refused_where_they_are_set(bad):
    from graph_weather_b200 import GraphCast

    for model in _wrappers():
        with pytest.raises(ValueError, match="checkpoint segments"):
            model.processor.set_checkpoint_segments(bad)
        assert model.processor.checkpoint_segments == 0
    gcast = GraphCast(_grid(30), num_processor_blocks=2)
    with pytest.raises(ValueError, match="checkpoint segments"):
        gcast.set_checkpoint_processor(bad)
    assert gcast._checkpoint_processor_segments == 0


def test_each_wrapper_reads_its_setting():
    from graph_weather_b200 import GraphCastConfig

    for model in _wrappers():
        for s in (-1, 1, 5):
            model.processor.set_checkpoint_segments(s)
            assert model._processor_segments() == s, type(model).__name__
    gcast = _wrappers()[2]
    GraphCastConfig.balanced_checkpointing(gcast)
    assert gcast._processor_segments() == -1 and gcast._bounded_step()
    GraphCastConfig.processor_only_checkpointing(gcast)
    assert gcast._processor_segments() == -1 and not gcast._bounded_step()
    gcast.processor.set_checkpoint_segments(3)
    assert gcast._processor_segments() == -1  # GraphCast's own setting first
    GraphCastConfig.no_checkpointing(gcast)
    assert gcast._processor_segments() == 3  # then the processor's
    gcast.set_checkpoint_processor(2)
    gcast.set_checkpoint_model(True)  # (the reference's full checkpointing clears the processor setting)
    assert gcast._processor_segments() == 3 and gcast._bounded_step()


class _FakeLib:
    def __init__(self):
        self.calls = []

    def gw_train_set_processor_segments(self, handle, segments):
        self.calls.append((handle.value, segments))
        return 0


def test_binding_passes_segments_through():
    from graph_weather_b200 import _capi

    plan = _capi.Plan.__new__(_capi.Plan)  # (no device: the library call is replaced)
    plan.lib, plan.handle = _FakeLib(), ctypes.c_void_p(0x1234)
    for s in (0, -1, 1, 7):
        plan.set_processor_segments(s)
    assert plan.lib.calls == [(0x1234, 0), (0x1234, -1), (0x1234, 1), (0x1234, 7)]
    plan.handle = ctypes.c_void_p()  # (keep __del__ away from the fake)


def test_library_entry_point_checks_its_arguments():
    from graph_weather_b200 import _capi

    ge.build()
    lib = _capi.load()
    assert lib.gw_train_set_processor_segments(None, 1) != 0
    assert b"null plan" in lib.gw_last_error()
