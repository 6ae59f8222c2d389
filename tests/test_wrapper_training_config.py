"""GraphCast and GraphWeatherAssimilator training without a GPU: `train_precision` is accepted and validated by both constructors
and by GraphWeatherAssimilatorConfig, the state_dict keys do not change, save_pretrained / from_pretrained carry
`train_precision`, and GraphCast's checkpoint controls select the taped or the bounded-memory step."""
import json

import pytest
import torch

from oracle import weights

LL = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]


@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_constructors_accept_train_precision(tp):
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator, GraphWeatherAssimilatorConfig

    assert GraphCast(LL, num_processor_blocks=2, train_precision=tp).train_precision == tp
    assert GraphWeatherAssimilator(output_lat_lons=LL, analysis_dim=5, num_blocks=1, train_precision=tp).train_precision == tp
    cfg = GraphWeatherAssimilatorConfig(output_lat_lons=LL, analysis_dim=5, num_blocks=1, train_precision=tp)
    assert cfg.build().train_precision == tp


def test_defaults_are_exact_fp32():
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator, GraphWeatherAssimilatorConfig

    assert GraphCast(LL, num_processor_blocks=1).train_precision == "fp32_simt"
    assert GraphWeatherAssimilator(output_lat_lons=LL, num_blocks=1).train_precision == "fp32_simt"
    assert GraphWeatherAssimilatorConfig(output_lat_lons=LL).train_precision == "fp32_simt"


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_precisions_need_the_default_trunk(tp):
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator, GraphWeatherAssimilatorConfig

    with pytest.raises(ValueError, match="train_precision"):
        GraphCast(LL, num_processor_blocks=1, hidden_layers=3, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        GraphCast(LL, num_processor_blocks=1, hidden_dim=128, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        GraphWeatherAssimilator(output_lat_lons=LL, num_blocks=1, node_dim=128, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        GraphWeatherAssimilatorConfig(output_lat_lons=LL, num_blocks=1, hidden_layers_processor_edge=3, train_precision=tp).build()
    # fp32_simt trains any size
    GraphCast(LL, num_processor_blocks=1, hidden_layers=3)


def test_unknown_train_precision_is_refused():
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator

    with pytest.raises(ValueError, match="expected one of"):
        GraphCast(LL, num_processor_blocks=1, train_precision="fp16")
    with pytest.raises(ValueError, match="expected one of"):
        GraphWeatherAssimilator(output_lat_lons=LL, num_blocks=1, train_precision="tf32")


def test_state_dict_keys_are_unchanged():
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator

    a = GraphWeatherAssimilator(output_lat_lons=LL, analysis_dim=24, train_precision="bf16")
    assert list(a.state_dict().keys()) == list(weights.forecaster_shapes(assimilator=True, output_dim=24).keys())
    g = GraphCast(LL, train_precision="bf16")
    shapes = weights.forecaster_shapes(feature_dim=78, aux_dim=0, hidden_dim_decoder=256)
    assert {k: tuple(v.shape) for k, v in g.state_dict().items()} == dict(shapes)


def test_assimilator_hub_round_trip(tmp_path):
    from graph_weather_b200 import GraphWeatherAssimilator

    torch.manual_seed(4)
    a = GraphWeatherAssimilator(output_lat_lons=LL, analysis_dim=5, num_blocks=1, train_precision="bf16", use_checkpointing=True)
    a.save_pretrained(tmp_path / "as")
    cfg = json.load(open(tmp_path / "as" / "config.json"))
    assert cfg["train_precision"] == "bf16"
    a2 = GraphWeatherAssimilator.from_pretrained(tmp_path / "as")
    assert a2.train_precision == "bf16" and a2.use_checkpointing is True
    assert all(torch.equal(v, a2.state_dict()[k]) for k, v in a.state_dict().items())


def test_graphcast_strategy_selects_the_step():
    """The bounded step for every strategy that checkpoints the encoder, the decoder or the whole model, or use_checkpointing;
    the taped step otherwise (the processor's segments alone keep the tape).  Only the selected engine is returned; the inference
    engine never becomes training-only."""
    from graph_weather_b200 import GraphCast, GraphCastConfig

    g = GraphCast(LL, num_processor_blocks=1)
    expect = {"no_checkpointing": False, "full_checkpointing": True, "balanced_checkpointing": True,
              "processor_only_checkpointing": False, "fine_grained_checkpointing": False}  # fmt: skip
    for name, bounded in expect.items():
        getattr(GraphCastConfig, name)(g)
        assert g._training_engine().train_only is bounded, name
        assert g._train_engine is g._training_engine()
    g.set_checkpoint_model(False), g.set_checkpoint_encoder(False), g.set_checkpoint_decoder(True)
    assert g._training_engine().train_only is True
    assert g._engine.train_only is False
    assert GraphCast(LL, num_processor_blocks=1, use_checkpointing=True)._training_engine().train_only is True


def test_use_checkpointing_assigned_later_selects_the_step():
    """Every wrapper reads use_checkpointing at each training forward, as GraphCast reads its checkpoint controls."""
    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator, GraphWeatherForecaster

    for m in (GraphWeatherForecaster(LL, num_blocks=1), GraphWeatherAssimilator(output_lat_lons=LL, analysis_dim=5, num_blocks=1),
              GraphCast(LL, num_processor_blocks=1)):  # fmt: skip
        for flag in (False, True, False):
            m.use_checkpointing = flag
            assert m._training_engine().train_only is flag, type(m).__name__
            assert m._train_engine is m._training_engine()


def test_graphcast_with_another_edge_width_in_the_decoder_is_refused():
    """GraphCast(hidden_dim=96): the reference's decoder keeps 256-wide edges while the encoder and processor use hidden_dim.  The
    CUDA plan has one edge width, so the model is refused at construction, in words, instead of failing at its first forward."""
    from graph_weather_b200 import GraphCast

    with pytest.raises(NotImplementedError, match="decoder edge width 256 differs from the encoder's 96"):
        GraphCast(LL, num_processor_blocks=1, hidden_dim=96)
    GraphCast(LL, num_processor_blocks=1, hidden_layers=3)  # the 256-wide trunk with three hidden layers is taken
