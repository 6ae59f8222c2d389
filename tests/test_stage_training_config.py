"""Training the standalone Encoder, AssimilatorEncoder, Processor, Decoder and AssimilatorDecoder, without a GPU: `train_precision`
defaults to None (inference only) on all five, is validated like the wrappers' value, leaves the state_dict keys alone, and only a
value makes a train-mode call with autograd on take the training step."""
import pytest
import torch

LL = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]


def _modules():
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, Decoder, Encoder, Processor

    return {
        "Encoder": lambda **k: Encoder(LL, input_dim=10, **k),
        "AssimilatorEncoder": lambda **k: AssimilatorEncoder(**k),
        "Processor": lambda **k: Processor(num_blocks=2, **k),
        "Decoder": lambda **k: Decoder(LL, output_dim=10, **k),
        "AssimilatorDecoder": lambda **k: AssimilatorDecoder(LL, output_dim=10, **k),
    }


NAMES = ["Encoder", "AssimilatorEncoder", "Processor", "Decoder", "AssimilatorDecoder"]


@pytest.mark.parametrize("name", NAMES)
def test_train_precision_defaults_to_none(name):
    assert _modules()[name]().train_precision is None


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("tp", ["fp32_simt", "fp32", "bf16"])
def test_train_precision_is_accepted(name, tp):
    assert _modules()[name](train_precision=tp).train_precision == tp


@pytest.mark.parametrize("name", NAMES)
def test_unknown_train_precision_is_refused(name):
    with pytest.raises(ValueError, match="expected one of"):
        _modules()[name](train_precision="fp16")


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_precisions_need_the_default_trunk(tp):
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, Decoder, Encoder, Processor

    with pytest.raises(ValueError, match="train_precision"):
        Encoder(LL, input_dim=10, output_dim=128, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        AssimilatorEncoder(hidden_layers_processor_edge=3, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        Processor(num_blocks=2, hidden_dim_processor_node=128, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        Decoder(LL, output_dim=10, output_edge_dim=128, train_precision=tp)
    with pytest.raises(ValueError, match="train_precision"):
        AssimilatorDecoder(LL, output_dim=10, hidden_layers_processor_node=1, train_precision=tp)
    # fp32_simt trains any size
    Processor(num_blocks=2, hidden_dim_processor_node=128, train_precision="fp32_simt")


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_keys_are_unchanged(name):
    a = _modules()[name]()
    b = _modules()[name](train_precision="bf16")
    assert list(a.state_dict()) == list(b.state_dict())
    assert [k for k, _ in a.named_parameters()] == [k for k, _ in b.named_parameters()]


@pytest.mark.training
@pytest.mark.parametrize("name", NAMES)
def test_only_a_train_precision_selects_the_training_step(name):
    from graph_weather_b200.models import _stage_wants_grad

    x = torch.zeros(2, 3, requires_grad=True)
    default = _modules()[name]().train()
    assert torch.is_grad_enabled()
    assert not _stage_wants_grad(default, x)  # inference: the output has no grad_fn (tests/test_gpu_stage_training.py)
    trained = _modules()[name](train_precision="fp32_simt").train()
    assert _stage_wants_grad(trained, x)
    assert _stage_wants_grad(trained, None)  # the parameters require grad
    assert not _stage_wants_grad(trained.eval(), x)
    with torch.no_grad():
        assert not _stage_wants_grad(trained.train(), x)
