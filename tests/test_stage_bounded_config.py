"""The standalone stages' choice of training step without a GPU: `use_checkpointing` selects a training-only engine for the Encoder,
the decoders and the AssimilatorEncoder, read again at every choice, with one engine per step kind; the Processor's engine stays
taped; inference keeps its own engine."""
import pytest

LL = [(float(a), float(b)) for a in range(-90, 90, 30) for b in range(0, 360, 30)]


def _modules(flag):
    from graph_weather_b200 import AssimilatorDecoder, AssimilatorEncoder, Decoder, Encoder

    return [Encoder(LL, input_dim=6, train_precision="bf16", use_checkpointing=flag),
            AssimilatorEncoder(train_precision="bf16", use_checkpointing=flag),
            Decoder(LL, output_dim=4, train_precision="bf16", use_checkpointing=flag),
            AssimilatorDecoder(LL, output_dim=4, train_precision="bf16", use_checkpointing=flag)]  # fmt: skip


@pytest.mark.parametrize("flag", [False, True])
def test_use_checkpointing_selects_the_engine(flag):
    from graph_weather_b200 import models

    for m in _modules(flag):
        name = type(m).__name__
        assert m.use_checkpointing is flag, name
        eng = models._stage_engine(m, m._dims, [], m.use_checkpointing)
        assert eng.train_only is flag and m._train_engine is eng, name
        assert eng.precision == "bf16" and m._engine is None, name  # (no inference engine is made for training)
        m.use_checkpointing = not flag  # read at every choice: the other step's engine, made on first use
        other = models._stage_engine(m, m._dims, [], m.use_checkpointing)
        assert other.train_only is (not flag) and m._train_engine is other, name
        m.use_checkpointing = flag  # and back to the same engine
        assert models._stage_engine(m, m._dims, [], m.use_checkpointing) is eng, name
        assert set(m._train_engines) == {False, True}, name


def test_processor_stays_taped():
    from graph_weather_b200 import Processor, models

    proc = Processor(num_blocks=2, train_precision="bf16", use_checkpointing=True)
    eng = models._stage_engine(proc, proc._plan_dims(10, 20), [])
    assert eng.train_only is False and proc._train_engine is eng
