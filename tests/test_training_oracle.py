"""The bars of tests/training_oracle.py, without a GPU: on a small case (30-degree grid, 2 blocks) each bar passes the fp32
oracle's own step given as "ours", and fails it when one parameter's gradient is off by 1 % (the fp32 bars) or is noise (the bf16
bar).  The same holds on the mixed shape of tests/test_gpu_model_shapes.py (unequal node / edge and hidden widths, 1 / 3 / 3
hidden layers), whose oracle takes its hidden-layer counts from the case's shape arguments."""
import pytest
import torch

from training_oracle import check_bf16_bars, check_fp32_bars, forecaster_case

pytestmark = pytest.mark.training  # (autograd on: the oracle differentiates)

PARAM = "processor.graph_processor.blocks.1.edge_model.edge_mlp.model.2.weight"

# the fp32 bars of the training tests that a 1 % error in one gradient fails
FP32_BARS = {
    "taped_simt": dict(n_params=None, floor=0.0, feat_floor=False, median=True, ill=None, skip_zero=False, norm_bar=None),
    "wide": dict(n_params=None, floor=2e-3, feat_floor=False, median=True, ill="norm", skip_zero=False, norm_bar=None),
    "constraint": dict(n_params=None, floor=2e-3, feat_floor=True, median=False, ill="max", skip_zero=True, norm_bar=None),
    # (the constraint tests' norm bar is 1e-2, which a 1 % error meets to rounding: 5e-3 tests the same path)
    "additive_tc": dict(n_params=None, floor=2e-3, feat_floor=True, median=False, ill="max", skip_zero=True, norm_bar=5e-3),
}
BF16_BARS = {
    "taped": dict(n_params=None, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=None, total_cos=0.999),
    "features": dict(n_params=None, cos_bar=0.99, ill_cos_bar=0.98, feat_cos=0.99, total_cos=None),
    "additive_tc": dict(n_params=None, cos_bar=0.9, ill_cos_bar=0.9, feat_cos=0.99, total_cos=None),
}


@pytest.fixture(scope="module")
def case():
    return forecaster_case(30, 1, 7, num_blocks=2)


# tests/test_gpu_model_shapes.py's mixed shape, and a parameter of its deepest edge MLP (model.4: the third hidden layer)
MIXED = dict(node_dim=48, edge_dim=80, hidden_dim_processor_node=96, hidden_dim_processor_edge=64, hidden_layers_processor_node=1,
             hidden_layers_processor_edge=3, hidden_dim_decoder=40, hidden_layers_decoder=3, feature_dim=7, aux_dim=5, num_blocks=2)
MIXED_PARAM = "processor.graph_processor.blocks.1.edge_model.edge_mlp.model.4.weight"


@pytest.fixture(scope="module")
def mixed_case():
    return forecaster_case(30, 1, 7, **MIXED)


def _with(ref32, k, g):
    out, loss, gx, grads = ref32
    return out, loss, gx, {**grads, k: g}


@pytest.mark.parametrize("name", list(FP32_BARS))
def test_fp32_bars(case, name):
    ref32, ref64 = case[5:]
    assert PARAM in ref32[3]
    check_fp32_bars(ref32, ref32, ref64, **FP32_BARS[name])
    with pytest.raises(AssertionError, match=PARAM):
        check_fp32_bars(_with(ref32, PARAM, ref32[3][PARAM] * 1.01), ref32, ref64, **FP32_BARS[name])


@pytest.mark.parametrize("name", list(BF16_BARS))
def test_bf16_bars(case, name):
    ref32, ref64 = case[5:]
    check_bf16_bars(ref32, ref32, ref64, **BF16_BARS[name])
    noise = torch.randn(ref32[3][PARAM].shape, generator=torch.Generator().manual_seed(0))
    with pytest.raises(AssertionError, match=PARAM):
        check_bf16_bars(_with(ref32, PARAM, noise), ref32, ref64, **BF16_BARS[name])


def test_the_parameter_count_is_checked(case):
    ref32, ref64 = case[5:]
    with pytest.raises(AssertionError):
        check_fp32_bars(ref32, ref32, ref64, **dict(FP32_BARS["taped_simt"], n_params=len(ref32[3]) + 1))
    with pytest.raises(AssertionError):
        check_bf16_bars(ref32, ref32, ref64, **dict(BF16_BARS["taped"], n_params=len(ref32[3]) - 1))


def test_mixed_shape_oracle_follows_the_shape(mixed_case):
    """Every parameter of the shape gets a gradient of its own shape, and the 3-deep edge MLPs' last hidden layer is reached."""
    from oracle import weights

    ref32, ref64 = mixed_case[5:]
    shapes = weights.forecaster_shapes(**MIXED)
    assert list(ref64[3]) == list(shapes)
    assert all(tuple(ref64[3][k].shape) == s for k, s in shapes.items())
    assert float(ref64[3][MIXED_PARAM].abs().max()) > 0
    assert float(ref64[3]["decoder.node_decoder.model.6.weight"].abs().max()) > 0  # Linear 3 of the 3-hidden-layer decoder


# the fp32 bars tests/test_gpu_model_shapes.py holds its fp32_simt and fp32-mode steps to
MIXED_FP32_BARS = {"fp32_simt": FP32_BARS["taped_simt"], "fp32_simt_floor": dict(FP32_BARS["taped_simt"], floor=2e-4),
                   "fp32": dict(FP32_BARS["taped_simt"], floor=8e-3, feat_floor=True, median=False)}


@pytest.mark.parametrize("name", list(MIXED_FP32_BARS))
def test_fp32_bars_mixed_shape(mixed_case, name):
    ref32, ref64 = mixed_case[5:]
    check_fp32_bars(ref32, ref32, ref64, **MIXED_FP32_BARS[name])
    with pytest.raises(AssertionError, match=MIXED_PARAM):
        check_fp32_bars(_with(ref32, MIXED_PARAM, ref32[3][MIXED_PARAM] * 1.01), ref32, ref64, **MIXED_FP32_BARS[name])


@pytest.mark.parametrize("bars", [BF16_BARS["taped"], dict(BF16_BARS["taped"], cos_bar=0.98, ill_cos_bar=0.975, total_cos=0.995)])
def test_bf16_bars_mixed_shape(mixed_case, bars):
    ref32, ref64 = mixed_case[5:]
    check_bf16_bars(ref32, ref32, ref64, **bars)
    noise = torch.randn(ref32[3][MIXED_PARAM].shape, generator=torch.Generator().manual_seed(0))
    with pytest.raises(AssertionError, match=MIXED_PARAM):
        check_bf16_bars(_with(ref32, MIXED_PARAM, noise), ref32, ref64, **bars)
