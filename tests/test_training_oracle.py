"""The bars of tests/training_oracle.py, without a GPU: on a small case (30-degree grid, 2 blocks) each bar passes the fp32
oracle's own step given as "ours", and fails it when one parameter's gradient is off by 1 % (the fp32 bars) or is noise (the bf16
bar)."""
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
