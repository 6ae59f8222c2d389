"""RegionalForecasterConfig.train_precision (no GPU needed): the field's contract, and the training oracle of this model
(regional_training_oracle.regional_oracle_step) against one training step of the reference's own RegionalForecaster
(tests/golden/regional_small_grads.npz, tests/golden/make_regional_grads.py)."""
import json
import os

import numpy as np
import pytest
import torch

from regional_training_oracle import regional_oracle_step
from training_oracle import rel_max

HERE = os.path.dirname(os.path.abspath(__file__))


def _small(**kw):
    from graph_weather_b200.regional import RegionalForecasterConfig

    return RegionalForecasterConfig(feature_dim=12, aux_dim=4, node_dim=32, edge_dim=32, num_blocks=2, hidden_dim_processor_node=32,
                                    hidden_dim_processor_edge=32, hidden_dim_decoder=32, **kw)  # fmt: skip


def _trunk(**kw):
    from graph_weather_b200.regional import RegionalForecasterConfig

    return RegionalForecasterConfig(num_blocks=2, **kw)


def test_default_refuses_to_train_and_names_the_field(monkeypatch):
    """The refusal comes before anything touches a device; here the CPU-tensor check is lifted so that a CPU test reaches it."""
    from graph_weather_b200 import regional

    monkeypatch.setattr(regional, "_no_host_path", lambda what: None)
    m = _small().build().train()
    assert m.train_precision is None
    with torch.enable_grad(), pytest.raises(NotImplementedError, match="train_precision"):
        m(torch.zeros(1, 5, 16), [(51.5, -0.1), (52.0, 0.5), (53.0, -1.0), (54.0, -2.0), (50.0, -3.0)])


def test_unknown_value_is_refused():
    with pytest.raises(ValueError, match="expected one of"):
        _small(train_precision="fp16").build()


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_values_need_the_256_wide_trunk(tp):
    with pytest.raises(ValueError, match="train_precision"):
        _small(train_precision=tp).build()
    _small(train_precision="fp32_simt").build()
    _trunk(train_precision=tp).build()


@pytest.mark.parametrize("tp", ["fp32", "bf16"])
def test_tensor_core_values_refuse_a_layernorm_wider_than_one_chain(tp):
    with pytest.raises(ValueError, match="LayerNorm"):
        _trunk(output_dim=300, feature_dim=300, train_precision=tp).build()
    _trunk(output_dim=300, feature_dim=300, train_precision="fp32_simt").build()
    _trunk(output_dim=256, feature_dim=256, train_precision=tp).build()


@pytest.mark.parametrize("tp", [None, "fp32_simt", "bf16"])
def test_state_dict_is_unchanged(tp):
    from graph_weather_b200.regional import RegionalForecasterConfig

    ref = {k: tuple(v.shape) for k, v in RegionalForecasterConfig(enable_nudging=True).build().state_dict().items()}
    got = RegionalForecasterConfig(enable_nudging=True, train_precision=tp).build().state_dict()
    assert list(got) == list(ref) and all(tuple(v.shape) == ref[k] for k, v in got.items())


@pytest.fixture(scope="module")
def fixture():
    z = np.load(os.path.join(HERE, "golden", "regional_small_grads.npz"))
    cfg = json.loads(str(z["config"]))
    idx = torch.from_numpy(z["h3_indices"])
    sd = {}
    for k, shape in zip(cfg["keys"], cfg["shapes"]):
        w = torch.from_numpy(z["w." + k])
        if k == "h3_embeddings":  # only the region's rows take part in the step
            w = torch.zeros(shape).index_copy_(0, idx, w)
        sd[k] = w
    ll = [tuple(p) for p in cfg["lat_lons"]]
    x, gc, target = (torch.from_numpy(z[k]) for k in ("x", "global_context", "target"))
    kw = dict(output_dim=12, num_blocks=2, global_context=gc)
    refs = {dt: regional_oracle_step(sd, ll, x, target, dt, **kw) for dt in (torch.float32, torch.float64)}
    return z, idx, refs


def test_oracle_matches_the_reference_training_step(fixture):
    """Output and loss within 1e-5; every gradient within 10x the fixture's own fp32 error against the fp64 oracle (+ 1e-5),
    h3_embeddings' zero off the region."""
    z, idx, refs = fixture
    out32, loss32, gx32, g32 = refs[torch.float32]
    _, _, gx64, g64 = refs[torch.float64]
    assert float((out32 - torch.from_numpy(z["out"])).abs().max()) < 1e-5
    assert abs(loss32 - float(z["loss"])) < 1e-5
    fails = []
    pairs = [("features", gx32, gx64, torch.from_numpy(z["grad_x"]))]
    for k in g32:
        fix = torch.from_numpy(z["g." + k])
        if k == "h3_embeddings":
            off = torch.ones(g64[k].shape[0], dtype=torch.bool)
            off[idx] = False
            assert not g64[k][off].any() and not g32[k][off].any()
            pairs.append((k, g32[k][idx], g64[k][idx], fix))
        else:
            pairs.append((k, g32[k], g64[k], fix))
    for k, ours, exact, fix in pairs:
        e_fix, e_ours = rel_max(fix, exact), rel_max(ours, fix)
        if not e_ours < 10 * e_fix + 1e-5:
            fails.append((k, e_ours, e_fix))
    assert len(pairs) == len(json.loads(str(z["config"]))["keys"]) + 1
    assert not fails, fails
