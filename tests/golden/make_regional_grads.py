"""Generates tests/golden/regional_small_grads.npz: one training step of the reference's OWN RegionalForecaster
(regional_forecast.py, located by oracle/ref_shims.py) under torch.autograd on the CPU.  Runs only where the reference sources are
present; the fixture travels with the repository.

    python tests/golden/make_regional_grads.py

The case is the reference suite's small config (12 + 4 features, 32 wide, 2 blocks; tests/test_regional_forecast.py) with boundary
nudging on, the UK region of its tests, a global context and a plain MSE loss.  It stores the seeded weights (h3_embeddings as
the region's rows, with their indices), the inputs, the output, the loss and the gradient of every parameter (h3_embeddings: the
region's rows; the generator checks that every other row is zero) and of the features.
"""

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_shims, weights  # noqa: E402

UK = [(51.5, -0.1), (52.0, 0.5), (53.0, -1.0), (54.0, -2.0), (50.0, -3.0)]
KW = dict(feature_dim=12, aux_dim=4, node_dim=32, edge_dim=32, num_blocks=2, hidden_dim_processor_node=32, hidden_dim_processor_edge=32,
          hidden_dim_decoder=32, enable_nudging=True)  # fmt: skip


def main(name="regional_small_grads"):
    R = ref_shims.load_reference()
    model = R.RegionalForecaster(R.RegionalForecasterConfig(**KW))
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = weights.make_state_dict(shapes, 31)
    model.load_state_dict(sd)
    x = weights.make_features(2, len(UK), 16, 31).requires_grad_(True)
    gc = weights.make_features(2, len(UK), 12, 32)
    target = weights.make_features(2, len(UK), 12, 33)
    out = model(x, UK, global_context=gc)
    loss = torch.nn.functional.mse_loss(out, target)
    loss.backward()
    _, _, _, h3_idx = model.graph_builder(UK)
    idx = np.array(h3_idx, dtype=np.int64)
    grads = {k: q.grad.numpy() for k, q in model.named_parameters()}
    assert not np.any(np.delete(grads["h3_embeddings"], idx, axis=0)), "h3_embeddings.grad outside the region"
    grads["h3_embeddings"] = grads["h3_embeddings"][idx]
    w = {k: v.numpy() for k, v in sd.items()}
    w["h3_embeddings"] = w["h3_embeddings"][idx]
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        config=json.dumps(dict(seed=31, lat_lons=UK, kw=KW, keys=list(shapes.keys()), shapes=[list(v) for v in shapes.values()])),
        h3_indices=idx, x=x.detach().numpy(), global_context=gc.numpy(), target=target.numpy(), out=out.detach().numpy(),
        loss=np.float64(float(loss.detach())), grad_x=x.grad.numpy(), **{"w." + k: v for k, v in w.items()}, **{"g." + k: v for k, v in grads.items()})  # fmt: skip
    print(name, "out", tuple(out.shape), "loss", float(loss.detach()), "cells", idx.size)


if __name__ == "__main__":
    main()
