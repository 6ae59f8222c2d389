"""What the RegionalForecaster training tests share: the CPU autograd oracle of one training step of this model (the reference's
own ops, oracle/restate.py), the renaming that holds its gradients to training_oracle's bars, and the bf16 bars with this model's
output bar."""
import numpy as np
import torch

from training_oracle import ILL_CONDITIONED, _numerically_zero, cos


def _regional_forward(sd, g, x, output_dim, num_blocks, hl_node, hl_edge, hl_dec, global_context, lat_lons):
    """restate.regional_forward (regional_forecast.py:233-298) under autograd, in the dtype of x and sd."""
    from oracle import restate

    dt, n = x.dtype, g["num_obs"]
    regional_h3 = sd["h3_embeddings"][torch.tensor(g["h3_indices"], dtype=torch.long)]
    enc_ea = restate.mlp(sd, "edge_encoder", g["enc_edge_attr"].to(dt), hl_edge)
    lat_ea = restate.mlp(sd, "latent_edge_encoder", g["lat_edge_attr"].to(dt), hl_edge)
    dec_ei = g["enc_edge_index"].flip(0)
    dec_ea = restate.mlp(sd, "decoder_edge_encoder", g["enc_edge_attr"].to(dt), hl_edge)
    outs = []
    for i in range(x.shape[0]):
        nodes = restate.mlp(sd, "node_encoder", torch.cat([x[i], regional_h3], dim=0), hl_node)
        nodes, _ = restate.graph_processor(sd, "encoder_gnn", nodes, g["enc_edge_index"], enc_ea, 1, hl_node, hl_edge)
        h = restate.processor_forward(sd, nodes[n:], g["lat_edge_index"], lat_ea, num_blocks, "processor", hl_node, hl_edge)
        dec_nodes = torch.cat([torch.zeros(n, h.shape[-1], dtype=dt), h], dim=0)
        dec_nodes, _ = restate.graph_processor(sd, "decoder_gnn", dec_nodes, dec_ei, dec_ea, 1, hl_node, hl_edge)
        outs.append(restate.mlp(sd, "node_decoder", dec_nodes[:n], hl_dec, norm=True))
    out = torch.stack(outs, dim=0) + x[..., :output_dim]
    if global_context is None:
        return out
    # BoundaryNudgingLayer (:68-130): the relaxation prior in float32, as the reference computes it
    ll = torch.tensor(lat_lons, dtype=torch.float32) * (np.pi / 180.0)
    lat, lon = ll[:, 0], ll[:, 1]
    a = torch.sin((lat - lat.mean()) / 2) ** 2 + torch.cos(lat) * torch.cos(lat.mean()) * torch.sin((lon - lon.mean()) / 2) ** 2
    dist = 2 * torch.asin(torch.sqrt(torch.clamp(a, 0.0, 1.0)))
    prior = dist / dist.max() if dist.max() > 0 else torch.zeros_like(dist)
    prior = prior.to(dt).unsqueeze(-1).unsqueeze(0).expand(out.shape[0], -1, -1)
    corr = restate.mlp(sd, "nudging.blend_mlp", torch.cat([out, global_context, prior], dim=-1), 1, norm=False)
    alpha = torch.clamp(prior + corr, 0.0, 1.0)
    return (1 - alpha) * out + alpha * global_context


def regional_oracle_step(sd, lat_lons, x, target, dtype, output_dim=78, num_blocks=9, hl_node=2, hl_edge=2, hl_dec=2, global_context=None,
                         rollout=1):
    """One training step of RegionalForecaster's reference arithmetic on the CPU under torch.autograd, in fp32 or fp64, with optional
    boundary nudging (global_context) and a plain MSE loss.  rollout K > 1: K forwards on the region, each fed the previous output
    and the auxiliary columns of x, and the sum of the K losses against target[0 .. K-1].  The gradient of h3_embeddings is
    table-shaped.  Returns (out of the last forward, loss, d features, {name: grad})."""
    from oracle import restate

    sd_g = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    xg = x.to(dtype).clone().requires_grad_(True)
    g = restate.regional_graphs(lat_lons)
    gc = None if global_context is None else global_context.to(dtype)
    inp, loss = xg, 0.0
    for t in range(rollout):
        out = _regional_forward(sd_g, g, inp, output_dim, num_blocks, hl_node, hl_edge, hl_dec, gc, lat_lons)
        loss = loss + torch.nn.functional.mse_loss(out, (target[t] if rollout > 1 else target).to(dtype))
        inp = torch.cat([out, xg[..., output_dim:]], dim=-1)
    loss.backward()
    return out.detach(), float(loss.detach()), xg.grad, {k: v.grad for k, v in sd_g.items()}


def plan_names(step):
    """A step's result (out, loss, d features, {name: grad}) with the gradients under the names the plan binds them by
    (RegionalForecaster._RENAME; h3_embeddings -> encoder.h3_nodes; the nudging layer's keep their own).  The parameters then
    play the forecaster's roles under the forecaster's names, so training_oracle.ILL_CONDITIONED marks the same ill-conditioned
    ones: the embedding table, the node encoder, the latent edge encoder and the encoder block's node model."""
    from graph_weather_b200.regional import RegionalForecaster

    def name(k):
        if k == "h3_embeddings":
            return "encoder.h3_nodes"
        for a, b in RegionalForecaster._RENAME:
            if k.startswith(a):
                return b + k[len(a):]
        return k

    out, loss, gx, grads = step
    return out, loss, gx, {name(k): v for k, v in grads.items()}


def check_bf16_bars_ln_out(ours, ref32, ref64, *, out_bar, cos_bar, ill_cos_bar, feat_cos, tag=""):
    """training_oracle.check_bf16_bars (loss within 1e-2 relative of the fp32 oracle's, each parameter's gradient at cosine >=
    cos_bar to fp64, ILL_CONDITIONED ones >= ill_cos_bar, numerically zero ones left out, the features' at >= feat_cos), with the
    output held to `out_bar` instead of 2e-2: this model's output leaves a LayerNorm, which scales the bf16 error of the value it
    normalises by 1 / std.  Gradients under plan_names()."""
    out, loss, gx, grads = ours
    out32, loss32 = ref32[:2]
    gx64, g64 = ref64[2:]
    fails = []
    e = float((out - out32).abs().max())
    print(f"{tag}: output max-abs difference to the fp32 oracle {e:.2e} (bar {out_bar})")
    if not e < out_bar:
        fails.append((tag, "out", e))
    if not abs(loss - loss32) <= 1e-2 * abs(loss32):
        fails.append((tag, "loss", loss, loss32))
    assert set(grads) == set(g64), set(grads) ^ set(g64)
    c = cos(gx, gx64)
    print(f"{tag}: d loss / d features: cosine vs fp64 {c:.5f} (bar {feat_cos})")
    if not c >= feat_cos:
        fails.append((tag, "features", c))
    skip = _numerically_zero(g64)
    worst = sorted((cos(g, g64[k]), k) for k, g in grads.items() if k not in skip)
    for c, k in worst[:8]:
        print(f"  {tag} {k}: cosine vs fp64 {c:.5f}")
    fails += [(tag, k, c) for c, k in worst if not c >= (ill_cos_bar if k.startswith(ILL_CONDITIONED) else cos_bar)]
    assert not fails, fails
