"""What the training tests share: the CPU autograd oracle of a training step (the reference's own ops, oracle/restate.py), the seeded
cases it runs on, one GPU training step, and the two bars a GPU step is held to against the oracle -- one for the fp32-type steps
(fp32_simt, fp32) and one for bf16.  Every number in which the tests' bars differ is an argument of the bar, so each test states
the bar it holds and the measurement behind it stays next to that call."""
import numpy as np
import torch


def grid(step):
    return [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]


# The ill-conditioned gradients of this model are those of the tensors shared by every sample and summed over the whole graph: the
# node encoder (its weights and the learned h3_nodes table, reached through the mesh-node rows), the encoder block's mesh-node MLP
# and the latent edge encoder (whose output is broadcast to every sample and every processor block).  The reference's own fp32
# arithmetic reaches only ~1e-2 (h3_nodes) and ~1e-3 (node_encoder.model.0.weight) max-relative error against fp64 on the
# 10-degree case, so two implementations differ there beyond the general bar.  Measured on an H100 (norm-relative vs fp32_simt):
# fp32 mode 2.9e-3 / 2.7e-3 / 1.5e-3 (node_encoder.0.weight / h3_nodes / encoder node MLP, features x1e5), 2.2e-3 (h3_nodes, x3e-4),
# 1.8e-3 (h3_nodes, 1 degree); bf16 mode at 1 degree 0.129 / 0.045 / 0.032 (h3_nodes / node_encoder.0.weight / latent edge
# encoder).  Those parameters get 5x the bar; every other parameter keeps it (all measured below 3e-4 in fp32 mode).
ILL_CONDITIONED = ("encoder.h3_nodes", "encoder.node_encoder.", "encoder.latent_edge_encoder.",
                   "encoder.graph_processor.blocks.0.node_model.")  # fmt: skip


def rel_max(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max()) / (float(b.double().abs().max()) + 1e-30)


def rel_norm(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm()) / (float(b.double().norm()) + 1e-30)


def cos(a, b):
    return float(torch.nn.functional.cosine_similarity(a.double().cpu().flatten(), b.double().cpu().flatten(), dim=0))


def forecaster_oracle_step(sd, ll, x, target, var, dtype, feature_dim=78, num_blocks=9, constraint=None, hl_node=2, hl_edge=2,
                           hl_dec=2):
    """One training step of the reference arithmetic on the CPU under torch.autograd, in fp32 (what the reference runs) or fp64
    (ground truth for the tolerances): encoder -> processor -> decoder + the first feature_dim features, then the restated
    PhysicalConstraintLayer (forecast.py:235-246) when `constraint` names one, then NormalizedMSELoss.  hl_node / hl_edge /
    hl_dec are the hidden-layer counts of the node MLPs, the edge MLPs and the node decoder.
    Returns (out, loss, d features, {name: grad})."""
    from oracle import restate

    sd_g = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    xg = x.to(dtype).clone().requires_grad_(True)
    g = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in restate.build_forecaster_graphs(ll).items()}
    hl = dict(hl_node=hl_node, hl_edge=hl_edge)
    ex, ei, ea = restate.encoder_forward(sd_g, g, xg, **hl)
    px = restate.processor_forward(sd_g, ex, ei, ea, num_blocks, **hl)
    out = restate.assimilator_decoder_forward(sd_g, g, px, x.shape[0], hl_dec=hl_dec, **hl) + xg[..., :feature_dim]
    if constraint is not None:
        from test_constraint_grads import grid_mapping, restate_constraint, rows_to_grid

        grid_shape, cell, last = grid_mapping(ll)
        lr = rows_to_grid(xg[..., :feature_dim], grid_shape)
        out = restate_constraint(constraint, rows_to_grid(out, grid_shape), lr, grid_shape, cell, last)
    loss = restate.normalized_mse_loss(out, target.to(dtype), var, ll, True)
    loss.backward()
    return out.detach(), float(loss.detach()), xg.grad, {k: v.grad for k, v in sd_g.items()}


def assimilator_oracle_step(sd, g_static, x, obs, target, dtype):
    """torch.autograd through analysis.py's forward (assimilator_encoder.py:118-168 + processor + assimilator decoder) and
    MSELoss: (out, loss, d features, {name: grad})."""
    from oracle import restate

    sd_g = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    g = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in g_static.items()}
    xg = x.to(dtype).clone().requires_grad_(True)
    B, nobs = x.shape[0], obs.shape[0]
    in_ei, in_ea = restate.assimilator_input_graph(obs, g["base_h3_grid"])
    h3_nodes = torch.zeros((g["num_h3"], x.shape[-1]), dtype=dtype)
    feats = torch.cat([xg, h3_nodes.unsqueeze(0).expand(B, -1, -1)], dim=1).reshape(-1, x.shape[-1])
    h = restate.mlp(sd_g, "encoder.node_encoder", feats)
    ea = restate.mlp(sd_g, "encoder.edge_encoder", in_ea.to(dtype)).repeat(B, 1)
    h, _ = restate.graph_processor(sd_g, "encoder.graph_processor", h, restate._replicate(in_ei, B), ea, 1)
    h = h.reshape(B, -1, h.shape[-1])[:, nobs:, :].reshape(-1, h.shape[-1])
    lat_ea = restate.mlp(sd_g, "encoder.latent_edge_encoder", g["lat_edge_attr"].repeat(B, 1))
    h = restate.processor_forward(sd_g, h, restate._replicate(g["lat_edge_index"], B), lat_ea, 9)
    out = restate.assimilator_decoder_forward(sd_g, g, h, B)
    loss = torch.nn.functional.mse_loss(out, target.to(dtype))
    loss.backward()
    return out.detach(), float(loss.detach()), xg.grad, {k: v.grad for k, v in sd_g.items()}


_CASES = {}


def forecaster_case(step, batch, seed, constraint=None, shift=0.0, **shape_kw):
    """A seeded forecaster case on the `step`-degree grid: (lat_lons, state_dict, features, target, variances, oracle step in fp32,
    oracle step in fp64).  `shape_kw` are weights.forecaster_shapes' arguments (and the oracle's feature_dim / num_blocks /
    hidden-layer counts); the first feature_dim input channels are shifted by `shift`.  Cached per key: the oracle steps are the slow part."""
    key = (step, batch, seed, constraint, shift, tuple(sorted(shape_kw.items())))
    if key not in _CASES:
        from oracle import weights

        ll = grid(step)
        F, A, nb = shape_kw.get("feature_dim", 78), shape_kw.get("aux_dim", 24), shape_kw.get("num_blocks", 9)
        sd = weights.make_state_dict(weights.forecaster_shapes(**shape_kw), seed)
        x = weights.make_features(batch, len(ll), F + A, seed)
        if shift:
            x[..., :F] += shift
        rng = np.random.Generator(np.random.PCG64(seed))
        target = torch.from_numpy(rng.standard_normal((batch, len(ll), F)).astype(np.float32))
        var = rng.uniform(0.5, 2.0, F).astype(np.float32).tolist()
        hl = dict(hl_node=shape_kw.get("hidden_layers_processor_node", 2), hl_edge=shape_kw.get("hidden_layers_processor_edge", 2),
                  hl_dec=shape_kw.get("hidden_layers_decoder", 2))
        refs = [forecaster_oracle_step(sd, ll, x, target, var, dt, F, nb, constraint, **hl) for dt in (torch.float32, torch.float64)]
        _CASES[key] = (ll, sd, x, target, var, *refs)
    return _CASES[key]


def train_step(model, loss_fn, x, target, obs=None, feat_grad=True):
    """One training forward + loss + backward on the GPU, from cleared gradients: (out, loss, d features, {name: grad}) on the
    host.  The plan's status word is read (it raises on a flagged fault)."""
    model.zero_grad(set_to_none=True)
    xc = x.cuda().requires_grad_(feat_grad)
    out = model(xc) if obs is None else model(xc, obs.cuda())
    assert out.requires_grad
    loss = loss_fn(out, target.cuda())
    loss.backward()
    model._train_engine.plan.status()
    grads = {k: q.grad.detach().cpu().clone() for k, q in model.named_parameters()}
    return out.detach().cpu(), float(loss), (xc.grad.cpu() if feat_grad else None), grads


def _common(ours, ref32, ref64, n_params, out_bar, loss_bar, tag):
    out, loss, gx, grads = ours
    out32, loss32 = ref32[:2]
    gx64, g64 = ref64[2:]
    fails = []
    if not float((out - out32).abs().max()) < out_bar:
        fails.append((tag, "out", float((out - out32).abs().max())))
    if not abs(loss - loss32) <= loss_bar * abs(loss32):
        fails.append((tag, "loss", loss, loss32))
    assert gx is not None and gx.shape == gx64.shape, "features.grad was not produced"
    if grads is not None:
        assert set(grads) == set(g64), set(grads) ^ set(g64)
        assert n_params is None or len(grads) == n_params, len(grads)
        assert all(g.shape == g64[k].shape for k, g in grads.items())
    return fails


def _numerically_zero(g64):
    big = max(float(g.abs().max()) for g in g64.values())
    return {k for k, g in g64.items() if float(g.abs().max()) <= 1e-6 * big}


def check_fp32_bars(ours, ref32, ref64, *, n_params, floor, feat_floor, median, ill, skip_zero, norm_bar, tag=""):
    """An fp32-type step (`ours` = train_step's result; `grads` None leaves the parameters to the caller) against the oracle:
    the output within 1e-4 and the loss within 1e-5 (relative) of the fp32 oracle's; each gradient's max-relative error against
    fp64 below 10x the fp32 oracle's own + 2e-5, or below `floor`.
      feat_floor  the features' gradient gets the floor too (else 10x + 2e-5 alone)
      median      the median of the parameters' errors within 3x the fp32 oracle's median + 1e-5
      ill         None, "max" (ILL_CONDITIONED parameters get 5x the bar) or "norm" (they are held to 5x the bar on the
                  norm-relative error instead, without the floor)
      skip_zero   numerically zero gradients (max |g| <= 1e-6 of the largest, in fp64) are left out
      norm_bar    None, or every parameter is held to norm-relative error < norm_bar against fp64 instead
    Failures are collected, printed and asserted together."""
    fails = _common(ours, ref32, ref64, n_params, 1e-4, 1e-5, tag)
    _, _, gx, grads = ours
    gx32, g32 = ref32[2:]
    gx64, g64 = ref64[2:]
    e_ours, e_ref = rel_max(gx, gx64), rel_max(gx32, gx64)
    feat_bar = max(10 * e_ref + 2e-5, floor) if feat_floor else 10 * e_ref + 2e-5
    print(f"{tag}: d loss / d features: rel err vs fp64 {e_ours:.2e} (fp32 oracle {e_ref:.2e}; bar {feat_bar:.2e})")
    if not e_ours < feat_bar:
        fails.append((tag, "features", e_ours, e_ref))
    if grads is not None:
        skip = _numerically_zero(g64) if skip_zero else set()
        errs = sorted(((rel_max(grads[k], g64[k]), rel_max(g32[k], g64[k]), k) for k in grads if k not in skip), reverse=True)
        for eo, er, k in errs[:8]:
            print(f"  {tag} {k}: max-rel err vs fp64 {eo:.2e} (fp32 oracle {er:.2e}; bar {max(10 * er + 2e-5, floor):.2e})")
        for eo, er, k in errs:
            is_ill = ill is not None and k.startswith(ILL_CONDITIONED)
            if norm_bar is not None:
                en = rel_norm(grads[k], g64[k])
                if not en < norm_bar:
                    fails.append((tag, k, "norm", en))
            elif is_ill and ill == "norm":
                no, nr = rel_norm(grads[k], g64[k]), rel_norm(g32[k], g64[k])
                print(f"  {tag} {k}: norm-rel err vs fp64 {no:.2e} (fp32 oracle {nr:.2e}; bar {5 * (10 * nr + 2e-5):.2e})")
                if not no < 5 * (10 * nr + 2e-5):
                    fails.append((tag, k, "norm", no, nr))
            elif not eo < max(10 * er + 2e-5, floor) * (5 if is_ill else 1):
                fails.append((tag, k, eo, er))
        if median:
            med_o, med_r = sorted(e[0] for e in errs)[len(errs) // 2], sorted(e[1] for e in errs)[len(errs) // 2]
            print(f"{tag}: median rel err vs fp64: ours {med_o:.2e}, fp32 oracle {med_r:.2e}")
            if not med_o < 3 * med_r + 1e-5:
                fails.append((tag, "median", med_o, med_r))
    assert not fails, fails


def check_bf16_bars(ours, ref32, ref64, *, n_params, cos_bar, ill_cos_bar, feat_cos, total_cos, tag=""):
    """A bf16 step (`ours` = train_step's result; `grads` None leaves the parameters to the caller) against the oracle: the
    output within 2e-2 and the loss within 1e-2 (relative) of the fp32 oracle's; each parameter's gradient at cosine >= cos_bar
    to fp64 (ILL_CONDITIONED ones >= ill_cos_bar), numerically zero gradients left out (their direction is noise).
      feat_cos   None, or the features' gradient at cosine >= feat_cos to fp64
      total_cos  None, or all parameter gradients concatenated at cosine >= total_cos to fp64
    Failures are collected, printed and asserted together."""
    fails = _common(ours, ref32, ref64, n_params, 2e-2, 1e-2, tag)
    _, _, gx, grads = ours
    gx64, g64 = ref64[2:]
    if feat_cos is not None:
        c = cos(gx, gx64)
        print(f"{tag}: d loss / d features: cosine vs fp64 {c:.5f} (bar {feat_cos})")
        if not c >= feat_cos:
            fails.append((tag, "features", c))
    if grads is not None:
        skip = _numerically_zero(g64)
        worst = sorted((cos(g, g64[k]), k) for k, g in grads.items() if k not in skip)
        for c, k in worst[:8]:
            print(f"  {tag} {k}: cosine vs fp64 {c:.5f}")
        fails += [(tag, k, c) for c, k in worst if not c >= (ill_cos_bar if k.startswith(ILL_CONDITIONED) else cos_bar)]
        if total_cos is not None:
            c = cos(torch.cat([grads[k].double().flatten() for k in sorted(grads)]), torch.cat([g64[k].double().flatten() for k in sorted(grads)]))
            if not c >= total_cos:
                fails.append((tag, "all parameters", c))
    assert not fails, fails
