"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch CPU tensors, fp32) of the reference's encode-process-decode
forward.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import it;
the product path (graph_weather_b200/) never does.

Parity status: PINNED.  tests/test_oracle.py checks this restatement against outputs of the reference's own,
unmodified source files executed in the build container through oracle/ref_shims.py (fixtures under tests/golden/,
generator tests/golden/make_golden.py).  The reference's test-suite holds no value-level golden vectors for this
path (SURVEY.md section 8(c)); its count KATs (5882 cells / 41162 latent edges / UK box 5-25-175-19) are checked in
tests/test_h3lite.py and tests/test_graphs.py.

Each function cites the reference lines it follows.  The arithmetic keeps the reference's op order exactly
(replicated-graph batching, concat -> Linear chain -> LayerNorm -> in-place residual, scatter_add by target).
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from graph_weather_b200 import h3lite as h3  # same API as the `h3` package the reference imports


# ----------------------------------------------------------------------------------------------------------------
# graph construction, loop for loop
# ----------------------------------------------------------------------------------------------------------------
def encoder_graph(lat_lons, resolution=2):
    """encoder.py:76-109. Returns (edge_index [2,N] long, edge_attr [N,2] float, base_h3_grid)."""
    num_latlons = len(lat_lons)
    base_h3_grid = sorted(list(h3.uncompact_cells(h3.get_res0_cells(), resolution)))
    h3_grid = [h3.latlng_to_cell(lat, lon, resolution) for lat, lon in lat_lons]
    h3_mapping = {}
    h_index = len(base_h3_grid)
    for h in base_h3_grid:
        if h not in h3_mapping:
            h_index -= 1
            h3_mapping[h] = h_index + num_latlons
    dists = []
    for idx, cell in enumerate(h3_grid):
        d = h3.great_circle_distance(lat_lons[idx], h3.cell_to_latlng(cell), unit="rads")
        dists.append([np.sin(d), np.cos(d)])
    edge_attr = torch.tensor(dists, dtype=torch.float)
    src = list(range(num_latlons))
    dst = [h3_mapping[c] for c in h3_grid]
    return torch.tensor([src, dst], dtype=torch.long), edge_attr, base_h3_grid


def latent_graph(base_h3_grid):
    """encoder.py:244-268 (== assimilator_encoder.py:218-242)."""
    base_h3_map = {h: i for i, h in enumerate(base_h3_grid)}
    src, dst, attrs = [], [], []
    for h3_index in base_h3_grid:
        for h in h3.grid_disk(h3_index, 1):
            d = h3.great_circle_distance(h3.cell_to_latlng(h3_index), h3.cell_to_latlng(h), unit="rads")
            attrs.append([np.sin(d), np.cos(d)])
            src.append(base_h3_map[h3_index])
            dst.append(base_h3_map[h])
    return torch.tensor([src, dst], dtype=torch.long), torch.tensor(attrs, dtype=torch.float)


def decoder_graph(lat_lons, resolution=2):
    """assimilator_decoder.py:69-106."""
    base_h3_grid = sorted(list(h3.uncompact_cells(h3.get_res0_cells(), resolution)))
    num_h3 = len(base_h3_grid)
    h3_grid = [h3.latlng_to_cell(lat, lon, resolution) for lat, lon in lat_lons]
    h3_to_index = {}
    h_index = len(base_h3_grid)
    for h in base_h3_grid:
        if h not in h3_to_index:
            h_index -= 1
            h3_to_index[h] = h_index
    src, dst, attrs = [], [], []
    for node_index, cell in enumerate(h3_grid):
        for h in h3.grid_disk(cell, 1):
            d = h3.great_circle_distance(lat_lons[node_index], h3.cell_to_latlng(h), unit="rads")
            attrs.append([np.sin(d), np.cos(d)])
            src.append(h3_to_index[h])
            dst.append(node_index + num_h3)
    return torch.tensor([src, dst], dtype=torch.long), torch.tensor(attrs, dtype=torch.float), num_h3


def assimilator_input_graph(lat_lon_heights, base_h3_grid, resolution=2):
    """assimilator_encoder.py:170-216 (edge attr = [sin d, cos d, height])."""
    num_latlons = lat_lon_heights.shape[0]
    h3_grid = [h3.latlng_to_cell(float(lat), float(lon), resolution) for lat, lon, _ in lat_lon_heights]
    h3_mapping = {}
    h_index = len(base_h3_grid)
    for h in base_h3_grid:
        if h not in h3_mapping:
            h_index -= 1
            h3_mapping[h] = h_index + num_latlons
    dists = []
    for idx, cell in enumerate(h3_grid):
        lat, lon, height = lat_lon_heights[idx]
        d = h3.great_circle_distance((float(lat), float(lon)), h3.cell_to_latlng(cell), unit="rads")
        dists.append([np.sin(d), np.cos(d), float(height)])
    edge_attr = torch.tensor(dists, dtype=torch.float)
    src = list(range(num_latlons))
    dst = [h3_mapping[c] for c in h3_grid]
    return torch.tensor([src, dst], dtype=torch.long), edge_attr


# ----------------------------------------------------------------------------------------------------------------
# arithmetic
# ----------------------------------------------------------------------------------------------------------------
def mlp(sd, prefix, x, hidden_layers=2, norm=True):
    """graph_net_block.py:45-61: Linear,ReLU,(Linear,ReLU)x(hl-1),Linear,[LayerNorm eps 1e-5]."""
    for i in range(hidden_layers):
        x = F.relu(F.linear(x, sd[f"{prefix}.model.{2 * i}.weight"], sd[f"{prefix}.model.{2 * i}.bias"]))
    j = 2 * hidden_layers
    x = F.linear(x, sd[f"{prefix}.model.{j}.weight"], sd[f"{prefix}.model.{j}.bias"])
    if norm:
        w = sd[f"{prefix}.model.{j + 1}.weight"]
        x = F.layer_norm(x, (w.shape[0],), w, sd[f"{prefix}.model.{j + 1}.bias"], 1e-5)
    return x


def gnn_block(sd, prefix, x, edge_index, edge_attr, hl_node=2, hl_edge=2):
    """One MetaLayer(EdgeProcessor, NodeProcessor): graph_net_block.py:131-135 and :184-191."""
    row, col = edge_index[0], edge_index[1]
    out = torch.cat([x[row], x[col], edge_attr], -1)
    out = mlp(sd, f"{prefix}.edge_model.edge_mlp", out, hl_edge)
    out += edge_attr
    edge_attr = out
    agg = torch.zeros((x.size(0), edge_attr.size(1)), dtype=x.dtype, device=x.device).scatter_add_(
        0, col.view(-1, 1).expand_as(edge_attr), edge_attr
    )
    out = torch.cat([x, agg], dim=-1)
    out = mlp(sd, f"{prefix}.node_model.node_mlp", out, hl_node)
    out += x
    return out, edge_attr


def graph_processor(sd, prefix, x, edge_index, edge_attr, num_blocks, hl_node=2, hl_edge=2):
    """graph_net_block.py:279-301."""
    for b in range(num_blocks):
        x, edge_attr = gnn_block(sd, f"{prefix}.blocks.{b}", x, edge_index, edge_attr, hl_node, hl_edge)
    return x, edge_attr


def _replicate(edge_index, batch):
    """encoder.py:212-218 / assimilator_decoder.py:180-186."""
    m = torch.max(edge_index)
    return torch.cat([edge_index + i * m + i for i in range(batch)], dim=1)


def encoder_forward(sd, g, features, prefix="encoder", hl_node=2, hl_edge=2):
    """encoder.py:197-242 (replicated-graph branch; the Forecaster never enables efficient_batching).
    g: dict with enc_edge_index, enc_edge_attr, lat_edge_index, lat_edge_attr, num_latlons, num_h3."""
    B = features.shape[0]
    h3_nodes = sd[f"{prefix}.h3_nodes"]
    feats = torch.cat([features, h3_nodes.unsqueeze(0).expand(B, -1, -1)], dim=1)
    feats = feats.reshape(-1, feats.shape[-1])
    out = mlp(sd, f"{prefix}.node_encoder", feats, hl_node)
    edge_attr = mlp(sd, f"{prefix}.edge_encoder", g["enc_edge_attr"], hl_edge)
    edge_attr = edge_attr.repeat(B, 1)
    edge_index = _replicate(g["enc_edge_index"], B)
    out, _ = graph_processor(sd, f"{prefix}.graph_processor", out, edge_index, edge_attr, 1, hl_node, hl_edge)
    out = out.reshape(B, -1, out.shape[-1])[:, g["num_latlons"] :, :].reshape(-1, out.shape[-1])
    lat_ei = _replicate(g["lat_edge_index"], B)
    lat_ea = mlp(sd, f"{prefix}.latent_edge_encoder", g["lat_edge_attr"].repeat(B, 1), hl_edge)
    return out, lat_ei, lat_ea


def processor_forward(sd, x, edge_index, edge_attr, num_blocks=9, prefix="processor", hl_node=2, hl_edge=2):
    """processor.py:123-128 (no thermalizer)."""
    out, _ = graph_processor(sd, f"{prefix}.graph_processor", x, edge_index, edge_attr, num_blocks, hl_node, hl_edge)
    return out


def assimilator_decoder_forward(sd, g, processor_features, batch_size, prefix="decoder", hl_node=2, hl_edge=2, hl_dec=2):
    """assimilator_decoder.py:173-200 (replicated-graph branch). edge_encoder has 2 hidden layers hard-coded (:109)."""
    edge_attr = mlp(sd, f"{prefix}.edge_encoder", g["dec_edge_attr"], 2)
    edge_attr = edge_attr.repeat(batch_size, 1)
    edge_index = _replicate(g["dec_edge_index"], batch_size)
    feats = processor_features.reshape(batch_size, -1, processor_features.shape[-1])
    latlon_nodes = torch.zeros((batch_size, g["num_latlons"], feats.shape[-1]), dtype=feats.dtype, device=feats.device)
    feats = torch.cat([feats, latlon_nodes], dim=1).reshape(-1, feats.shape[-1])
    out, _ = graph_processor(sd, f"{prefix}.graph_processor", feats, edge_index, edge_attr, 1, hl_node, hl_edge)
    out = mlp(sd, f"{prefix}.node_decoder", out, hl_dec, norm=False)
    out = out.reshape(batch_size, -1, out.shape[-1])
    return out[:, g["num_h3"] :, :]


def build_forecaster_graphs(lat_lons, resolution=2):
    lat_lons = [tuple(map(float, p)) for p in lat_lons]
    enc_ei, enc_ea, base = encoder_graph(lat_lons, resolution)
    lat_ei, lat_ea = latent_graph(base)
    dec_ei, dec_ea, num_h3 = decoder_graph(lat_lons, resolution)
    return dict(
        enc_edge_index=enc_ei, enc_edge_attr=enc_ea, lat_edge_index=lat_ei, lat_edge_attr=lat_ea,
        dec_edge_index=dec_ei, dec_edge_attr=dec_ea, num_latlons=len(lat_lons), num_h3=num_h3,
    )  # fmt: skip


def forecaster_forward(sd, g, features, feature_dim=78, num_blocks=9, hl_node=2, hl_edge=2, hl_dec=2):
    """forecast.py:226-228 + decoder.py:92-94 (constraint_type='none', no thermalizer)."""
    with torch.no_grad():
        x, ei, ea = encoder_forward(sd, g, features, "encoder", hl_node, hl_edge)
        x = processor_forward(sd, x, ei, ea, num_blocks, "processor", hl_node, hl_edge)
        out = assimilator_decoder_forward(sd, g, x, features.shape[0], "decoder", hl_node, hl_edge, hl_dec)
        return out + features[..., :feature_dim]


def regional_graphs(lat_lons, resolution=2):
    """DynamicGraphBuilder.__call__ (dynamic_graph_builder.py:31-66, :100-155), loop for loop: the encoder graph (one edge per
    coordinate -> its cell, cells numbered over the sorted unique cells), the latent graph among those cells, and the cells' ranks
    in the global sorted cell list (rows of the embedding table)."""
    lat_lons = [tuple(map(float, p)) for p in lat_lons]
    all_h3 = sorted(h3.uncompact_cells(h3.get_res0_cells(), resolution))
    global_map = {c: i for i, c in enumerate(all_h3)}
    cells = [h3.latlng_to_cell(lat, lon, resolution) for lat, lon in lat_lons]
    unique_cells = sorted(set(cells))
    local = {c: i for i, c in enumerate(unique_cells)}
    n = len(lat_lons)
    src, dst, attr = [], [], []
    for i, (coord, cell) in enumerate(zip(lat_lons, cells)):
        d = h3.great_circle_distance(coord, h3.cell_to_latlng(cell), unit="rads")
        src.append(i), dst.append(n + local[cell]), attr.append([np.sin(d), np.cos(d)])
    enc_ei = torch.tensor([src, dst], dtype=torch.long)
    enc_ea = torch.tensor(attr, dtype=torch.float)
    ls, ld, la = [], [], []
    for cell in unique_cells:
        for h in h3.grid_disk(cell, 1):
            if h in local:
                d = h3.great_circle_distance(h3.cell_to_latlng(cell), h3.cell_to_latlng(h), unit="rads")
                ls.append(local[cell]), ld.append(local[h]), la.append([np.sin(d), np.cos(d)])
    return dict(enc_edge_index=enc_ei, enc_edge_attr=enc_ea, lat_edge_index=torch.tensor([ls, ld], dtype=torch.long),
                lat_edge_attr=torch.tensor(la, dtype=torch.float), h3_indices=[global_map[c] for c in unique_cells], num_obs=n)  # fmt: skip


def regional_forward(sd, g, features, output_dim=78, num_blocks=9, hl_node=2, hl_edge=2, hl_dec=2, global_context=None, lat_lons=None):
    """RegionalForecaster.forward (regional_forecast.py:233-298), one sample at a time as there; sd has the reference's keys."""
    with torch.no_grad():
        n = g["num_obs"]
        regional_h3 = sd["h3_embeddings"][torch.tensor(g["h3_indices"], dtype=torch.long)]
        enc_ea = mlp(sd, "edge_encoder", g["enc_edge_attr"], hl_edge)
        lat_ea = mlp(sd, "latent_edge_encoder", g["lat_edge_attr"], hl_edge)
        dec_ei = g["enc_edge_index"].flip(0)
        dec_ea = mlp(sd, "decoder_edge_encoder", g["enc_edge_attr"], hl_edge)
        outs = []
        for i in range(features.shape[0]):
            nodes = mlp(sd, "node_encoder", torch.cat([features[i], regional_h3], dim=0), hl_node)
            nodes, _ = graph_processor(sd, "encoder_gnn", nodes, g["enc_edge_index"], enc_ea.clone(), 1, hl_node, hl_edge)
            x = processor_forward(sd, nodes[n:], g["lat_edge_index"], lat_ea.clone(), num_blocks, "processor", hl_node, hl_edge)
            dec_nodes = torch.cat([torch.zeros(n, x.shape[-1]), x], dim=0)
            dec_nodes, _ = graph_processor(sd, "decoder_gnn", dec_nodes, dec_ei, dec_ea.clone(), 1, hl_node, hl_edge)
            outs.append(mlp(sd, "node_decoder", dec_nodes[:n], hl_dec, norm=True))  # built WITH the configured norm (:224-231)
        out = torch.stack(outs, dim=0) + features[..., :output_dim]
        if global_context is not None:  # BoundaryNudgingLayer.forward (:68-90) with the relaxation prior of :92-130
            lats = torch.tensor([ll[0] for ll in lat_lons], dtype=torch.float32) * (np.pi / 180.0)
            lons = torch.tensor([ll[1] for ll in lat_lons], dtype=torch.float32) * (np.pi / 180.0)
            a = torch.sin((lats - lats.mean()) / 2) ** 2 + torch.cos(lats) * torch.cos(lats.mean()) * torch.sin((lons - lons.mean()) / 2) ** 2
            dist = 2 * torch.asin(torch.sqrt(torch.clamp(a, 0.0, 1.0)))
            prior = (dist / dist.max() if dist.max() > 0 else torch.zeros_like(dist)).unsqueeze(-1).unsqueeze(0).expand(out.shape[0], -1, -1)
            h = torch.cat([out, global_context, prior], dim=-1)
            corr = mlp(sd, "nudging.blend_mlp", h, 1, norm=False)
            alpha = torch.clamp(prior + corr, 0.0, 1.0)
            out = (1 - alpha) * out + alpha * global_context
        return out


def assimilator_forward(sd, g_static, features, lat_lon_heights, resolution=2, num_blocks=9, hl_node=2, hl_edge=2, hl_dec=2):
    """analysis.py:147-149 with assimilator_encoder.py:118-168 (input graph rebuilt per call; h3_nodes is a plain
    zero tensor, not a parameter, assimilator_encoder.py:80). g_static: base_h3_grid, lat_*, dec_*, num_latlons(out), num_h3."""
    with torch.no_grad():
        B = features.shape[0]
        in_ei, in_ea = assimilator_input_graph(lat_lon_heights, g_static["base_h3_grid"], resolution)
        nobs = lat_lon_heights.shape[0]
        h3_nodes = torch.zeros((g_static["num_h3"], features.shape[-1]), dtype=torch.float)
        feats = torch.cat([features, h3_nodes.unsqueeze(0).expand(B, -1, -1)], dim=1).reshape(-1, features.shape[-1])
        out = mlp(sd, "encoder.node_encoder", feats, hl_node)
        edge_attr = mlp(sd, "encoder.edge_encoder", in_ea, hl_edge).repeat(B, 1)
        out, _ = graph_processor(sd, "encoder.graph_processor", out, _replicate(in_ei, B), edge_attr, 1, hl_node, hl_edge)
        out = out.reshape(B, -1, out.shape[-1])[:, nobs:, :].reshape(-1, out.shape[-1])
        lat_ei = _replicate(g_static["lat_edge_index"], B)
        lat_ea = mlp(sd, "encoder.latent_edge_encoder", g_static["lat_edge_attr"].repeat(B, 1), hl_edge)
        x = processor_forward(sd, out, lat_ei, lat_ea, num_blocks, "processor", hl_node, hl_edge)
        return assimilator_decoder_forward(sd, g_static, x, B, "decoder", hl_node, hl_edge, hl_dec)


def build_assimilator_graphs(output_lat_lons, resolution=2):
    output_lat_lons = [tuple(map(float, p)) for p in output_lat_lons]
    base = sorted(list(h3.uncompact_cells(h3.get_res0_cells(), resolution)))
    lat_ei, lat_ea = latent_graph(base)
    dec_ei, dec_ea, num_h3 = decoder_graph(output_lat_lons, resolution)
    return dict(
        base_h3_grid=base, lat_edge_index=lat_ei, lat_edge_attr=lat_ea, dec_edge_index=dec_ei, dec_edge_attr=dec_ea,
        num_latlons=len(output_lat_lons), num_h3=num_h3,
    )  # fmt: skip


def normalized_mse_loss(pred, target, feature_variance, lat_lons, normalize=False):
    """NormalizedMSELoss.forward restated op for op (graph_weather/models/losses.py:37-42, 60-94): squared error, optional
    division by the feature variance, mean over features, cos(lat) weights tiled per unique latitude, mean over batch x nodes."""
    fv = torch.tensor(feature_variance)
    unique_lats = sorted(set(lat for lat, _ in lat_lons))  # losses.py:38
    weights = torch.tensor([np.cos(lat * np.pi / 180.0) for lat in unique_lats], dtype=torch.float)  # losses.py:40-42
    out = (pred - target) ** 2  # losses.py:66
    if normalize:
        out = out / fv  # losses.py:69-70
    out = out.mean(-1)  # losses.py:74
    B = out.shape[0]
    num_nodes = int(np.prod(out.shape[1:]))  # losses.py:77-80
    out = out.view(B, num_nodes)
    num_unique = weights.shape[0]
    num_lon = num_nodes // num_unique  # losses.py:84-85
    weight_grid = weights.unsqueeze(1).expand(num_unique, num_lon).reshape(1, num_nodes).expand(B, num_nodes)  # losses.py:88-89
    return (out * weight_grid).mean()  # losses.py:92-95
