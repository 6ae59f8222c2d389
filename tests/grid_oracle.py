"""The reference arithmetic of GraphWeatherForecaster on a grid of any size: oracle/restate.py's forward and its training step
(tests/training_oracle.py) walked in chunks of grid rows, on any device and in any dtype, so the fp64 ground truth reaches the
0.25-degree ERA5 grid on the GPU (one fp64 tensor of its decoder edge rows alone is 7.27 M x 256 x 8 B = 14.9 GB per sample).

Every grid-sized stage of the model is separable by rows, so the chunks change the order of some sums and nothing else:
  * encoder: the node encoder and the edge MLP of each chunk of encoder edges (one per point, src = the point, dst = its mesh
    cell), summed into the mesh nodes' aggregate, which is carried from chunk to chunk.  The node MLP of the grid rows is not
    run: restate.encoder_forward discards its output (`[:, num_latlons:]`);
  * processor: mesh-sized, restate.processor_forward itself;
  * decoder: independent per output point given the mesh rows.  Its edges are grouped by destination point, so a chunk of points
    is a contiguous range of edges.  The node MLP and node decoder of the mesh rows are not run either: their output is the
    `[:, :num_h3]` that restate.assimilator_decoder_forward discards.
The batch-shared edge encoders run once per chunk of edge rows and are `.repeat(B, 1)`'d as there, so their gradients sum over the
samples the way the reference's do.  Every MLP is restate.mlp; concat orders, in-place residuals and LayerNorm eps are restate's.
Under autograd each chunk runs inside torch.utils.checkpoint: memory is one chunk's activations plus mesh-sized tensors, and the
decoder chunks return their share of the loss sum, so [B, N, 78] is never taped.

The graphs are graphs.py's vectorised builders (tests/test_graphs.py pins them to the reference's loops up to 0.25 degrees).  A
caller may hand in altered graphs: that is how the tests show what a single dropped or misplaced row does to the result."""
import contextlib

import numpy as np
import torch
from torch.utils.checkpoint import checkpoint

from graph_weather_b200 import graphs as gr
from oracle import restate


def build_graphs(lat_lons, resolution=2):
    """The encoder, mesh and decoder graphs of `lat_lons` (graphs.py's EncoderGraph, MeshGraph, DecoderGraph)."""
    return dict(enc=gr.build_encoder_graph(lat_lons, resolution), mesh=gr.build_mesh_graph(resolution),
                dec=gr.build_decoder_graph(lat_lons, resolution))  # fmt: skip


@contextlib.contextmanager
def exact_fp32():
    """fp32 matmuls in fp32 (no TF32) inside, the caller's settings restored after."""
    tf32, prec = torch.backends.cuda.matmul.allow_tf32, torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(prec)
        torch.backends.cuda.matmul.allow_tf32 = tf32


def _ckpt(fn, *args):
    """fn(*args), taped by recomputation when autograd records (checkpoint) and plainly otherwise."""
    if torch.is_grad_enabled():
        return checkpoint(fn, *args, use_reentrant=False, preserve_rng_state=False)
    return fn(*args)


class _Graphs:
    """The graphs as index / attribute tensors on `device`, attributes in `dtype`."""

    def __init__(self, graphs, batch, dtype, device):
        e, m, d = graphs["enc"], graphs["mesh"], graphs["dec"]
        self.N, self.H = e.num_latlons, e.num_h3
        # The reference batches by replicating each graph with offsets max(edge_index) + 1 (restate._replicate).  That is one
        # sample's node count only when the highest mesh id has an edge; otherwise its samples >= 1 are misaligned, and the
        # per-sample arithmetic here would not be what it computes.
        assert batch == 1 or int(e.edge_index.max()) == self.N + self.H - 1, "the reference's encoder replication is misaligned"

        def t(a, dt=torch.long):
            return torch.as_tensor(np.ascontiguousarray(a)).to(device=device, dtype=dt)

        self.enc_src, self.enc_slot, self.enc_attr = t(e.edge_index[0]), t(e.edge_index[1] - self.N), t(e.edge_attr, dtype)
        self.lat_ei, self.lat_attr = t(m.edge_index), t(m.edge_attr, dtype)
        self.dec_src, self.dec_dst, self.dec_attr = t(d.edge_index[0]), t(d.edge_index[1] - self.H), t(d.edge_attr, dtype)
        self.dec_ptr = np.asarray(d.ptr, dtype=np.int64)
        assert self.dec_ptr[-1] == d.edge_index.shape[1] and np.all(np.diff(d.edge_index[1]) >= 0), "decoder edges not grouped by point"


def _mesh_side(sd, g, x, B, chunk, hl_node, hl_edge):
    """restate.encoder_forward: the mesh nodes after the encoder block [B * H, D] and the replicated latent graph."""
    H, dev = g.H, x.device
    # node encoder on the mesh rows (the h3_nodes table broadcast to every sample, as the reference concatenates it)
    xm = restate.mlp(sd, "encoder.node_encoder", sd["encoder.h3_nodes"].unsqueeze(0).expand(B, -1, -1).reshape(B * H, -1), hl_node)
    De = sd["encoder.edge_encoder.model.%d.weight" % (2 * hl_edge)].shape[0]
    off = (torch.arange(B, device=dev) * H)[:, None]

    def enc_chunk(agg, xm, x, e0, e1):
        src, slot = g.enc_src[e0:e1], g.enc_slot[e0:e1]
        xp = restate.mlp(sd, "encoder.node_encoder", x[:, src].reshape(B * (e1 - e0), -1), hl_node)  # x[row]: the points
        ea = restate.mlp(sd, "encoder.edge_encoder", g.enc_attr[e0:e1], hl_edge).repeat(B, 1)
        col = (slot[None, :] + off).reshape(-1)
        out = torch.cat([xp, xm[col], ea], -1)
        out = restate.mlp(sd, "encoder.graph_processor.blocks.0.edge_model.edge_mlp", out, hl_edge)
        out += ea
        return agg.scatter_add(0, col.view(-1, 1).expand_as(out), out)

    agg = torch.zeros((B * H, De), dtype=xm.dtype, device=dev)
    E = int(g.enc_src.numel())
    for e0 in range(0, E, chunk):
        agg = _ckpt(enc_chunk, agg, xm, x, e0, min(E, e0 + chunk))
    out = restate.mlp(sd, "encoder.graph_processor.blocks.0.node_model.node_mlp", torch.cat([xm, agg], dim=-1), hl_node)
    out += xm
    lat_ei = restate._replicate(g.lat_ei, B)
    lat_ea = restate.mlp(sd, "encoder.latent_edge_encoder", g.lat_attr.repeat(B, 1), hl_edge)
    return out, lat_ei, lat_ea


def _decoder_chunk(sd, g, px, x, B, p0, p1, feature_dim, hl_node, hl_edge, hl_dec):
    """restate.assimilator_decoder_forward + the residual of forecaster_forward on points [p0, p1): [B, p1 - p0, feature_dim]."""
    e0, e1 = int(g.dec_ptr[p0]), int(g.dec_ptr[p1])
    c, ce, dev = p1 - p0, e1 - e0, px.device
    ea = restate.mlp(sd, "decoder.edge_encoder", g.dec_attr[e0:e1], 2).repeat(B, 1)
    b = torch.arange(B, device=dev)[:, None]
    row = (g.dec_src[e0:e1][None, :] + b * g.H).reshape(-1)
    col = (g.dec_dst[e0:e1][None, :] - p0 + b * c).reshape(-1)  # the chunk's points, sample-major
    xn = torch.zeros((B * c, px.shape[-1]), dtype=px.dtype, device=dev)  # the decoder's lat/lon nodes enter as zeros
    out = torch.cat([px[row], xn[col], ea], -1)
    out = restate.mlp(sd, "decoder.graph_processor.blocks.0.edge_model.edge_mlp", out, hl_edge)
    out += ea
    agg = torch.zeros((B * c, out.size(1)), dtype=out.dtype, device=dev).scatter_add_(0, col.view(-1, 1).expand_as(out), out)
    out = restate.mlp(sd, "decoder.graph_processor.blocks.0.node_model.node_mlp", torch.cat([xn, agg], dim=-1), hl_node)
    out += xn
    out = restate.mlp(sd, "decoder.node_decoder", out, hl_dec, norm=False)
    return out.reshape(B, c, -1) + x[:, p0:p1, :feature_dim]


def _trunk(sd, g, x, chunk, num_blocks, hl_node, hl_edge):
    B = x.shape[0]
    ex, ei, ea = _mesh_side(sd, g, x, B, chunk, hl_node, hl_edge)
    return _ckpt(restate.processor_forward, sd, ex, ei, ea, num_blocks, "processor", hl_node, hl_edge)


def _on(sd, x, dtype, device, grad):
    sd = {k: v.to(device=device, dtype=dtype).clone().requires_grad_(grad) for k, v in sd.items()}
    return sd, x.to(device=device, dtype=dtype).clone().requires_grad_(grad)


def forward(sd, graphs, x, dtype, device, chunk, feature_dim=78, num_blocks=9, hl_node=2, hl_edge=2, hl_dec=2):
    """restate.forecaster_forward: the forecast [B, N, feature_dim] in `dtype` on `device`, `chunk` grid rows at a time."""
    with torch.no_grad(), exact_fp32():
        sd, x = _on(sd, x, dtype, device, False)
        g = _Graphs(graphs, x.shape[0], dtype, device)
        px = _trunk(sd, g, x, chunk, num_blocks, hl_node, hl_edge)
        out = torch.empty((x.shape[0], g.N, feature_dim), dtype=dtype, device=device)
        for p0 in range(0, g.N, chunk):
            p1 = min(g.N, p0 + chunk)
            out[:, p0:p1] = _decoder_chunk(sd, g, px, x, x.shape[0], p0, p1, feature_dim, hl_node, hl_edge, hl_dec)
        return out


def loss_weights(lat_lons, var, dtype, device):
    """restate.normalized_mse_loss's feature variances [F] and its per-row latitude weights [N] (cos(lat) of the unique latitudes,
    tiled by position), in fp32 as there, then in `dtype`."""
    unique_lats = sorted(set(lat for lat, _ in lat_lons))
    w = torch.tensor([np.cos(lat * np.pi / 180.0) for lat in unique_lats], dtype=torch.float)
    num_lon = len(lat_lons) // len(unique_lats)
    return torch.tensor(var).to(device=device, dtype=dtype), w.repeat_interleave(num_lon).to(device=device, dtype=dtype)


def train_step(sd, graphs, x, target, var, ll, dtype, device, chunk, feature_dim=78, num_blocks=9, hl_node=2, hl_edge=2, hl_dec=2):
    """training_oracle.forecaster_oracle_step (no constraint) chunk by chunk: encoder -> processor -> decoder + the first
    feature_dim features, NormalizedMSELoss(normalize=True) as restate.normalized_mse_loss states it, backward.
    Returns (out, loss, d features, {name: grad}) on the host."""
    with torch.enable_grad(), exact_fp32():
        sd, x = _on(sd, x, dtype, device, True)
        B = x.shape[0]
        g = _Graphs(graphs, B, dtype, device)
        fv, w = loss_weights(ll, var, dtype, device)
        t = target.to(device=device, dtype=dtype)
        out = torch.empty((B, g.N, feature_dim), dtype=dtype, device=device)
        px = _trunk(sd, g, x, chunk, num_blocks, hl_node, hl_edge)

        def loss_chunk(px, x, p0, p1):
            y = _decoder_chunk(sd, g, px, x, B, p0, p1, feature_dim, hl_node, hl_edge, hl_dec)
            out[:, p0:p1] = y.detach()
            return ((((y - t[:, p0:p1]) ** 2) / fv).mean(-1) * w[p0:p1]).sum()

        total = sum(_ckpt(loss_chunk, px, x, p0, min(g.N, p0 + chunk)) for p0 in range(0, g.N, chunk))
        loss = total / (B * g.N)
        loss.backward()
        return out.cpu(), float(loss.detach()), x.grad.cpu(), {k: v.grad.cpu() for k, v in sd.items()}
