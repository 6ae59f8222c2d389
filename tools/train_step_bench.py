"""Times one training step (forward with tape + NormalizedMSELoss + backward + SGD update) of GraphWeatherForecaster, GraphCast,
GraphWeatherAssimilator or RegionalForecaster.
    python tools/train_step_bench.py [--model forecaster|graphcast|assimilator|regional] [--grid 0.25deg|1deg|2deg|5deg|10deg]
                                     [--batch B] [--steps K] [--train-precision fp32_simt|fp32|bf16] [--feature-dim F] [--aux-dim A]
                                     [--num-blocks NB] [--width W] [--constraint-type none|additive|multiplicative|softmax]
                                     [--use-checkpointing] [--fit-batch] [--n-obs N] [--rollout K [--compare-plain]]
                                     [--extent DEG] [--max-points N] [--moving-region] [--processor-segments S] [--deterministic]
The model defaults to the README's 78 + 24 features, 9 blocks, 256-wide.  --model graphcast: GraphCast(input_dim = output_dim =
--feature-dim, hidden_dim = --width or 256); its bounded step is selected by --use-checkpointing (the same step
GraphCastConfig.balanced_checkpointing / full_checkpointing select).  --model assimilator: GraphWeatherAssimilator(output_lat_lons =
the grid, analysis_dim = --feature-dim) on --n-obs observations (2 values each) at random (lat, lon, height), a new set for every
step, so every step rebuilds the observation graph; the reference README's configuration is --grid 5deg --feature-dim 24 --batch 1
--n-obs 2660.  The reference's ERA5 training scripts:
    train/run_fulll.py  --feature-dim 597 --aux-dim 24 --num-blocks 6 (1-degree grid)
    train/run.py        --feature-dim 605 --aux-dim 40 --num-blocks 6 --width 1024 --grid 2deg
(--width sets the node / edge / hidden / decoder widths together.)
Prints one JSON line: ms/step, samples/s, the device time of the step's phases (libgwb200 timing tags train_*; one extra timed
step after the measured ones, since the per-launch events add a little host work), peak device memory, and the card name and
power limit read in the same run.  --use-checkpointing runs the bounded-memory step (a training-only plan; 0.25deg is the 721 x 1440
grid bench.py uses).  Every run reports train_peak_bytes (the step's working allocations, gw_train_peak_bytes) and the plan's
device_bytes.  --fit-batch: the largest batch whose step should fit on the card, from the device bytes the step needs at
batches 1 and 2 (train_peak_bytes + plan bytes + torch's reserved peak, each linear in the batch), confirmed by one run at that
batch in a fresh process.
--rollout K: one step is a K-step autoregressive rollout trained as one -- K forwards inside model.multi_step(), each fed the
previous forecast (the forecaster's auxiliary columns stay those of the first input), the summed loss, one backward chain and the
SGD update; "rollout" reports gw_tape_bytes of each of the K tapes (what each forward keeps until the backward), and
train_peak_bytes covers all of them.  --compare-plain (with --rollout 1) also times the window's one-step step and the plain step
alternately, step by step, and reports both medians.
--model regional: RegionalForecaster (--feature-dim + --aux-dim features, --num-blocks, --width; the loss is torch's MSELoss) on
synthetic regions shaped like the reference's RegionalDataset samples: a square box of side --extent degrees at a seeded random
centre on the 0.25-degree grid, --max-points of its points drawn without replacement (--grid is not used).  One box is reused for
every step, or with --moving-region a new box is drawn for every step, as the dataset does: that step also builds the region's
graphs on the host, creates its plans and uploads the graphs and weights, so the difference of the two is the per-region set-up cost.
--processor-segments S: processor.set_checkpoint_segments(S) -- the backward recomputes the processor in segments of S blocks
(-1: one segment) instead of keeping its tape; "tape_bytes" (gw_tape_bytes of every tape of the last step, read before its backward)
shows what that saves.
--deterministic: torch.use_deterministic_algorithms(True) for the whole run, so that every backward sums its parameter gradients in
a fixed order (gw_train_set_deterministic); "deterministic_ws_bytes" is the fixed-order workspace the plan holds after the run.
With --constraint-type the step includes PhysicalConstraintLayer; the constraint backward
(gw_constraint_backward, no timing tag of the plan) is also timed on its own with CUDA events around it, on the step's shapes."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """Name, enforced power limit and SM clocks (now and at most) of cuda:0 (read-only query; None where nvidia-smi is unavailable)."""
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_clock_mhz": None, "sm_clock_max_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)  # fmt: skip
        if r.returncode == 0 and r.stdout.strip():
            name, pl, clk, clk_max = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
            info["name"], info["power_limit_w"], info["sm_clock_mhz"], info["sm_clock_max_mhz"] = name, float(pl), float(clk), float(clk_max)
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return info


def constraint_backward_time(model, x, F, reps=20):
    """Device time of one gw_constraint_backward on the step's shapes (d_hr and d_lr; CSR build included), CUDA events around
    `reps` calls, and the bytes it must move at least: the passes over B x N x F floats each type makes."""
    layer = model.constraint
    B, N = x.shape[0], x.shape[1]
    g = torch.Generator(device="cuda").manual_seed(2)
    hr32, lr32 = layer._prepare(torch.randn(B, N, F, device="cuda", generator=g), x[..., :F])
    dy = torch.randn(B, N, F, device="cuda", generator=g)
    src = model._constraint_cell(hr32)
    layer._backward(dy, hr32, lr32, src, True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        layer._backward(dy, hr32, lr32, src, True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    # additive: dy (sums) + dy (rows) + d_hr + d_lr; multiplicative: + hr, lr (means) + hr (sums); softmax: dy, hr, lr, d_hr, d_lr
    passes = {"additive": 4, "multiplicative": 7, "softmax": 5}[layer.constraint_type]
    nbytes = passes * B * N * F * 4
    return {"ms": round(ms, 4), "min_bytes": nbytes, "achieved_gb_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="forecaster", choices=["forecaster", "graphcast", "assimilator", "regional"])
    ap.add_argument("--grid", default="1deg", choices=["0.25deg", "1deg", "2deg", "5deg", "10deg"])
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--train-precision", default="fp32_simt", choices=["fp32_simt", "fp32", "bf16"])
    ap.add_argument("--feature-dim", type=int, default=78)
    ap.add_argument("--aux-dim", type=int, default=24)
    ap.add_argument("--num-blocks", type=int, default=9)
    ap.add_argument("--width", type=int, default=None, help="node / edge / hidden / decoder width (default: the model's 256 / 128)")
    ap.add_argument("--constraint-type", default="none", choices=["none", "additive", "multiplicative", "softmax"])
    ap.add_argument("--use-checkpointing", action="store_true", help="the bounded-memory training step (training-only plan)")
    ap.add_argument("--fit-batch", action="store_true", help="report the largest batch that should fit, confirmed by one run")
    ap.add_argument("--n-obs", type=int, default=2660, help="observations per step (--model assimilator)")
    ap.add_argument("--rollout", type=int, default=0, help="K: one step is K forwards inside model.multi_step() and one backward")
    ap.add_argument("--compare-plain", action="store_true", help="with --rollout 1: alternate the window's step with the plain one")
    ap.add_argument("--extent", type=float, default=20.0, help="side of the square region in degrees (--model regional)")
    ap.add_argument("--max-points", type=int, default=2000, help="points per region (--model regional)")
    ap.add_argument("--moving-region", action="store_true", help="a new region for every step (--model regional)")
    ap.add_argument("--processor-segments", type=int, default=0, help="processor.set_checkpoint_segments(S): 0 none, N blocks, -1 one")
    ap.add_argument("--deterministic", action="store_true", help="torch.use_deterministic_algorithms(True): bit-repeatable gradients")
    a = ap.parse_args()
    if a.model == "regional" and (a.rollout or a.fit_batch):
        ap.error("--model regional: no --rollout or --fit-batch")
    if a.model != "forecaster" and a.constraint_type != "none":
        ap.error("--constraint-type applies to --model forecaster")
    if a.rollout and a.model == "assimilator":
        ap.error("--rollout: GraphWeatherAssimilator has no multi_step()")
    if a.compare_plain and a.rollout != 1:
        ap.error("--compare-plain compares the window's K = 1 step with the plain step: use --rollout 1")
    import __graft_entry__ as ge

    ge.build()
    import numpy as np

    from graph_weather_b200 import GraphCast, GraphWeatherAssimilator, GraphWeatherForecaster, NormalizedMSELoss
    from graph_weather_b200.regional import RegionalForecasterConfig

    if a.grid == "0.25deg":
        ll = [(float(lat), float(lon)) for lat in np.linspace(-90.0, 90.0, 721) for lon in np.arange(0.0, 360.0, 0.25)]
    else:
        step = {"1deg": 1, "2deg": 2, "5deg": 5, "10deg": 10}[a.grid]
        ll = [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]
    torch.manual_seed(0)
    F = a.feature_dim
    if a.model == "graphcast":
        dims = dict(input_dim=F, output_dim=F, num_processor_blocks=a.num_blocks, hidden_dim=a.width or 256)
        model = GraphCast(ll, train_precision=a.train_precision, use_checkpointing=a.use_checkpointing, **dims).cuda().train()
        n_in, f_in = len(ll), F
    elif a.model == "assimilator":
        dims = dict(analysis_dim=F, num_blocks=a.num_blocks, n_obs=a.n_obs)
        if a.width is not None:
            dims.update(node_dim=a.width, edge_dim=a.width, hidden_dim_processor_node=a.width, hidden_dim_processor_edge=a.width,
                        hidden_dim_decoder=a.width)  # fmt: skip
        model = GraphWeatherAssimilator(output_lat_lons=ll, train_precision=a.train_precision, use_checkpointing=a.use_checkpointing,
                                        **{k: v for k, v in dims.items() if k != "n_obs"}).cuda().train()  # fmt: skip
        n_in, f_in = a.n_obs, 2
    elif a.model == "regional":
        dims = dict(feature_dim=F, aux_dim=a.aux_dim, num_blocks=a.num_blocks, extent=a.extent, max_points=a.max_points,
                    moving_region=a.moving_region)  # fmt: skip
        if a.width is not None:
            dims.update(node_dim=a.width, edge_dim=a.width, hidden_dim_processor_node=a.width, hidden_dim_processor_edge=a.width,
                        hidden_dim_decoder=a.width)  # fmt: skip
        cfg = {k: v for k, v in dims.items() if k not in ("extent", "max_points", "moving_region")}
        model = RegionalForecasterConfig(train_precision=a.train_precision, use_checkpointing=a.use_checkpointing, **cfg).build().cuda().train()
        box_rng = np.random.default_rng(0)
        lat_g, lon_g = np.arange(-90.0, 90.001, 0.25), np.arange(0.0, 360.0, 0.25)

        def box():
            """RegionalDataset._sample_box on the 0.25-degree grid: a new list of (lat, lon)."""
            half = a.extent / 2.0
            lat_c, lon_c = box_rng.uniform(lat_g.min() + half, lat_g.max() - half), box_rng.uniform(lon_g.min() + half, lon_g.max() - half)
            glat, glon = np.meshgrid(lat_g[np.abs(lat_g - lat_c) <= half], lon_g[np.abs(lon_g - lon_c) <= half], indexing="ij")
            pick = box_rng.choice(glat.size, size=min(a.max_points, glat.size), replace=False)
            return [(float(p), float(q)) for p, q in zip(glat.ravel()[pick], glon.ravel()[pick])]

        fixed = box()
        ll = fixed
        n_in, f_in = len(fixed), F + a.aux_dim
    else:
        dims = dict(feature_dim=F, aux_dim=a.aux_dim, num_blocks=a.num_blocks)
        if a.width is not None:
            dims.update(node_dim=a.width, edge_dim=a.width, hidden_dim_processor_node=a.width, hidden_dim_processor_edge=a.width,
                        hidden_dim_decoder=a.width)  # fmt: skip
        model = GraphWeatherForecaster(ll, train_precision=a.train_precision, constraint_type=a.constraint_type,
                                       use_checkpointing=a.use_checkpointing, **dims).cuda().train()  # fmt: skip
        n_in, f_in = len(ll), F + a.aux_dim
    model.processor.set_checkpoint_segments(a.processor_segments)
    torch.use_deterministic_algorithms(a.deterministic)
    crit = torch.nn.functional.mse_loss if a.model == "regional" else NormalizedMSELoss([1.0] * F, ll, normalize=True)
    opt = torch.optim.SGD(model.parameters(), lr=1e-3)
    tape_bytes = []  # gw_tape_bytes of every tape of the last step, read before its backward

    def measure(batch, steps):
        """(ms/step, losses, torch peak bytes, train_peak_bytes, plan device_bytes, step function, inputs) of `steps` timed steps."""
        x = torch.randn(batch, n_in, f_in, device="cuda")
        y = torch.randn(batch, n_in if a.model == "regional" else len(ll), F, device="cuda")
        g = torch.Generator(device="cuda").manual_seed(1)

        def obs():  # a new observation set: (lat, lon, height)
            u = torch.rand(n_in, 3, device="cuda", generator=g)
            return torch.stack([u[:, 0] * 180.0 - 90.0, u[:, 1] * 360.0, u[:, 2]], 1)

        def one(rollout=a.rollout):
            opt.zero_grad(set_to_none=True)
            if rollout:  # K forwards in one multi_step() window, each fed the previous forecast (+ the fixed aux columns)
                with model.multi_step():
                    inp, loss = x, 0.0
                    for t in range(rollout):
                        out = model(inp)
                        loss = loss + crit(out, y)
                        if t + 1 < rollout:
                            inp = torch.cat([out, x[..., F:]], -1) if f_in > F else out
            elif a.model == "regional":  # (every box has max_points points: the inputs keep their shapes)
                loss = crit(model(x, box() if a.moving_region else fixed), y)
            else:
                loss = crit(model(x, obs()) if a.model == "assimilator" else model(x), y)
            tape_bytes[:] = [t.bytes() for t in model._train_engine.plan.live_tapes()]
            loss.backward()
            opt.step()
            return loss.detach()

        for _ in range(2):
            one()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.reset_peak_memory_stats()
        losses = []
        e0.record()
        for _ in range(steps):
            losses.append(one())
        e1.record()
        torch.cuda.synchronize()
        plan = model._train_engine.plan
        return e0.elapsed_time(e1) / steps, losses, torch.cuda.max_memory_allocated(), plan.train_peak_bytes(), plan.device_bytes(), one, x

    if a.fit_batch:
        need = {}
        for b in (1, 2):
            _, _, _, trp, pb, _, _ = measure(b, 1)
            need[b] = torch.cuda.max_memory_reserved() + trp + pb
        per = need[2] - need[1]
        total = torch.cuda.mem_get_info()[1]
        # a tenth of the card for the CUDA context and the allocators' slack (the stream-ordered pool holds more than its live bytes)
        bfit = max(1, int((0.9 * total - (need[1] - per)) // per))
        # the confirming run is a fresh process: this one's allocators still cache the blocks of batches 1 and 2
        argv = [v for v in sys.argv[1:] if v != "--fit-batch"] + ["--batch", str(bfit)]
        r = subprocess.run([sys.executable, os.path.abspath(__file__), *argv], capture_output=True, text=True)
        lines = [v for v in r.stdout.splitlines() if v.startswith("{")]
        res = json.loads(lines[-1]) if r.returncode == 0 and lines else {"failed": r.stderr[-2000:]}
        res["fit_batch"] = {"need_bytes_b1": need[1], "need_bytes_b2": need[2], "card_bytes": total, "batch": bfit}
        print(json.dumps(res))
        return
    ms, losses, peak, train_peak, plan_bytes, one, x = measure(a.batch, a.steps)
    free, total = torch.cuda.mem_get_info()
    rollout = None
    if a.rollout:
        rollout = {"K": a.rollout, "tape_bytes": list(tape_bytes), "tape_gib": [round(v / 2**30, 3) for v in tape_bytes]}
    if a.compare_plain:  # the window's K = 1 step and the plain step, alternated step by step (CUDA events around each)
        times = {"window": [], "plain": []}
        for i in range(2 * a.steps):
            kind = "window" if i % 2 == 0 else "plain"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            one(rollout=1 if kind == "window" else 0)
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1))
        rollout["compare_plain_median_ms"] = {k: round(sorted(v)[len(v) // 2], 3) for k, v in times.items()}
    # per-phase device time of one more step (the plan's stream-ordered tape allocations are outside torch's allocator: the
    # device-wide figure is reported too)
    plan = model._train_engine.plan
    plan.timing_enable(True)
    one()
    tags = plan.timing_read()
    plan.timing_enable(False)
    phases = {k: round(v[1], 3) for k, v in tags.items() if k.startswith("train_") or k == "const"}
    plan.status()
    cbwd = constraint_backward_time(model, x, F) if a.constraint_type != "none" else None
    print(json.dumps({"what": "training step (fwd + loss + bwd + SGD)", "model": a.model, "train_precision": a.train_precision, "grid": None if a.model == "regional" else a.grid, "batch": a.batch,
                      "use_checkpointing": a.use_checkpointing, "processor_segments": a.processor_segments,
                      "deterministic": a.deterministic, "deterministic_ws_bytes": plan.deterministic_bytes(),
                      "tape_bytes": list(tape_bytes), "rollout": rollout, "train_peak_gib": round(train_peak / 2**30, 3),
                      "plan_device_gib": round(plan_bytes / 2**30, 3),
                      "dims": dims, "constraint_type": a.constraint_type, "constraint_backward": cbwd,
                      "n_params": sum(q.numel() for q in model.parameters()),
                      "ms_per_step": ms, "samples_per_s": a.batch / (ms * 1e-3), "phase_ms": phases,
                      "phase_launches": {k: v[0] for k, v in tags.items() if k.startswith("train_")},
                      "torch_peak_alloc_gib": round(peak / 2**30, 2), "device_mem_used_gib": round((total - free) / 2**30, 1),
                      "card": card(), "losses": [float(v) for v in losses]}))  # fmt: skip


if __name__ == "__main__":
    main()
