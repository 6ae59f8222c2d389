"""RegionalForecaster training on moving boxes: B new boxes every step, run as one `forward_regions` call on the union plan, against
the same boxes run one `forward` per region (each a new region: its own graphs, plans and weight uploads).  Both paths end every
step with an SGD step, so both upload (and, on tensor cores, repack) the changed weights at their next forward; they run the same
draw of boxes in alternating order.

    python tools/regional_batch_bench.py --regions 4 --max-points 2000 --extent 10 --train-precision bf16 [--use-checkpointing]

One JSON line: median ms/step and regions/s of both, the union plan's train_peak_bytes and device bytes, and the host set-up shares of the union
step (graph build; weight upload after the SGD step; upload of the graphs and h3_nodes rows, which also launches the per-graph
constants), with the GPU's name, power
limit and SM clock read in the same run.  Model: the 256-wide trunk, 9 blocks, 9 channels (RegionalDataset's samples)."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graph_weather_b200.regional import RegionalForecasterConfig  # noqa: E402


def boxes(rng, b, n, extent):
    """b boxes of n points on a regular grid `extent` degrees wide, at random centres."""
    k = math.ceil(math.sqrt(n))
    step = extent / k
    out = []
    for _ in range(b):
        lat0, lon0 = rng.uniform(-60, 60 - extent), rng.uniform(-180, 180 - extent)
        out.append([(lat0 + step * (i // k), lon0 + step * (i % k)) for i in range(n)])
    return out


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)  # fmt: skip
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=4)
    ap.add_argument("--max-points", type=int, default=2000)
    ap.add_argument("--extent", type=float, default=10.0)
    ap.add_argument("--train-precision", default="bf16", choices=["fp32_simt", "fp32", "bf16"])
    ap.add_argument("--use-checkpointing", action="store_true")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("regional_batch_bench.py measures on a CUDA device; none is available")
    torch.manual_seed(0)
    model = RegionalForecasterConfig(feature_dim=9, aux_dim=0, num_blocks=9, train_precision=a.train_precision,
                                     use_checkpointing=a.use_checkpointing).build().cuda().train()  # fmt: skip
    with torch.no_grad():
        model.h3_embeddings.normal_(0, 0.1)
    rng = np.random.default_rng(0)
    B, N = a.regions, a.max_points
    x = torch.randn(B, N, 9, device="cuda")
    t = torch.randn(B, N, 9, device="cuda")

    opt = torch.optim.SGD(model.parameters(), lr=1e-4)

    def union_step(regions):
        opt.zero_grad(set_to_none=True)
        out = model.forward_regions(x, regions)
        torch.nn.functional.mse_loss(out, t).backward()
        opt.step()

    def loop_step(regions):
        opt.zero_grad(set_to_none=True)
        for i, r in enumerate(regions):
            (torch.nn.functional.mse_loss(model(x[i: i + 1], r), t[i: i + 1]) / B).backward()
        opt.step()

    result = dict(regions=B, points=N, extent=a.extent, train_precision=a.train_precision, bounded=a.use_checkpointing, steps=a.steps)
    for _ in range(a.warmup):
        regions = boxes(rng, B, N, a.extent)
        union_step(regions), loop_step(regions)
    times = {"union": [], "per_region": []}
    setup = {"build": 0.0, "weights": 0.0, "upload": 0.0}
    for s in range(a.steps):
        regions = boxes(rng, B, N, a.extent)  # one draw per step, run by both paths (in alternating order)
        order = [("union", union_step), ("per_region", loop_step)]
        for name, step in order if s % 2 == 0 else order[::-1]:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(regions)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            if name == "union":
                for k in setup:
                    setup[k] += model.last_setup_s[k]
    for name, ts in times.items():
        ms = 1e3 * float(np.median(ts))
        result[f"{name}_ms_step"] = round(ms, 2)
        result[f"{name}_regions_per_s"] = round(B / (ms / 1e3), 1)
    total = sum(times["union"])
    for k, v in setup.items():
        result[f"union_setup_{k}_share"] = round(v / total, 3)
    plan = model._batch_engines[a.use_checkpointing].plan
    result["train_peak_bytes"] = plan.train_peak_bytes()
    result["plan_bytes"] = plan.device_bytes()
    result["capacity"] = model._batch_cap
    result["gpu"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
