"""Times the training step of Encoder -> Processor -> Decoder composed by hand (the reference's tests/test_model.py::test_end2end,
each stage built with `train_precision`) against GraphWeatherForecaster's own step on the same weights.
    python tools/stage_train_bench.py [--grid 0.25deg|1deg|2deg|5deg|10deg] [--batch B] [--steps K]
                                      [--train-precision fp32_simt|fp32|bf16] [--use-checkpointing]
One step = forward + NormalizedMSELoss + backward + SGD update.  --use-checkpointing builds the Encoder, the Decoder and the wrapper
with use_checkpointing=True: both sides take the bounded-memory step (the processor stays taped).  0.25deg is the 721 x 1440 ERA5
grid.  The two steps alternate step by step after two warm-up steps each, CUDA events around each step; prints one JSON line with
both medians, each plan's train_peak_bytes and device bytes after the last step, and the card name, power limit and SM clocks read
in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", default="1deg", choices=["0.25deg", "1deg", "2deg", "5deg", "10deg"])
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--train-precision", default="bf16", choices=["fp32_simt", "fp32", "bf16"])
    ap.add_argument("--use-checkpointing", action="store_true")
    a = ap.parse_args()
    import __graft_entry__ as ge

    ge.build()
    from train_step_bench import card

    from graph_weather_b200 import Decoder, Encoder, GraphWeatherForecaster, NormalizedMSELoss, Processor

    if a.grid == "0.25deg":
        ll = [(float(lat), float(lon)) for lat in np.linspace(-90.0, 90.0, 721) for lon in np.arange(0.0, 360.0, 0.25)]
    else:
        step = {"1deg": 1, "2deg": 2, "5deg": 5, "10deg": 10}[a.grid]
        ll = [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]
    torch.manual_seed(0)
    tp, cp = a.train_precision, a.use_checkpointing
    wrapper = GraphWeatherForecaster(ll, train_precision=tp, use_checkpointing=cp).cuda().train()
    stages = [Encoder(ll, input_dim=102, train_precision=tp, use_checkpointing=cp), Processor(train_precision=tp),
              Decoder(ll, train_precision=tp, use_checkpointing=cp)]  # fmt: skip
    for m, name in zip(stages, ("encoder", "processor", "decoder")):
        m.load_state_dict(getattr(wrapper, name).state_dict())
    enc, proc, dec = [m.cuda().train() for m in stages]
    crit = NormalizedMSELoss([1.0] * 78, ll, normalize=True)
    x = torch.randn(a.batch, len(ll), 102, device="cuda")
    y = torch.randn(a.batch, len(ll), 78, device="cuda")
    opts = {"composed": torch.optim.SGD([q for m in stages for q in m.parameters()], lr=1e-3),
            "wrapper": torch.optim.SGD(wrapper.parameters(), lr=1e-3)}  # fmt: skip

    def one(kind):
        opts[kind].zero_grad(set_to_none=True)
        if kind == "wrapper":
            out = wrapper(x)
        else:
            h, ei, ea = enc(x)
            out = dec(proc(h, ei, ea), x[..., :78])
        crit(out, y).backward()
        opts[kind].step()

    for _ in range(2):
        one("composed"), one("wrapper")
    times = {"composed": [], "wrapper": []}
    for i in range(2 * a.steps):
        kind = "composed" if i % 2 == 0 else "wrapper"
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        one(kind)
        e1.record()
        torch.cuda.synchronize()
        times[kind].append(e0.elapsed_time(e1))
    mods = {"encoder": enc, "processor": proc, "decoder": dec, "wrapper": wrapper}
    for m in mods.values():
        m._train_engine.plan.status()
    med = {k: round(sorted(v)[len(v) // 2], 2) for k, v in times.items()}
    print(json.dumps({"what": "training step (fwd + loss + bwd + SGD), stages composed vs the wrapper", "train_precision": tp,
                      "grid": a.grid, "batch": a.batch, "steps": a.steps, "use_checkpointing": cp, "median_ms": med,
                      "ratio": round(med["composed"] / med["wrapper"], 3),
                      "train_only": {k: m._train_engine.plan.train_only for k, m in mods.items()},
                      "train_peak_bytes": {k: m._train_engine.plan.train_peak_bytes() for k, m in mods.items()},
                      "plan_bytes": {k: m._train_engine.plan.device_bytes() for k, m in mods.items()}, "card": card()}))  # fmt: skip


if __name__ == "__main__":
    main()
