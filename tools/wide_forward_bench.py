"""Times the inference forward of train/run.py's model (605 + 40 features, node / edge / processor-hidden / decoder-hidden widths
of 1024, 6 blocks) in fp32_simt, fp32 and bf16, on the same seeded weights and inputs.
    python tools/wide_forward_bench.py [--grids 1deg,2deg] [--batches 1,4] [--steps K] [--out results.json]
Per (grid, batch, precision): median ms/step over K steps after two warm-up calls (CUDA events around each call), device time per
timing tag (gw_timing_*, one extra timed call), and max |tensor-core - fp32_simt| of the forecast.  Prints one JSON line per
configuration and the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

WIDE = dict(node_dim=1024, edge_dim=1024, hidden_dim_processor_node=1024, hidden_dim_processor_edge=1024, hidden_dim_decoder=1024,
            feature_dim=605, aux_dim=40, num_blocks=6)  # fmt: skip


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="1deg,2deg")
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as ge

    ge.build()
    from train_step_bench import card

    from graph_weather_b200 import GraphWeatherForecaster

    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    for g in a.grids.split(","):
        step = {"1deg": 1, "2deg": 2}[g]
        ll = [(float(lat), float(lon)) for lat in range(-90, 90, step) for lon in range(0, 360, step)]
        torch.manual_seed(0)
        sd = GraphWeatherForecaster(ll, **WIDE).state_dict()
        for b in (int(s) for s in a.batches.split(",")):
            x = torch.randn(b, len(ll), WIDE["feature_dim"] + WIDE["aux_dim"], generator=torch.Generator().manual_seed(1)).cuda()
            ref = None
            for prec in ("fp32_simt", "fp32", "bf16"):
                model = GraphWeatherForecaster(ll, **WIDE, precision=prec).cuda().eval()
                model.load_state_dict(sd)
                with torch.no_grad():
                    for _ in range(2):
                        out = model(x)
                    ts = []
                    for _ in range(a.steps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        out = model(x)
                        e1.record()
                        e1.synchronize()
                        ts.append(e0.elapsed_time(e1))
                    plan = model._engine.plan
                    plan.timing_enable(True)
                    model(x)
                    tags = plan.timing_read()
                    plan.timing_enable(False)
                if ref is None:
                    ref = out.double()
                r = {"grid": g, "batch": b, "precision": prec, "ms_per_step": sorted(ts)[len(ts) // 2], "ms_all": ts,
                     "max_abs_vs_fp32_simt": float((out.double() - ref).abs().max()), "device_ms_per_tag": tags}  # fmt: skip
                rows.append(r)
                print(json.dumps(r), flush=True)
                del model, out
                torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
