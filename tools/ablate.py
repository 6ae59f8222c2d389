"""Timing attribution for the tensor-core chain kernel: builds the library with -DGW_ABLATE (into build_abl/, here in the
build container: `python tools/ablate.py --build-only`) and, on the GPU box, times every kernel class of the 1-degree
forward with parts of the pipeline switched off (results are wrong under a non-zero mask; only the times mean anything).

    GW_B200_LIB=build_abl/libgwb200.so python tools/ablate.py --masks 0,1,2,4,...
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BITS = {1: "fence", 2: "loads", 4: "convert", 8: "stores", 16: "ln", 128: "weights"}


def build_abl(extra=()):
    import __graft_entry__ as ge

    out = os.path.join(ROOT, "build_abl")
    os.makedirs(out, exist_ok=True)
    objs = []
    for s in ge.SOURCES:
        o = os.path.join(out, s[:-3] + ".o")
        subprocess.run([ge.NVCC, *ge.FLAGS, *ge.EXTRA_FLAGS.get(s, []), "-DGW_ABLATE", *extra, "-c", os.path.join(ge.CSRC, s), "-o", o], check=True)
        objs.append(o)
    subprocess.run([ge.NVCC, "-shared", "-o", os.path.join(out, "libgwb200.so"), *objs, "-lcudart"], check=True)
    print("built", out)


def name(mask):
    return "+".join(v for k, v in BITS.items() if mask & k) or "none"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--masks", default="0,1,2,4,8,16,128,159")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default="gpurun_out/ablate.json")
    a = ap.parse_args()
    if a.build_only:
        build_abl()
        return
    os.environ.setdefault("GW_B200_LIB", os.path.join(ROOT, "build_abl", "libgwb200.so"))
    import torch

    from graph_weather_b200 import GraphWeatherForecaster

    ll = [(-90.0 + i, float(j)) for i in range(180) for j in range(360)]
    torch.manual_seed(0)
    model = GraphWeatherForecaster(ll, precision=a.precision).cuda().eval()
    x = torch.randn(a.batch, len(ll), 102, device="cuda")
    plan = None
    res = {}
    for m in [int(t) for t in a.masks.split(",")]:
        os.environ["GW_ABLATE"] = str(m)
        for _ in range(2):
            model(x)
        torch.cuda.synchronize()
        plan = model._engine.plan
        plan.timing_enable(True)
        for _ in range(a.iters):
            model(x)
        tags = plan.timing_read()
        plan.timing_enable(False)
        row = {k: round(v / a.iters, 3) for k, (c, v) in tags.items() if c}
        row["total"] = round(sum(row.values()), 3)
        res[name(m)] = row
        print(f"{m:4d} {name(m):40s}", json.dumps(row), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
