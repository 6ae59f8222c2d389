"""-m gpu: a plan gives back its device memory when it is closed.  Ten plans of each kind are created, used and closed through
`_capi.Plan.close()`: a 1-degree inference plan at batch 8, a taped training plan after one bf16 step, and a bounded
(use_checkpointing=True) training plan closed while two multi_step() tapes are alive, which leaves those tapes dead.  A create
that runs out of device memory after its first allocations succeeded raises the allocation's error and keeps nothing, and the
next plan runs.  After a warm-up, the free device memory comes back to its starting value within one plan's device_bytes(): a
leaked plan or training state would be ten of them."""
import gc

import pytest
import torch

import __graft_entry__ as ge
from training_oracle import grid

pytestmark = pytest.mark.gpu

OOM = r"^libgwb200: cudaMalloc\(\d+ B\): out of memory$"


@pytest.fixture(scope="module", autouse=True)
def _built():
    ge.build()


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def _close(engine):
    """Closes the engine's plan; its next forward makes a new one.  Returns the closed plan's device_bytes()."""
    size = engine.plan.device_bytes()
    engine.plan.close()
    engine.plan = None
    return size


def _inference_cycle():
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(0)
    model = GraphWeatherForecaster(grid(1)).cuda().eval()
    x = torch.randn(8, len(grid(1)), 102, device="cuda")

    def cycle():
        with torch.no_grad():
            model(x)
        return _close(model._engine)

    return model, cycle


def _taped_cycle():
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(0)
    model = GraphWeatherForecaster(grid(5), train_precision="bf16").cuda().train()
    x = torch.randn(1, len(grid(5)), 102, device="cuda")

    def cycle():
        model(x).square().mean().backward()
        return _close(model._train_engine)

    return model, cycle


def _bounded_cycle():
    from graph_weather_b200 import GraphWeatherForecaster

    torch.manual_seed(0)
    model = GraphWeatherForecaster(grid(5), train_precision="bf16", use_checkpointing=True).cuda().train()
    x = torch.randn(1, len(grid(5)), 102, device="cuda")

    def cycle():
        with model.multi_step():
            ys = [model(x), model(x)]
        tapes = [y.grad_fn.tape for y in ys]
        assert model._train_engine.plan.train_only and all(t.bytes() > 0 for t in tapes)
        size = _close(model._train_engine)
        assert all(t.bytes() == 0 and not t.plan.handle.value for t in tapes)  # dead: their memory went with the plan
        return size

    return model, cycle


@pytest.mark.training
@pytest.mark.parametrize("make", [_inference_cycle, _taped_cycle, _bounded_cycle], ids=["inference", "taped", "bounded"])
def test_closed_plans_give_their_memory_back(make):
    model, cycle = make()
    cycle()  # warm-up: module loads, and the first allocations of torch's and the tapes' stream-ordered pools
    start = _free()
    sizes = [cycle() for _ in range(10)]
    end = _free()
    print(f"free before {start / 2**20:.0f} MiB, after ten plans {end / 2**20:.0f} MiB; plan {sizes[-1] / 2**20:.0f} MiB")
    assert start - end <= sizes[-1]


def test_a_create_that_runs_out_of_memory_keeps_nothing():
    from graph_weather_b200 import _capi

    model, cycle = _inference_cycle()
    size = cycle()
    # 2**16 samples: the batch-sized scratch (xbuf0 alone is 394 GB) fails after the graphs and the chunk-sized scratch were allocated
    dims = dict(model._engine.dims, max_batch=1 << 16, precision=_capi.PRECISIONS["fp32"])
    start = _free()
    with pytest.raises(RuntimeError, match=OOM) as err:
        _capi.Plan("cuda", **dims)
    end = _free()
    print(f"{err.value}; free before {start / 2**20:.0f} MiB, after {end / 2**20:.0f} MiB")
    assert start - end <= size
    cycle()  # a plan made after the failed one runs: the allocation's error was reported once, by the create
