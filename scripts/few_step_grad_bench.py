"""Time one few-step actor step -- ``sample(requires_grad=True)`` + ``backward()`` over DQLMlp (obs 17, act 6, actions clipped
to [-1, 1]) -- on the engine against the PyTorch loop, for the samplers consistency and flow policies differentiate through:
ContinuousConsistencyModel at 1 and 2 steps (CPQL, Consistency-AC) and ContinuousRectifiedFlow at 5 Euler steps.  CUDA
events, warm-up and alternating windows (engine, torch, engine, ...) as in scripts/dql_grad_bench.py.  Prints one JSON line per
(sampler, batch, math mode) with the card's name and power limit, the median / min / max per-step time of each back end, and
the engine's launches per iteration of the forward and backward programs.

    python scripts/few_step_grad_bench.py [--batches 256 4096] [--windows 5] [--iters 20] [--math tf32 fp32]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from cleandiffuser_b200.diffusion import ContinuousConsistencyModel, ContinuousRectifiedFlow  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402
from cleandiffuser_b200.nn_condition import IdentityCondition  # noqa: E402
from cleandiffuser_b200.nn_diffusion import DQLMlp  # noqa: E402
from cleandiffuser_b200.testing import load_synth  # noqa: E402
from dql_grad_bench import card  # noqa: E402

SAMPLERS = {"consistency-1": (ContinuousConsistencyModel, 1), "consistency-2": (ContinuousConsistencyModel, 2),
            "rectified_flow-5": (ContinuousRectifiedFlow, 5)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samplers", nargs="+", default=list(SAMPLERS), choices=list(SAMPLERS))
    ap.add_argument("--batches", type=int, nargs="+", default=[256, 4096])
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--math", nargs="+", default=["tf32", "fp32"])
    ap.add_argument("--obs", type=int, default=17)
    ap.add_argument("--act", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "few_step_grad_bench.py measures on a CUDA device"
    dev = "cuda:0"
    name, power = card()
    for sampler in args.samplers:
        cls, steps = SAMPLERS[sampler]
        for math_mode in args.math:
            os.environ["CDS_MATH"] = math_mode
            for B in args.batches:
                net = load_synth(DQLMlp(args.obs, args.act, emb_dim=16), seed=0).to(dev)
                a = args.act
                agent = cls(net, IdentityCondition(dropout=0.0), x_max=torch.ones(1, a), x_min=-torch.ones(1, a), device=dev)
                g = torch.Generator(device=dev).manual_seed(0)
                obs = torch.randn(B, args.obs, device=dev, generator=g)
                w = torch.randn(B, a, device=dev, generator=g)
                prior = torch.zeros(B, a, device=dev)

                def step():
                    x0, _ = agent.sample(prior, n_samples=B, sample_steps=steps, use_ema=False, condition_cfg=obs, w_cfg=1.0,
                                         requires_grad=True)
                    (x0 * w).sum().backward()

                def window(backend, n):
                    os.environ["CDS_BACKEND"] = backend
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(n):
                        step()
                    e1.record()
                    torch.cuda.synchronize()
                    return e0.elapsed_time(e1) / n

                times = {"cuda": [], "torch": []}
                for backend in times:                 # warm-up: plan build, graph capture, cuBLAS algorithm choice
                    window(backend, 3)
                calls = runtime.STATS["engine_calls"]
                for _ in range(args.windows):
                    for backend in times:
                        times[backend].append(window(backend, args.iters))
                assert runtime.STATS["engine_calls"] == calls + args.windows * args.iters, "the engine did not serve every step"
                plan = [p for p in agent._engine_plans.values() if isinstance(p, runtime.GradSamplerPlan)][0]
                med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
                print(json.dumps({
                    "card": name, "power_limit": power, "sampler": sampler, "math": math_mode, "batch": B,
                    "network_evaluations": plan.n_iters, "obs_dim": args.obs, "act_dim": a,
                    "engine_ms_median": round(med["cuda"], 4), "engine_ms_min": round(min(times["cuda"]), 4),
                    "engine_ms_max": round(max(times["cuda"]), 4),
                    "torch_ms_median": round(med["torch"], 4), "torch_ms_min": round(min(times["torch"]), 4),
                    "torch_ms_max": round(max(times["torch"]), 4),
                    "speedup_median": round(med["torch"] / med["cuda"], 3),
                    "forward_launches_per_iter": plan.handle.launches_per_iter(),
                    "backward_launches_per_iter": plan.back_handle.launches_per_iter(),
                    "windows": args.windows, "steps_per_window": args.iters}), flush=True)
                agent._engine_plans.clear()


if __name__ == "__main__":
    main()
