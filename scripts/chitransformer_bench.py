"""sample() time of the ChiTransformer pipelines on the engine and on the PyTorch loop, on one GPU.

    python scripts/chitransformer_bench.py [--steps 50] [--reps 5]

For each Diffusion Policy ChiTransformer shape (tests/golden/chi_cases.py: pusht / robomimic image, robomimic low-dim,
kitchen) at batch 1 and 2048: the legacy DDPM agent the dp_* pipelines build (identity condition, w_cfg = 1, actions clipped
to [-1, 1]), a `steps`-step sample(), timed with a host clock around the call and a device synchronise, median of `reps`
calls after two warm-up calls, once with CDS_BACKEND=cuda (the engine) and once with CDS_BACKEND=torch (the PyTorch loop) on
the same GPU.  Prints the card's name and power limit, one JSON line per measurement and a markdown table."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import torch  # noqa: E402

import chi_cases as cc  # noqa: E402
from cleandiffuser_b200.diffusion import DDPM  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402
from cleandiffuser_b200.nn_condition import IdentityCondition  # noqa: E402
from cleandiffuser_b200.nn_diffusion import ChiTransformer  # noqa: E402
from cleandiffuser_b200.testing import synth_state_dict  # noqa: E402

SHAPES = ["pusht", "robomimic", "kitchen"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the timing below still runs; the card line says why it is missing
        q = f"nvidia-smi unavailable ({e})"
    return torch.cuda.get_device_name(0), q


def time_calls(agent, prior, cond, steps, reps, backend):
    os.environ["CDS_BACKEND"] = backend
    kw = dict(n_samples=prior.shape[0], sample_steps=steps, condition_cfg=cond, w_cfg=1.0, use_ema=True)
    times = []
    with torch.no_grad():
        for r in range(reps + 2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            agent.sample(prior, **kw)
            torch.cuda.synchronize()
            if r >= 2:
                times.append(time.perf_counter() - t0)
    return sorted(times)[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="1,2048")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    name, smi = card()
    print(f"# device: {name} | nvidia-smi name, power.limit: {smi} | CDS_MATH={os.environ.get('CDS_MATH', 'tf32')}", flush=True)
    rows = []
    for shape in SHAPES:
        ctor = cc.NETS[shape]
        net = ChiTransformer(**ctor)
        net.load_state_dict(cc.weights(net.state_dict(), synth_state_dict))
        net = net.eval().to("cuda")
        x_max = torch.ones((1, ctor["Ta"], ctor["act_dim"]), device="cuda")
        agent = DDPM(net, IdentityCondition(dropout=0.0), x_max=x_max, x_min=-x_max, diffusion_steps=args.steps, device="cuda")
        agent.model_ema.eval()
        for B in (int(b) for b in args.batches.split(",")):
            g = torch.Generator().manual_seed(B)
            prior = torch.zeros(B, ctor["Ta"], ctor["act_dim"], device="cuda")
            cond = torch.randn(B, ctor["To"], ctor["obs_dim"], generator=g).to("cuda")
            calls, falls = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
            t_eng = time_calls(agent, prior, cond, args.steps, args.reps, "cuda")
            assert runtime.STATS["engine_calls"] == calls + args.reps + 2 and runtime.STATS["fallbacks"] == falls
            t_pt = time_calls(agent, prior, cond, args.steps, args.reps, "torch")
            rec = dict(shape=shape, d_model=ctor["d_model"], layers=ctor["num_layers"], batch=B, steps=args.steps,
                       engine_ms=round(1e3 * t_eng, 3), torch_ms=round(1e3 * t_pt, 3),
                       engine_traj_per_s=round(B / t_eng, 1), torch_traj_per_s=round(B / t_pt, 1),
                       speedup=round(t_pt / t_eng, 2))
            rows.append(rec)
            print(json.dumps(rec), flush=True)
    print()
    print("| shape | d_model x layers | batch | engine ms | engine traj/s | PyTorch ms | PyTorch traj/s | speed-up |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['d_model']} x {r['layers']} | {r['batch']} | {r['engine_ms']:.2f} | {r['engine_traj_per_s']:.0f} "
              f"| {r['torch_ms']:.2f} | {r['torch_traj_per_s']:.0f} | {r['speedup']:.2f} |")


if __name__ == "__main__":
    main()
