"""Time guided sample() calls with a CumRewClassifier over HalfDiT1d three ways, alternating within one process:

  torch     the PyTorch reverse loop (CDS_BACKEND=torch)
  callback  the engine with the classifier evaluated by a host callback between the denoiser and the update of every step
            (the same classifier wrapped in a class the lowering does not recognise)
  graph     the engine with the classifier's input gradient inside the replayed program

    python scripts/half_dit_cg_bench.py [--repeats 5] [--calls 3] [--out results/half_dit_cg_bench.json]

Calls: DiscreteDiffusionSDE over a DiT1d planner (in_dim 14, d_model 256, 8 heads, depth 2: the shape of Decision Diffuser's
and DiffuserLite's planners), x0 prediction, the first step fixed by the mask, 20 DDPM steps, w_cg 0.1, guided by
  planner_h32 / planner_h64  HalfDiT1d(14, 1, 64, d_model 256, 8 heads, depth 2), horizon 32 / 64, batch 3200
  default_h32                HalfDiT1d(14, 1, 64) with the reference's defaults (d_model 384, 6 heads, depth 12), horizon 32,
                             batch 256
A timed sample is the mean over --calls back-to-back calls.  Synthetic weights; x0 of the engine paths is compared with the
PyTorch loop's under the same noise draws.  Prints the card name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cleandiffuser_b200.classifier import CumRewClassifier  # noqa: E402
from cleandiffuser_b200.diffusion import DiscreteDiffusionSDE  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402
from cleandiffuser_b200.nn_classifier import HalfDiT1d  # noqa: E402
from cleandiffuser_b200.nn_diffusion import DiT1d  # noqa: E402
from cleandiffuser_b200.testing import NoiseTape, load_synth  # noqa: E402

D_IN, STEPS, W_CG = 14, 20, 0.1
# name: (batch, horizon, HalfDiT1d keyword arguments)
PLANNER = dict(d_model=256, n_heads=8, depth=2)
CALLS = {"planner_h32": (3200, 32, PLANNER), "planner_h64": (3200, 64, PLANNER), "default_h32": (256, 32, {})}

class Wrapped:
    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("half_dit_cg_bench.py measures on a CUDA device; none found")
    dev = "cuda:0"
    os.environ["CDS_MATH"] = os.environ.get("CDS_MATH", "tf32")
    result = {"card": card(), "math": os.environ["CDS_MATH"], "w_cg": W_CG, "calls_per_sample": a.calls, "calls": {}}
    print("card:", result["card"], flush=True)
    for name, (batch, horizon, ckw) in CALLS.items():
        torch.manual_seed(0)
        net = load_synth(DiT1d(D_IN, emb_dim=64, **PLANNER), seed=41)
        clf = CumRewClassifier(load_synth(HalfDiT1d(D_IN, 1, 64, **ckw), seed=1), device=dev)
        mask = torch.zeros(horizon, D_IN)
        mask[0] = 1.
        agent = DiscreteDiffusionSDE(net, fix_mask=mask, classifier=clf, predict_noise=False, diffusion_steps=STEPS, device=dev)
        agent.eval()
        clf.eval()
        prior = torch.zeros(batch, horizon, D_IN, device=dev)
        prior[:, 0] = torch.randn(batch, D_IN, device=dev)
        steps = STEPS
        ways = {"torch": ("torch", clf), "callback": ("cuda", Wrapped(clf)), "graph": ("cuda", clf)}
        draws = None                                            # the first call's noise, replayed by every later call
        times = {k: [] for k in ways}
        outs, launches = {}, {}

        def call(tape):
            with tape.active():
                return agent.sample(prior, solver="ddpm", n_samples=batch, sample_steps=steps, w_cg=W_CG)[0]
        for rep in range(a.repeats + 2):                       # two warm-up rounds, then alternating timed rounds
            for k, (backend, c) in ways.items():
                os.environ["CDS_BACKEND"] = backend
                agent.classifier = c
                if draws is None:
                    tape = NoiseTape()
                    outs[k] = call(tape)
                    draws = [z.clone() for z in tape.draws]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.calls):
                    x0 = call(NoiseTape(draws))
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) / a.calls
                if k != "torch":
                    assert runtime.STATS["guidance_path"] == k, (k, runtime.STATS["guidance_path"])
                    launches[k] = runtime.STATS["launches"]
                if rep >= 2:
                    times[k].append(dt * 1e3)
                outs[k] = x0
        row = {k: {"median_ms": sorted(v)[len(v) // 2], "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}
        for k in ("callback", "graph"):
            row[k]["max_abs_dx0_vs_torch"] = float((outs[k] - outs["torch"]).abs().max())
            # engine launches per reverse iteration (the callback's PyTorch forward / backward kernels come on top)
            row[k]["engine_launches_per_iter"] = round((launches[k] - 1) / steps, 2)
        row["max_abs_dx0_graph_vs_callback"] = float((outs["graph"] - outs["callback"]).abs().max())
        row["batch"], row["steps"], row["horizon"], row["classifier"] = batch, steps, horizon, dict(dict(d_model=384, n_heads=6,
                                                                                                         depth=12), **ckw)
        row["graph_speedup_vs_callback"] = row["callback"]["median_ms"] / row["graph"]["median_ms"]
        row["graph_speedup_vs_torch"] = row["torch"]["median_ms"] / row["graph"]["median_ms"]
        result["calls"][name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
