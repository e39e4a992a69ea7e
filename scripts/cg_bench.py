"""Time one classifier-guided sample() (CumRewClassifier over HalfJannerUNet1d, JannerUNet1d denoiser, 20 DDPM steps,
w_cg = 0.3, the Diffuser pipelines' call) three ways, alternating within one process:

  torch     the PyTorch reverse loop (CDS_BACKEND=torch)
  callback  the engine with the classifier evaluated by a host callback between the denoiser and the update of every step
            (the same classifier wrapped in a class the lowering does not recognise)
  graph     the engine with the classifier's input gradient inside the replayed program

    python scripts/cg_bench.py [--repeats 5] [--out results/cg_bench.json]

Shapes: hopper (horizon 32, obs + act 14) and antmaze (horizon 64, 37), batch 3200.  Synthetic weights; x0 of the engine
paths is compared with the PyTorch loop's under the same noise draws.  Prints the card name and power limit with the numbers."""
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
from cleandiffuser_b200.nn_classifier import HalfJannerUNet1d  # noqa: E402
from cleandiffuser_b200.nn_diffusion import JannerUNet1d  # noqa: E402
from cleandiffuser_b200.testing import NoiseTape, load_synth  # noqa: E402

SHAPES = {"hopper": (32, 14, 11), "antmaze": (64, 37, 29)}       # horizon, obs + act, obs


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
    ap.add_argument("--batch", type=int, default=3200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cg_bench.py measures on a CUDA device; none found")
    dev = "cuda:0"
    os.environ["CDS_MATH"] = os.environ.get("CDS_MATH", "tf32")
    result = {"card": card(), "batch": a.batch, "steps": 20, "math": os.environ["CDS_MATH"], "shapes": {}}
    for name, (H, D, obs) in SHAPES.items():
        net = load_synth(JannerUNet1d(D, model_dim=32, emb_dim=32, kernel_size=5, dim_mult=[1, 2, 2, 2]), seed=0)
        clf = CumRewClassifier(load_synth(HalfJannerUNet1d(H, D), seed=1), device=dev)
        mask = torch.zeros(H, D)
        mask[0, :obs] = 1.
        agent = DiscreteDiffusionSDE(net, None, fix_mask=mask, predict_noise=True, diffusion_steps=20, device=dev, classifier=clf)
        prior = torch.zeros(a.batch, H, D, device=dev)
        prior[:, 0, :obs] = torch.randn(a.batch, obs, device=dev)
        ways = {"torch": ("torch", clf), "callback": ("cuda", Wrapped(clf)), "graph": ("cuda", clf)}
        draws = None                                            # the first call's noise, replayed by every later call
        times = {k: [] for k in ways}
        outs = {}
        for rep in range(a.repeats + 2):                       # two warm-up rounds, then alternating timed rounds
            for k, (backend, c) in ways.items():
                os.environ["CDS_BACKEND"] = backend
                agent.classifier = c
                tape = NoiseTape(draws) if draws is not None else NoiseTape()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with tape.active():
                    x0, _ = agent.sample(prior, solver="ddpm", n_samples=a.batch, sample_steps=20, use_ema=True,
                                         temperature=0.5, w_cg=0.3)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if draws is None:
                    draws = [z.clone() for z in tape.draws]
                if k != "torch":
                    assert runtime.STATS["guidance_path"] == k, (k, runtime.STATS["guidance_path"])
                if rep >= 2:
                    times[k].append(dt * 1e3)
                outs[k] = x0
        row = {k: {"median_ms": sorted(v)[len(v) // 2], "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}
        for k in ("callback", "graph"):
            row[k]["max_abs_dx0_vs_torch"] = float((outs[k] - outs["torch"]).abs().max())
        row["graph_launches_per_call"] = runtime.STATS["launches"]
        result["shapes"][name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
