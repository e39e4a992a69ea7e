"""Time one QGPO-guided sample() (QGPOClassifier over QGPONNClassifier(obs, act, 64, [256, 256, 256]), ContinuousDiffusionSDE
over SfBCUNet with MLPCondition, "ddpm" on "quad_continuous" steps, w_cfg = 1, condition_cg = obs, w_cg = 3, clip to [-1, 1]:
QGPO's D4RL MuJoCo inference call) three ways, alternating within one process:

  torch     the PyTorch reverse loop (CDS_BACKEND=torch)
  callback  the engine with the classifier evaluated by a host callback between the denoiser and the update of every step
            (the same classifier wrapped in a class the lowering does not recognise)
  graph     the engine with the classifier's input gradient inside the replayed program

    python scripts/qgpo_bench.py [--repeats 15] [--calls 20] [--out results/qgpo_bench.json]

Shapes: halfcheetah (obs 17, act 6) at batch 50 x 5 steps, hopper-medium-replay (obs 11, act 3) at 800 x 10 steps (50 envs x
16 candidates), and hopper at 5000 x 10 steps.  A timed sample is the mean over --calls back-to-back calls (one call of the
small shapes takes milliseconds).  Synthetic weights; x0 of the engine paths is compared with the PyTorch loop's under the
same noise draws.  Prints the card name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cleandiffuser_b200.classifier import QGPOClassifier  # noqa: E402
from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402
from cleandiffuser_b200.nn_classifier import QGPONNClassifier  # noqa: E402
from cleandiffuser_b200.nn_condition import MLPCondition  # noqa: E402
from cleandiffuser_b200.nn_diffusion import SfBCUNet  # noqa: E402
from cleandiffuser_b200.testing import NoiseTape, load_synth  # noqa: E402

SHAPES = {"halfcheetah": (17, 6, 50, 5), "hopper-medium-replay": (11, 3, 800, 10), "hopper-5000": (11, 3, 5000, 10)}
W_CG = 3.0


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
    ap.add_argument("--repeats", type=int, default=15)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qgpo_bench.py measures on a CUDA device; none found")
    dev = "cuda:0"
    os.environ["CDS_MATH"] = os.environ.get("CDS_MATH", "tf32")
    result = {"card": card(), "math": os.environ["CDS_MATH"], "w_cg": W_CG, "calls_per_sample": a.calls, "shapes": {}}
    print("card:", result["card"], flush=True)
    for name, (obs_dim, act_dim, batch, steps) in SHAPES.items():
        net = load_synth(SfBCUNet(act_dim), seed=41)
        cond = load_synth(MLPCondition(obs_dim, 64, [64], torch.nn.SiLU()), seed=42)
        clf = QGPOClassifier(load_synth(QGPONNClassifier(obs_dim, act_dim, 64, [256, 256, 256], "untrainable_fourier"), seed=1),
                             device=dev)
        agent = ContinuousDiffusionSDE(net, cond, x_max=torch.ones(act_dim), x_min=-torch.ones(act_dim), device=dev)
        agent.eval()
        obs = torch.randn(batch, obs_dim, device=dev)
        prior = torch.zeros(batch, act_dim, device=dev)
        ways = {"torch": ("torch", clf), "callback": ("cuda", Wrapped(clf)), "graph": ("cuda", clf)}
        draws = None                                            # the first call's noise, replayed by every later call
        times = {k: [] for k in ways}
        outs, launches = {}, {}

        def call(tape):
            with tape.active():
                return agent.sample(prior, "ddpm", n_samples=batch, sample_steps=steps, sample_step_schedule="quad_continuous",
                                    condition_cfg=obs, w_cfg=1.0, condition_cg=obs, w_cg=W_CG)[0]
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
        row["batch"], row["steps"], row["obs_dim"], row["act_dim"] = batch, steps, obs_dim, act_dim
        row["graph_speedup_vs_callback"] = row["callback"]["median_ms"] / row["graph"]["median_ms"]
        result["shapes"][name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
