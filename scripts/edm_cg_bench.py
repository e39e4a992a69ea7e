"""Time guided ContinuousEDM and legacy DDPM sample() calls three ways, alternating within one process:

  torch     the PyTorch reverse loop (CDS_BACKEND=torch)
  callback  the engine with the classifier evaluated by a host callback between the denoiser and the update of every network
            evaluation (the same classifier wrapped in a class the lowering does not recognise)
  graph     the engine with the classifier's input gradient inside the replayed program

    python scripts/edm_cg_bench.py [--repeats 5] [--calls 3] [--out results/edm_cg_bench.json]

Calls (synthetic weights, the first step / action dimension fixed by the mask, clipped to [-1, 1]):
  edm_heun_janner   ContinuousEDM, Heun, 20 steps (39 network evaluations), w_cg 0.1: JannerUNet1d(14, model_dim 32,
                    dim_mult [1, 2, 2, 2]) at Diffuser's hopper shape (horizon 32), guided by a CumRewClassifier over
                    HalfJannerUNet1d(32, 14), batch 3200
  ddpm_mlp          legacy DDPM, x0 prediction, 20 diffusion steps, w_cg 0.5: DQLMlp(obs 11, act 3) with the observations as
                    condition, guided by an MSEClassifier over MLPNNClassifier(3, 11, 32, [256, 256]), batch 3200
A timed sample is the mean over --calls back-to-back calls.  x0 of the engine paths is compared with the PyTorch loop's under
the same noise draws.  Prints the card name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from cleandiffuser_b200.classifier import CumRewClassifier, MSEClassifier  # noqa: E402
from cleandiffuser_b200.diffusion import ContinuousEDM  # noqa: E402
from cleandiffuser_b200.diffusion.legacy import DDPM  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402
from cleandiffuser_b200.nn_classifier import HalfJannerUNet1d, MLPNNClassifier  # noqa: E402
from cleandiffuser_b200.nn_condition import IdentityCondition  # noqa: E402
from cleandiffuser_b200.nn_diffusion import DQLMlp, JannerUNet1d  # noqa: E402
from cleandiffuser_b200.testing import NoiseTape, load_synth  # noqa: E402

BATCH, STEPS = 3200, 20


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


def edm_heun_janner(dev):
    H, D = 32, 14
    mask = torch.zeros(H, D)
    mask[0] = 1.
    clf = CumRewClassifier(load_synth(HalfJannerUNet1d(H, D), seed=1), device=dev)
    agent = ContinuousEDM(load_synth(JannerUNet1d(D, model_dim=32, emb_dim=32, dim_mult=[1, 2, 2, 2]), seed=41), fix_mask=mask,
                          classifier=clf, x_max=torch.ones(H, D), x_min=-torch.ones(H, D), device=dev)
    prior = torch.zeros(BATCH, H, D, device=dev)
    prior[:, 0] = torch.randn(BATCH, D, device=dev)
    kw = dict(solver="heun", n_samples=BATCH, sample_steps=STEPS, w_cg=0.1, condition_cg=torch.zeros(BATCH, 1, device=dev))
    return agent, clf, prior, agent.sample, kw


def ddpm_mlp(dev):
    A, OBS = 3, 11
    mask = torch.zeros(A)
    mask[0] = 1.
    clf = MSEClassifier(load_synth(MLPNNClassifier(A, OBS, 32, [256, 256]), seed=1), device=dev)
    agent = DDPM(load_synth(DQLMlp(OBS, A), seed=41), IdentityCondition(dropout=0.0), fix_mask=mask, classifier=clf,
                 diffusion_steps=STEPS, predict_noise=False, x_max=torch.ones(A), x_min=-torch.ones(A), device=dev)
    prior = torch.zeros(BATCH, A, device=dev)
    obs = torch.randn(BATCH, OBS, device=dev)
    kw = dict(n_samples=BATCH, sample_steps=STEPS, w_cg=0.5, condition_cfg=obs, w_cfg=1.0, condition_cg=obs)
    return agent, clf, prior, agent.sample, kw


CALLS = {"edm_heun_janner": edm_heun_janner, "ddpm_mlp": ddpm_mlp}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("edm_cg_bench.py measures on a CUDA device; none found")
    dev = "cuda:0"
    os.environ["CDS_MATH"] = os.environ.get("CDS_MATH", "tf32")
    result = {"card": card(), "math": os.environ["CDS_MATH"], "calls_per_sample": a.calls, "calls": {}}
    print("card:", result["card"], flush=True)
    for name, make in CALLS.items():
        torch.manual_seed(0)
        agent, clf, prior, fn, kw = make(dev)
        agent.eval()
        clf.eval()
        ways = {"torch": ("torch", clf), "callback": ("cuda", Wrapped(clf)), "graph": ("cuda", clf)}
        draws = None                                            # the first call's noise, replayed by every later call
        times = {k: [] for k in ways}
        outs = {}

        def call(tape):
            with tape.active():
                return fn(prior, **kw)[0]
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
                if rep >= 2:
                    times[k].append(dt * 1e3)
                outs[k] = x0
        row = {k: {"median_ms": sorted(v)[len(v) // 2], "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}
        for k in ("callback", "graph"):
            row[k]["max_abs_dx0_vs_torch"] = float((outs[k] - outs["torch"]).abs().max())
        row["max_abs_dx0_graph_vs_callback"] = float((outs["graph"] - outs["callback"]).abs().max())
        row["batch"], row["steps"] = BATCH, STEPS
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
