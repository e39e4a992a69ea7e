"""Time guided sample() calls with an MLPNNClassifier three ways, alternating within one process:

  torch     the PyTorch reverse loop (CDS_BACKEND=torch)
  callback  the engine with the classifier evaluated by a host callback between the denoiser and the update of every step
            (the same classifier wrapped in a class the lowering does not recognise)
  graph     the engine with the classifier's input gradient inside the replayed program

    python scripts/mlp_cg_bench.py [--repeats 15] [--calls 20] [--out results/mlp_cg_bench.json]

Calls:
  tutorial  the reference's classifier-guidance tutorial (tutorials/3_classifier_guidance.py) at kitchen's shapes:
            DiscreteDiffusionSDE over PearceMlp(9, To=0, emb_dim=64, hidden_dim=256), x0 prediction clipped to [-1, 1],
            MSEClassifier over MLPNNClassifier(9, 60, 32, [256], SiLU), batch 50, 5 DDPM steps, temperature 0.5, w_cg 0.1
  large     the same actor guided by MSEClassifier over MLPNNClassifier(9, 60, 32, [256, 256]) with its default ReLU,
            batch 4096, 10 DDPM steps (diffusion_steps 10), w_cg 0.1
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

from cleandiffuser_b200.classifier import MSEClassifier  # noqa: E402
from cleandiffuser_b200.diffusion import DiscreteDiffusionSDE  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402
from cleandiffuser_b200.nn_classifier import MLPNNClassifier  # noqa: E402
from cleandiffuser_b200.nn_diffusion import PearceMlp  # noqa: E402
from cleandiffuser_b200.testing import NoiseTape, load_synth  # noqa: E402

ACT, OBS = 9, 60
# name: (batch, steps, hidden dims, activation)
CALLS = {"tutorial": (50, 5, [256], torch.nn.SiLU), "large": (4096, 10, [256, 256], torch.nn.ReLU)}
W_CG = 0.1


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
        raise SystemExit("mlp_cg_bench.py measures on a CUDA device; none found")
    dev = "cuda:0"
    os.environ["CDS_MATH"] = os.environ.get("CDS_MATH", "tf32")
    result = {"card": card(), "math": os.environ["CDS_MATH"], "w_cg": W_CG, "calls_per_sample": a.calls, "calls": {}}
    print("card:", result["card"], flush=True)
    for name, (batch, steps, hidden, act) in CALLS.items():
        net = load_synth(PearceMlp(ACT, To=0, emb_dim=64, hidden_dim=256, timestep_emb_type="positional"), seed=41)
        clf = MSEClassifier(load_synth(MLPNNClassifier(ACT, OBS, 32, hidden, activation=act()), seed=1), temperature=1.0,
                            device=dev)
        agent = DiscreteDiffusionSDE(net, classifier=clf, predict_noise=False, x_max=torch.ones((1, ACT)),
                                     x_min=-torch.ones((1, ACT)), diffusion_steps=steps, device=dev)
        agent.eval()
        clf.eval()
        obs = torch.randn(batch, OBS, device=dev)
        prior = torch.zeros(batch, ACT, device=dev)
        ways = {"torch": ("torch", clf), "callback": ("cuda", Wrapped(clf)), "graph": ("cuda", clf)}
        draws = None                                            # the first call's noise, replayed by every later call
        times = {k: [] for k in ways}
        outs, launches = {}, {}

        def call(tape):
            with tape.active():
                return agent.sample(prior, solver="ddpm", n_samples=batch, sample_steps=steps, temperature=0.5, w_cg=W_CG,
                                    condition_cg=obs)[0]
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
        row["batch"], row["steps"], row["hidden"], row["activation"] = batch, steps, hidden, act.__name__
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
