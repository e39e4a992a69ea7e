"""Per-operator device times and throughput of BASELINE configs 3 / 4 / 5 on one GPU (workloads of cleandiffuser_b200/workloads.py,
per-GPU batch).  Not the headline benchmark (bench.py = cfg2 + an other_configs block): per-operator detail.
  python scripts/bench_other_cfgs.py [cfg3 cfg4 cfg5] [--math tf32|bf16|fp32] [--reps 3] [--once]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("cfgs", nargs="*", default=["cfg3", "cfg5", "cfg4"])
ap.add_argument("--math", default="tf32")
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--once", action="store_true", help="one sample() call per config and nothing else (for profilers)")
args = ap.parse_args()
os.environ.update(CDS_BACKEND="cuda", CDS_MATH=args.math)

from cleandiffuser_b200 import workloads  # noqa: E402
from cleandiffuser_b200.engine import runtime  # noqa: E402

DEV = "cuda:0"
KINDS = {0: "conv", 1: "update", 2: "lnmod", 3: "attn", 4: "prep", 5: "cast"}


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def per_op(agent, tag):
    plan = next(iter(agent._engine_plans.values()))
    ops = plan.program.ops
    st = torch.cuda.current_stream().cuda_stream
    it = min(1, plan.n_iters - 1)
    plan.handle.profile(it, st, len(ops))
    t = plan.handle.profile(it, st, len(ops))
    tot = sum(t)
    for i, (op, ms) in enumerate(zip(ops, t)):
        d = ""
        if op.kind == 0:
            c = op.u.conv
            flops = 2.0 * c.batch * c.L_out * c.C_out * c.phases * c.taps * c.C_in
            d = (f"{('f32', 'bf16', 'tf32')[c.math]:4s} rows {c.batch} L {c.L_in}->{c.L_out * c.phases} C {c.C_in}->{c.C_out} k{c.taps} "
                 f"gn{c.groups} {flops / (ms * 1e-3) / 1e12 if ms > 0 else 0:6.0f} TF/s")
        print(f"[{tag}] op {i:2d} {KINDS[op.kind]:6s} {d:64s} {ms * 1e3:9.1f} us ({ms / tot * 100:4.1f} %)", file=sys.stderr)
    print(f"[{tag}] iteration total {tot * 1e3:.1f} us (direct launches)", file=sys.stderr)


with torch.no_grad():
    for name in args.cfgs:
        wl = workloads.BUILDERS[name](DEV)
        prior, cond = wl.prior.to(DEV), None if wl.cond is None else wl.cond.to(DEV)
        call = lambda: wl.sample(DEV, prior=prior, cond=cond)  # noqa: E731
        if args.once:
            call()
            torch.cuda.synchronize()
            continue
        ms = timed(call, args.reps)
        per_op(wl.agent, name)
        v = prior.shape[0] / (ms * 1e-3)
        print(json.dumps({"config": name, "describe": wl.describe, "math": args.math, "batch": prior.shape[0], "ms_per_sample_call": ms,
                          "trajectories_per_s": v, "tflops_effective": v * wl.gflop / 1e3,
                          "engine": dict(calls=runtime.STATS["engine_calls"], fallbacks=runtime.STATS["fallbacks"])}), flush=True)
        del wl, prior, cond
        torch.cuda.empty_cache()
