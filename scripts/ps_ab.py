"""A/B of two builds of libcds on the flagship workload: bit-identity and speed of the conv_ps operators.

    python scripts/ps_ab.py --base DIR [--out OUT] [--windows 5] [--bench-runs 3]

DIR is another checkout of this repository (for instance the parent commit, from ``git worktree add``) whose extension
has been built with ``__graft_entry__.build()``; the other build is this tree.  Every measurement runs each build in a
process of its own, so that each one loads only its own libcds.so.

1. Every ``ps_*`` case of tests/conv_cases.py on the same seeded operands: the output buffers must be equal bit for bit.
2. The per-operator device times of one cfg2 reverse iteration (``cds_plan_profile``: event-bracketed direct launches,
   the same numbers bench.py logs as ``op NN conv ...``), in ``--windows`` windows that alternate the two builds; each
   window is the mean of 20 profiles.  Reported per operator as median (min..max) over the windows.
3. ``bench.py --steps 5 --warmup 3 --no-cpu-baseline --no-eager-baseline --dump-outputs`` ``--bench-runs`` times per
   build, alternating: the headline values, the other configurations', and x0.npy.  The runs of one build must be
   byte-identical; between the builds the largest difference is reported (a change of kernel for an operator sums in
   another order).

The operators are matched by shape; the kernel family each build picks is reported beside them.  Writes OUT/ps_ab.json
and prints a summary; exits 1 if a ps_* case differs or a build's x0.npy differs between its runs.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILE_REPS = 20


# ------------------------------------------------------------------------------------------------ workers (one build each)
def _import_root(root):
    sys.path[:0] = [root, os.path.join(root, "tests")]


def worker_cases(root, out):
    """run every ps_* case once at iteration 1 and save the raw bytes of each output buffer"""
    _import_root(root)
    import numpy as np
    import torch
    import conv_cases as cc
    from cleandiffuser_b200.engine import cabi
    assert os.path.realpath(cabi.lib_path()).startswith(os.path.realpath(root)), cabi.lib_path()
    res = {}
    for name, c in cc.CASES.items():
        if c["want"][0] != "ps":
            continue
        d = cc.make(c, "cuda:0")
        op = cc.descriptor(c, d)
        assert cc.choice_key(cabi.conv_choice(op.u.conv)) == c["want"], name
        cabi.run_op(0, op, 1, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        res[name] = d["buf/out"].cpu().contiguous().view(torch.uint8).numpy().ravel()
    np.savez(out, **res)


def worker_profile(root):
    """build cfg2's plan, then answer 'profile' lines on stdin with the per-operator times (ms) of one iteration"""
    _import_root(root)
    import torch
    import bench
    from cleandiffuser_b200.engine import cabi
    assert os.path.realpath(cabi.lib_path()).startswith(os.path.realpath(root)), cabi.lib_path()
    os.environ["CDS_BACKEND"] = "cuda"
    torch.cuda.set_device(0)
    with torch.no_grad():
        agent, _, _ = bench.build_agent("cuda:0")
        prior = bench.make_prior(bench.BATCH, seed=1).to("cuda:0")
        torch.manual_seed(2)
        agent.sample(prior, solver="ddpm", n_samples=bench.BATCH, sample_steps=bench.S_STEPS, temperature=0.5)
        torch.cuda.synchronize()
        plan = next(iter(agent._engine_plans.values()))
        ops = plan.program.ops
        g = torch.Generator(device="cuda:0").manual_seed(3)
        plan.x.copy_(torch.randn(plan.x.shape, generator=g, device="cuda:0") * 0.5)
        stream = torch.cuda.current_stream().cuda_stream
        plan.handle.profile(50, stream, len(ops))
        desc, fams = [], []
        for op in ops:
            if op.kind == 0:
                c = op.u.conv
                desc.append(f"conv L{c.L_in}->{c.L_out * c.phases} C{c.C_in}->{c.C_out} k{c.taps}"
                            f"{' resW' if c.res_w else ''}")
                fams.append(cabi.conv_choice(c)["family"])
            else:
                desc.append(f"kind {op.kind}")
                fams.append("")
        print(json.dumps({"ready": True, "ops": desc, "families": fams}), flush=True)
        for line in sys.stdin:
            if line.strip() != "profile":
                break
            per_op = [0.0] * len(ops)
            for _ in range(PROFILE_REPS):
                for i, v in enumerate(plan.handle.profile(50, stream, len(ops))):
                    per_op[i] += v / PROFILE_REPS
            print(json.dumps(per_op), flush=True)


# ------------------------------------------------------------------------------------------------ driver
def _gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def compare_cases(roots, out):
    import numpy as np
    files = {}
    for tag, root in roots.items():
        files[tag] = os.path.join(out, f"ps_cases_{tag}.npz")
        subprocess.run([sys.executable, __file__, "--worker", "cases", "--root", root, "--dump", files[tag]], check=True)
    a, b = np.load(files["base"]), np.load(files["new"])
    diff = sorted(k for k in a.files if k not in b.files or not np.array_equal(a[k], b[k]))
    return {"cases": sorted(a.files), "differ": diff}


def profile_windows(roots, windows):
    procs, ops, fams = {}, None, {}
    for tag, root in roots.items():
        procs[tag] = subprocess.Popen([sys.executable, __file__, "--worker", "profile", "--root", root],
                                      stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        hello = json.loads(procs[tag].stdout.readline())
        assert ops is None or ops == hello["ops"], "the two builds lowered different programs"
        ops = hello["ops"]
        fams[tag] = hello["families"]
    times = {tag: [] for tag in roots}
    try:
        for _ in range(windows):
            for tag, p in procs.items():
                p.stdin.write("profile\n")
                p.stdin.flush()
                times[tag].append(json.loads(p.stdout.readline()))
    finally:
        for p in procs.values():
            p.stdin.close()
            p.wait()
    rows = []
    for i, name in enumerate(ops):
        row = {"op": i, "what": name}
        for tag in roots:
            us = [w[i] * 1e3 for w in times[tag]]
            row[tag] = {"median_us": statistics.median(us), "min_us": min(us), "max_us": max(us), "family": fams[tag][i]}
        rows.append(row)
    totals = {tag: [sum(w) * 1e3 for w in times[tag]] for tag in roots}
    return rows, totals


def bench_runs(roots, runs, out, tmp):
    import numpy as np
    res = {tag: [] for tag in roots}
    x0 = {}
    for r in range(runs):
        for tag, root in roots.items():
            dump = os.path.join(tmp, f"x0_{tag}_{r}")
            p = subprocess.run([sys.executable, "bench.py", "--steps", "5", "--warmup", "3", "--no-cpu-baseline",
                                "--no-eager-baseline", "--dump-outputs", dump], cwd=root, capture_output=True, text=True)
            with open(os.path.join(out, f"bench_{tag}_{r}.log"), "w") as f:
                f.write(p.stderr)
            if p.returncode != 0:
                raise RuntimeError(f"bench.py failed for {tag}:\n{p.stderr[-3000:]}")
            line = json.loads(p.stdout.strip().splitlines()[-1])
            others = {k: v.get("value") for k, v in (line.get("other_configs") or {}).items() if isinstance(v, dict)}
            res[tag].append({"value": line["value"], "ms_per_step": line["ms_per_step"], "other_configs": others,
                             "clocks": line.get("clocks")})
            x0[(tag, r)] = open(os.path.join(dump, "x0.npy"), "rb").read()
    nondet = sorted(f"{t}/{r}" for (t, r), v in x0.items() if v != x0[(t, 0)])
    load = lambda t: np.load(os.path.join(tmp, f"x0_{t}_0", "x0.npy")).astype(np.float64)
    base, new = load("base"), load("new")
    diff = {"max_abs": float(np.abs(new - base).max()), "max_abs_base": float(np.abs(base).max()),
            "max_rel": float((np.abs(new - base) / np.maximum(np.abs(base), 1e-30)).max()),
            "elements_differ": int((new != base).sum()), "elements": int(base.size)}
    return res, nondet, diff


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--base", help="the other checkout (built)")
    ap.add_argument("--out", default="ps_ab_out")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--bench-runs", type=int, default=3)
    ap.add_argument("--worker", choices=["cases", "profile"], help=argparse.SUPPRESS)
    ap.add_argument("--root", help=argparse.SUPPRESS)
    ap.add_argument("--dump", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker == "cases":
        return worker_cases(args.root, args.dump)
    if args.worker == "profile":
        return worker_profile(args.root)
    if not args.base:
        ap.error("--base is required")
    roots = {"base": os.path.abspath(args.base), "new": HERE}
    args.out = os.path.abspath(args.out)
    os.makedirs(args.out, exist_ok=True)
    report = {"gpu_before": _gpu_info(), "roots": roots}
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        report["cases"] = compare_cases(roots, tmp)
    print(f"ps cases: {len(report['cases']['cases'])} compared, differ: {report['cases']['differ']}", flush=True)
    rows, totals = profile_windows(roots, args.windows)
    report["per_op"], report["iteration_total_us"] = rows, totals
    for row in rows:
        if "conv" in row["what"]:
            b, n = row["base"], row["new"]
            print(f"op {row['op']:2d} {row['what']:34s} base {b['family']:2s} {b['median_us']:7.1f} ({b['min_us']:.1f}..{b['max_us']:.1f})"
                  f"  new {n['family']:2s} {n['median_us']:7.1f} ({n['min_us']:.1f}..{n['max_us']:.1f}) us", flush=True)
    for tag, t in totals.items():
        print(f"iteration total {tag}: median {statistics.median(t):.1f} ({min(t):.1f}..{max(t):.1f}) us", flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        report["bench"], report["x0_nondeterministic"], report["x0_base_vs_new"] = bench_runs(roots, args.bench_runs, args.out, tmp)
    for tag, runs in report["bench"].items():
        print(f"bench {tag}: " + ", ".join(f"{r['value']:.0f}" for r in runs) + " traj/s; other configs "
              + "; ".join(json.dumps(r["other_configs"]) for r in runs), flush=True)
    print(f"x0.npy differs from its own build's run 0: {report['x0_nondeterministic']}", flush=True)
    print(f"x0.npy, new vs base: {json.dumps(report['x0_base_vs_new'])}", flush=True)
    report["gpu_after"] = _gpu_info()
    print("gpu:", report["gpu_before"], "/", report["gpu_after"], flush=True)
    with open(os.path.join(args.out, "ps_ab.json"), "w") as f:
        json.dump(report, f, indent=1)
    return 1 if report["cases"]["differ"] or report["x0_nondeterministic"] else 0


if __name__ == "__main__":
    sys.exit(main() or 0)
