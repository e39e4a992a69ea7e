"""Audit of the programs bench.py measures, at the batch each is benchmarked with (tests/program_audit.py does the work).

Programs: cfg2 (fp32, tf32, bf16), cfg3 / cfg4 / cfg5 (tf32, bf16) from cleandiffuser_b200/workloads.py, and the
ChiTransformer kitchen shape (tests/golden/chi_cases.py) at batch 2048 as scripts/chitransformer_bench.py builds it (tf32,
bf16).  "dit256" adds cfg4 with a DiT1d of d_model 256 over x_t of 96 channels: the only audited program with 256-wide
gated Linears (attention out-projection, second MLP Linear) and a 256-wide x_proj that reads x_t shared by the two CFG
halves (in_batch_mod), i.e. conv_tc's gated and table epilogue lanes, each followed by a LayerNorm, at a width other than
cfg4's 320.  "cg_<shape>" is scripts/cg_bench.py's classifier-guided call with the classifier of a reference pipeline
(cg_ref.PIPELINES).  Each is built by one ``sample()``, so that the plan, its tables and its per-call fills are what
production builds; its handle is then driven directly.  The differentiable programs of sample(requires_grad=True) over
DQLMlp (grad_ref.GRAD_CASES) have their own test: all 5 forward and all 5 backward iterations.

- Every operator of iterations 0, 1, the middle one (loops of 50 steps or more) and the last, reached by graph replay, is
  run alone and checked on every trajectory against fp64 under its kernel family's bound, and for writes outside its
  outputs; one iteration is one launch per operator, plus the iteration-counter advance.
- ``min(12, n_iters - f)`` whole iterations from a snapshot at iteration f give the same bits operator by operator (with a
  synchronisation after each: no launch overlaps another), by graph replay (the 10-iteration graph plus single graphs)
  and by direct launches.
- Parallel branches (CDS_BRANCHES) at full size give the bits of the single-branch operator-by-operator run.

The module prints the largest error as a fraction of the bound per (program, kernel instantiation), the wall time and the
peak device memory each audit adds to its program."""
import math
import time

import pytest
import torch

import cg_ref
import chi_cases as cc
import emulator
import grad_ref
import program_audit as pa
from cleandiffuser_b200 import workloads
from cleandiffuser_b200.diffusion import DDPM
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import ChiTransformer
from cleandiffuser_b200.testing import load_synth, synth_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PROGRAMS = ["cfg2-fp32", "cfg2-tf32", "cfg2-bf16", "cfg3-tf32", "cfg3-bf16", "cfg4-tf32", "cfg4-bf16", "cfg5-tf32",
            "cfg5-bf16", "chi-tf32", "chi-bf16", "dit256-tf32"] + \
    [f"cg_{n}-tf32" for n in cg_ref.PIPELINES] + ["cg_hopper-fp32", "cg_halfcheetah-fp32"]
CHI_BATCH, CHI_STEPS = 2048, 50
WORST, COST = {}, {}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    WORST.clear()
    COST.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n[audit] {torch.cuda.get_device_name(0)}: largest error as a fraction of the bound")
        for line in pa.report_lines(WORST):
            print("[audit] " + line)
        for k, (sec, extra, base) in sorted(COST.items()):
            print(f"[audit] {k}: {sec:.1f} s, peak {extra / 2 ** 30:.2f} GB on top of the program's {base / 2 ** 30:.2f} GB")


@pytest.fixture(autouse=True)
def _engine(monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.delenv("CDS_BRANCHES", raising=False)
    torch.backends.cuda.matmul.allow_tf32 = False


def _sample(name):
    """the program's agent after one sample() at its benchmarked batch"""
    if name == "chi":
        ctor = cc.NETS["kitchen"]
        net = ChiTransformer(**ctor)
        net.load_state_dict(cc.weights(net.state_dict(), synth_state_dict))
        x_max = torch.ones((1, ctor["Ta"], ctor["act_dim"]), device=DEV)
        agent = DDPM(net.eval().to(DEV), IdentityCondition(dropout=0.0), x_max=x_max, x_min=-x_max,
                     diffusion_steps=CHI_STEPS, device=DEV)
        agent.model_ema.eval()
        g = torch.Generator().manual_seed(CHI_BATCH)
        prior = torch.zeros(CHI_BATCH, ctor["Ta"], ctor["act_dim"], device=DEV)
        cond = torch.randn(CHI_BATCH, ctor["To"], ctor["obs_dim"], generator=g).to(DEV)
        with torch.no_grad():
            agent.sample(prior, n_samples=CHI_BATCH, sample_steps=CHI_STEPS, condition_cfg=cond, w_cfg=1.0, use_ema=True)
        return agent
    if name == "dit256":
        return _dit256()
    if name.startswith("cg_"):
        return _guided(name[3:])
    w = workloads.BUILDERS[name](DEV)
    with torch.no_grad():
        w.sample(DEV)
    return w.agent


def _dit256(batch=2048, steps=20, w_cfg=6.0):
    """cfg4 (cleandiffuser_b200/workloads.py) with a DiT1d of d_model 256 (8 heads of 32) over x_t of 96 channels"""
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE
    from cleandiffuser_b200.nn_condition import MLPCondition
    from cleandiffuser_b200.nn_diffusion import DiT1d
    from cleandiffuser_b200.testing import load_synth
    H, D = 100, 96
    net = load_synth(DiT1d(D, emb_dim=128, d_model=256, n_heads=8, depth=2, timestep_emb_type="fourier"), seed=0)
    nc = load_synth(MLPCondition(1, 128, [128], torch.nn.SiLU(), dropout=0.25), seed=3)
    mask = torch.zeros(H, D)
    mask[0] = 1.
    agent = ContinuousDiffusionSDE(net, nc, fix_mask=mask, predict_noise=True, noise_schedule="linear", device=DEV)
    agent.model.eval()
    agent.model_ema.eval()
    g = torch.Generator().manual_seed(1)
    prior = torch.zeros(batch, H, D)
    prior[:, 0] = torch.randn(batch, D, generator=g)
    cond = torch.rand(batch, 1, generator=g)
    with torch.no_grad():
        agent.sample(prior.to(DEV), n_samples=batch, solver="ode_dpmsolver++_2M", sample_steps=steps,
                     sample_step_schedule="uniform_continuous", temperature=0.5, w_cfg=w_cfg, condition_cfg=cond.to(DEV))
    return agent


def _guided(shape, batch=3200, steps=20, w_cg=0.3):
    """scripts/cg_bench.py's guided call (DiscreteDiffusionSDE, JannerUNet1d denoiser, 20 DDPM steps, w_cg = 0.3) with the
    classifier of a reference pipeline (cg_ref.PIPELINES); the horizon-4 halfcheetah denoiser halves twice, not three times"""
    from cleandiffuser_b200.diffusion import DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_diffusion import JannerUNet1d
    kw = cg_ref.PIPELINES[shape]
    H, D, obs = kw["horizon"], kw["in_dim"], cg_ref.OBS_DIM[shape]
    net = load_synth(JannerUNet1d(D, model_dim=32, emb_dim=32, kernel_size=5, dim_mult=[1, 4, 2] if H == 4 else [1, 2, 2, 2]),
                     seed=0)
    mask = torch.zeros(H, D)
    mask[0, :obs] = 1.
    agent = DiscreteDiffusionSDE(net, None, fix_mask=mask, predict_noise=True, diffusion_steps=steps, device=DEV,
                                 classifier=cg_ref.make_classifier(kw, 31, DEV))
    g = torch.Generator().manual_seed(1)
    prior = torch.zeros(batch, H, D)
    prior[:, 0, :obs] = torch.randn(batch, obs, generator=g)
    agent.sample(prior.to(DEV), solver="ddpm", n_samples=batch, sample_steps=steps, use_ema=True, temperature=0.5, w_cg=w_cg)
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS.get("guidance_reason")
    return agent


def _centre_tap_dgrad(op):
    """the data gradient of a Downsample1d over a length-1 map: one 1x1 conv of its centre tap, no bias"""
    c = op.u.conv
    return op.kind == cabi.OP_CONV and c.taps == 1 and c.L_in == c.L_out == 1 and c.C_in == c.C_out and \
        not (c.bias.step or c.bias.sample)


def _build(prog, monkeypatch):
    name, math_mode = prog.split("-")
    monkeypatch.setenv("CDS_MATH", math_mode)
    agent = _sample(name)
    assert len(agent._engine_plans) == 1
    plan = next(iter(agent._engine_plans.values()))
    torch.cuda.synchronize()
    return agent, plan


def _start(plan):
    """a seeded x_t at iteration 0"""
    g = torch.Generator(device=DEV).manual_seed(7)
    plan.x.copy_(torch.randn(plan.x.shape, generator=g, device=DEV))


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Cost:
    def __init__(self, key):
        self.key = key

    def __enter__(self):
        torch.cuda.synchronize()
        self.base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.perf_counter()

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        COST[self.key] = (time.perf_counter() - self.t0, torch.cuda.max_memory_allocated() - self.base, self.base)


@pytest.mark.parametrize("prog", PROGRAMS)
def test_every_operator_matches_fp64(prog, monkeypatch):
    agent, plan = _build(prog, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    its = sorted({0, 1, n // 2 if n >= 50 else 0, n - 1} & set(range(n)))
    with _Cost(f"{prog} per-operator audit ({len(its)} iterations)"):
        aud = pa.Auditor(prog, ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
        _start(plan)
        aud.audit_once(0)
        nxt = 0
        for it in its:
            if it > nxt:
                plan.handle.run(nxt, it - nxt, st, True)         # graph replay up to the audited iteration
                torch.cuda.synchronize()
            aud.audit_iteration(it)
            nxt = it + 1
    for inst, (frac, where) in aud.worst.items():
        WORST[(prog, inst)] = (frac, where)
    assert not aud.failures, "\n".join(aud.failures[:20])
    # every launch of an iteration is one of the operators checked above, or the counter advance
    assert plan.handle.launches_per_iter() == pa.launches_per_iter(ops)
    if prog.startswith("cg_halfcheetah"):       # horizon 4: the last Downsample's input has length 1
        assert any(_centre_tap_dgrad(op) for op in ops)


@pytest.mark.parametrize("prog", PROGRAMS)
def test_replay_gives_the_bits_of_operator_by_operator_runs(prog, monkeypatch):
    agent, plan = _build(prog, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    f = min(1, n - 1)
    K = min(12, n - f)
    with _Cost(f"{prog} whole iterations {f}..{f + K - 1}"):
        mem = emulator.Owned(pa.plan_owners(plan))
        written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(f, f + K))]
        _start(plan)
        plan.handle.run(0, f, st, True)
        torch.cuda.synchronize()
        snap = [t.cpu() for t in written]                   # (host copies: the programs' buffers are several GB)
        outs = []
        for mode in ("op by op", "graph", "direct"):
            for t, s in zip(written, snap):
                t.copy_(s)
            if mode == "op by op":
                pa.run_op_by_op(plan.handle, ops, f, K, st, torch.cuda.synchronize)
            else:
                plan.handle.run(f, K, st, mode == "graph")
            torch.cuda.synchronize()
            if mode == "op by op":
                outs = [t.cpu() for t in written]
                continue
            diff = [f"{tuple(t.shape)} {t.dtype}" for t, o in zip(written, outs) if not pa.same_bits(t.cpu(), o)]
            assert not diff, f"{mode}: {len(diff)} buffers differ from the operator-by-operator run: {diff[:8]}"
        assert torch.isfinite(plan.x).all()
        assert any(t.data_ptr() == plan.x.data_ptr() for t in written)


@pytest.mark.parametrize("prog,branches", [("cfg2-tf32", 2), ("cfg2-tf32", 4), ("cfg4-tf32", 2)])
def test_parallel_branches_give_the_operator_by_operator_bits(prog, branches, monkeypatch):
    """Branch programs cap conv_tc at one CTA per SM: their whole iterations must give the bits of the single-branch program
    run one operator at a time"""
    agent, plan = _build(prog, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    f = min(1, n - 1)
    K = min(12, n - f)
    carried = ("x", "xhat_prev", "aux", "noise")                 # the root buffers that carry state across iterations
    _start(plan)
    plan.handle.run(0, f, st, True)
    torch.cuda.synchronize()
    state = {k: getattr(plan, k).clone() for k in carried if getattr(plan, k) is not None}
    pa.run_op_by_op(plan.handle, ops, f, K, st, torch.cuda.synchronize)
    torch.cuda.synchronize()
    want = {k: getattr(plan, k).clone() for k in state}
    plan.close()
    agent._engine_plans.clear()
    monkeypatch.setenv("CDS_BRANCHES", str(branches))
    name = prog.split("-")[0]
    w = workloads.BUILDERS[name](DEV)                           # same weights, inputs and tables; the noise tape is copied
    with torch.no_grad():
        w.sample(DEV)
    planb = next(iter(w.agent._engine_plans.values()))
    assert planb.n_branches == branches
    for graph in (True, False):
        for k, v in state.items():
            getattr(planb, k).copy_(v)
        planb.handle.run(f, K, st, graph)
        torch.cuda.synchronize()
        for k in want:
            if k != "noise":
                assert pa.same_bits(getattr(planb, k), want[k]), (k, "graph" if graph else "direct")
    assert math.isfinite(float(planb.x.abs().max()))


GRAD_BATCH = {"dql-eps": 4096, "dql-x0": 256}


def _grad_plan(case, math_mode, monkeypatch):
    """a GradSamplerPlan after one sample(requires_grad=True) of grad_ref.GRAD_CASES[case] at its batch"""
    monkeypatch.setenv("CDS_MATH", math_mode)
    agent, kw = grad_ref.grad_agent(case, DEV)
    B, spec = GRAD_BATCH[case], grad_ref.GRAD_CASES[case]
    g = torch.Generator().manual_seed(B)
    prior = torch.randn(B, spec["net"]["act_dim"], generator=g).to(DEV)
    cond = torch.randn(B, spec["net"]["obs_dim"], generator=g).to(DEV)
    agent.sample(prior, n_samples=B, condition_cfg=cond, **kw)
    (plan,) = agent._engine_plans.values()
    torch.cuda.synchronize()
    assert isinstance(plan, runtime.GradSamplerPlan) and plan.n_iters == 5
    return plan


@pytest.mark.parametrize("case", list(grad_ref.GRAD_CASES))
@pytest.mark.parametrize("math_mode", ["fp32", "tf32"])
def test_differentiable_programs_match_fp64_and_replay_bits(case, math_mode, monkeypatch):
    """Every operator of the 5 forward iterations and of the 5 backward iterations (from a seeded d x0, accumulators zeroed
    as GradSamplerPlan.backward does) against fp64; then both programs' whole iterations give the same bits operator by
    operator, by graph replay and by direct launches."""
    plan = _grad_plan(case, math_mode, monkeypatch)
    prog, st = f"{case}-{math_mode}", _stream()
    with _Cost(f"{prog} per-operator audit (5 + 5 iterations)"):
        _start(plan)
        fa, ba = pa.audit_grad_plan(prog, plan, plan.handle, plan.back_handle, st, torch.cuda.synchronize)
    for aud in (fa, ba):
        for inst, (frac, where) in aud.worst.items():
            WORST[(aud.name, inst)] = (frac, where)
    assert not fa.failures and not ba.failures, "\n".join((fa.failures + ba.failures)[:20])
    assert plan.handle.launches_per_iter() == pa.launches_per_iter(plan.program.ops)
    assert plan.back_handle.launches_per_iter() == pa.launches_per_iter(plan.back.ops)

    n = plan.n_iters
    with _Cost(f"{prog} whole iterations, both programs"):
        mem = emulator.Owned(pa.plan_owners(plan))
        for ops, handle, first in ((plan.program.ops, plan.handle, None), (plan.back.ops, plan.back_handle, 0)):
            written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(n))]
            if first is None:
                _start(plan)
            else:
                pa.seed_backward(plan, 3)
            torch.cuda.synchronize()
            snap = [t.cpu() for t in written]
            outs = None
            for mode in ("op by op", "graph", "direct"):
                for t, s in zip(written, snap):
                    t.copy_(s)
                if mode == "op by op":
                    pa.run_op_by_op(handle, ops, 0, n, st, torch.cuda.synchronize)
                else:
                    handle.run(0, n, st, mode == "graph")
                torch.cuda.synchronize()
                if outs is None:
                    outs = [t.cpu() for t in written]
                    continue
                diff = [f"{tuple(t.shape)}" for t, o in zip(written, outs) if not pa.same_bits(t.cpu(), o)]
                assert not diff, f"{prog} {mode}: {len(diff)} buffers differ from the operator-by-operator run: {diff[:8]}"
