"""Audit of the programs bench.py measures, at the batch each is benchmarked with (tests/program_audit.py does the work).

Programs: cfg2 (fp32, tf32, bf16), cfg3 / cfg4 / cfg5 (tf32, bf16) from cleandiffuser_b200/workloads.py, and the
ChiTransformer kitchen shape (tests/golden/chi_cases.py) at batch 2048 as scripts/chitransformer_bench.py builds it (tf32,
bf16).  None of them launches linear_ln (csrc/linear_ln.cuh serves 256 output channels only: cfg4's d_model is 320, and
ChiTransformer's Linear layers are not gated), so "dit256" adds cfg4 with a DiT1d whose widths it serves -- d_model 256 and
x_t of 96 channels, so that x_proj, which reads x_t shared by the two CFG halves (in_batch_mod), is fused as well.  Each
is built by one ``sample()``, so that the plan, its tables and its per-call fills are what production builds; its handle
is then driven directly.

- Every operator of iterations 0, 1, the middle one (loops of 50 steps or more) and the last, reached by graph replay, is
  run alone and checked on every trajectory against fp64 under its kernel family's bound, and for writes outside its
  outputs; every CONV -> LNMOD pair once more as one range (the fused linear_ln launch where the plan fused it).
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

import chi_cases as cc
import emulator
import program_audit as pa
from cleandiffuser_b200 import workloads
from cleandiffuser_b200.diffusion import DDPM
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import ChiTransformer
from cleandiffuser_b200.testing import synth_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PROGRAMS = ["cfg2-fp32", "cfg2-tf32", "cfg2-bf16", "cfg3-tf32", "cfg3-bf16", "cfg4-tf32", "cfg4-bf16", "cfg5-tf32",
            "cfg5-bf16", "chi-tf32", "chi-bf16", "dit256-tf32"]
# CONV -> LNMOD pairs per iteration the plan runs as one linear_ln launch: dit256's x_proj -> LN and, per block, the gated
# out-projection -> LN and fc2 -> LN (the last one feeding the final LayerNorm); no other program reaches linear_ln (see above),
# and bf16 / fp32 programs never fuse.  Not every CONV -> LNMOD pair fuses: cfg4's and ChiTransformer's widths are not served,
# ChiTransformer's out-projections have no gate, and x_proj reads x_t padded to 32 channels (fewer than linear_ln's 96).
FUSED_EXPECTED = {"dit256-tf32": 5}
CHI_BATCH, CHI_STEPS = 2048, 50
WORST, COST, FUSED = {}, {}, {}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    WORST.clear()
    COST.clear()
    FUSED.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n[audit] {torch.cuda.get_device_name(0)}: largest error as a fraction of the bound")
        for line in pa.report_lines(WORST):
            print("[audit] " + line)
        for k, (fused, pairs) in sorted(FUSED.items()):
            print(f"[audit] {k}: {pairs} CONV -> LNMOD pairs per iteration, {fused} of them fused into one linear_ln launch")
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
    pairs = [i for i in range(len(ops)) if pa.is_pair(ops, i)]
    assert aud.pairs == len(pairs) * len(its)
    # launches_per_iter() says how many pairs the plan fused; every pair ran as one range above, so each fused launch was checked
    fused = pa.fused_pairs(plan.handle, ops)
    FUSED[prog] = (fused, len(pairs))
    assert fused == FUSED_EXPECTED.get(prog, 0), (fused, len(pairs))


@pytest.mark.parametrize("prog", PROGRAMS)
def test_replay_gives_the_bits_of_operator_by_operator_runs(prog, monkeypatch):
    agent, plan = _build(prog, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    f = min(1, n - 1)
    K = min(12, n - f)
    with _Cost(f"{prog} whole iterations {f}..{f + K - 1}"):
        mem = emulator.Owned(pa.plan_owners(plan))
        written = [mem.owners[i] for i in pa.written_owners(mem, ops)]
        _start(plan)
        plan.handle.run(0, f, st, True)
        torch.cuda.synchronize()
        snap = [t.cpu() for t in written]                   # (host copies: the programs' buffers are several GB)
        outs = []
        for mode in ("op by op", "graph", "direct"):
            for t, s in zip(written, snap):
                t.copy_(s)
            if mode == "op by op":
                pa.run_op_by_op(plan.handle, ops, f, K, st, torch.cuda.synchronize, pairs=True)
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
    """Branch programs cap conv_tc at one CTA per SM and never fuse linear_ln: their whole iterations must give the bits of
    the single-branch program run one operator at a time (no pair fused)"""
    agent, plan = _build(prog, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    f = min(1, n - 1)
    K = min(12, n - f)
    carried = ("x", "xhat_prev", "aux", "noise")                 # the root buffers that carry state across iterations
    _start(plan)
    plan.handle.run(0, f, st, True)
    torch.cuda.synchronize()
    state = {k: getattr(plan, k).clone() for k in carried if getattr(plan, k) is not None}
    pa.run_op_by_op(plan.handle, ops, f, K, st, torch.cuda.synchronize, pairs=False)
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
