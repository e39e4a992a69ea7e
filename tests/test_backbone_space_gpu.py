"""The constructor space of the lowered backbones (tests/backbone_space.py) on the H100, in fp32, TF32 and bf16.

Every served case, in every math mode, is built by one 2-step ``sample()`` at a batch of 256 (every conv_tc / conv_ps
launch has two or more row tiles) and then checked three ways:

- every operator of iteration 1 alone against fp64 under its kernel family's bound (tests/program_audit.py), and for
  writes outside its outputs -- this is what names the failing kernel;
- both iterations give the same bits operator by operator, by graph replay and by direct launches;
- the lowered denoiser against the float64 module (mlp_programs.LOWERING_TOL), at iteration 1.

Cases labelled "refused" or "unsupported" must take the PyTorch loop (no engine call) and give its result.  The module
prints the largest error as a fraction of the bound per (math mode, kernel instantiation + the conv's taps and GroupNorm
length) and asserts that the forms this table exists for were reached: conv_tc with 7 taps, conv_simt + GroupNorm at
L_out 64 and 128, the CUDA-core attention at head_dim 16 and 64."""
import time

import pytest
import torch

import backbone_space as bs
import emulator
import mlp_programs as mp
import program_audit as pa
from cleandiffuser_b200.engine import cabi, runtime

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODES = ["fp32", "tf32", "bf16"]
BATCH, STEPS = 256, 2
WORST, LOWERING, COST = {}, {}, {}
SERVED = [(n, m) for n, c in bs.CASES.items() if c["want"] == "served" for m in MODES]
FALLBACK = [(n, "fp32") for n, c in bs.CASES.items() if c["want"] != "served"] + \
    [(n, m) for n, c in bs.CASES.items() if c["want"] == "refused" for m in ("tf32", "bf16")]


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n[backbone space] {torch.cuda.get_device_name(0)}: largest error as a fraction of the bound")
        for line in pa.report_lines(WORST):
            print("[backbone space] " + line)
        worst = sorted(LOWERING.items(), key=lambda kv: -kv[1] / mp.LOWERING_TOL[kv[0][1]])[:10]
        print("[backbone space] largest whole-denoiser errors: " +
              ", ".join(f"{n}-{m} {e:.2e}" for (n, m), e in worst))
        for k, v in sorted(COST.items()):
            print(f"[backbone space] {k}: {v:.1f} s")


@pytest.fixture(autouse=True)
def _engine(monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.delenv("CDS_BRANCHES", raising=False)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


_instantiation = pa.instantiation


def _form(op):
    """the kernel instantiation of ``op`` and, for convolutions, the taps and the length L_out of a GroupNorm tile"""
    inst = _instantiation(op)
    if op.kind == cabi.OP_CONV:
        c = op.u.conv
        inst += f" taps {c.taps}" + (f" gn L {c.L_out}" if c.groups else "")
    return inst


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("name,math_mode", SERVED)
def test_served_backbone(name, math_mode, monkeypatch):
    t0 = time.perf_counter()
    monkeypatch.setenv("CDS_MATH", math_mode)
    case = bs.CASES[name]
    net = bs.build(case).to(DEV)
    agent = bs.agent(case, net, DEV, STEPS)
    calls = runtime.STATS["engine_calls"]
    with torch.no_grad():
        bs.sample(agent, case, BATCH, STEPS, DEV)
    assert runtime.STATS["engine_calls"] == calls + 1
    (plan,) = agent._engine_plans.values()
    ops, st = plan.program.ops, _stream()
    prog = f"{name}-{math_mode}"
    torch.cuda.synchronize()

    # every operator of iteration 1 against fp64, its worst fraction recorded per form
    monkeypatch.setattr(pa, "instantiation", _form)
    aud = pa.Auditor(prog, ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    g = torch.Generator(device=DEV).manual_seed(7)
    plan.x.copy_(torch.randn(plan.x.shape, generator=g, device=DEV))
    aud.audit_once(0)
    plan.handle.run(0, 1, st, True)
    torch.cuda.synchronize()
    aud.audit_iteration(1)
    for inst, (frac, where) in aud.worst.items():
        key = (math_mode, inst)
        if frac > WORST.get(key, (-1.0, ""))[0]:
            WORST[key] = (frac, f"{name} {where}")
    assert not aud.failures, "\n".join(aud.failures[:20])
    assert plan.handle.launches_per_iter() == pa.launches_per_iter(ops)

    # whole iterations: operator by operator, graph replay and direct launches give the same bits
    mem = emulator.Owned(pa.plan_owners(plan))
    written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(STEPS))]
    plan.x.copy_(torch.randn(plan.x.shape, generator=g, device=DEV))
    torch.cuda.synchronize()
    snap = [t.clone() for t in written]
    outs = None
    for mode in ("op by op", "graph", "direct"):
        for t, s in zip(written, snap):
            t.copy_(s)
        if mode == "op by op":
            pa.run_op_by_op(plan.handle, ops, 0, STEPS, st, torch.cuda.synchronize)
        else:
            plan.handle.run(0, STEPS, st, mode == "graph")
        torch.cuda.synchronize()
        if outs is None:
            outs = [t.clone() for t in written]
            continue
        diff = [f"{tuple(t.shape)} {t.dtype}" for t, o in zip(written, outs) if not pa.same_bits(t, o)]
        assert not diff, f"{mode}: {len(diff)} buffers differ from the operator-by-operator run: {diff[:8]}"

    # the lowered denoiser at iteration 1 against the fp64 module
    tab = next(iter(agent._engine_tables.values()))
    gc = torch.Generator().manual_seed(5)
    cond = None if case["cond"] is None else torch.randn(BATCH, *case["cond"], generator=gc).to(DEV)
    plan.fill_tables(tab.t, cond)
    plan.x.copy_(torch.randn(plan.x.shape, generator=gc).to(DEV))
    j = mp.prediction_op(ops)
    plan.handle.run(1, 0, st, False)
    plan.handle.run_range(1, 0, j + 1, st)
    torch.cuda.synchronize()
    y = emulator.view(emulator.Owned(pa.plan_owners(plan)), *pa.declared_outputs(ops[j], 1)[0])
    err = bs.rel_err(y, bs.reference(net, case, plan.x.clone(), tab.t[1:2], cond))
    LOWERING[(name, math_mode)] = err
    COST[f"served {math_mode}"] = COST.get(f"served {math_mode}", 0.0) + time.perf_counter() - t0
    assert err <= mp.LOWERING_TOL[math_mode], (name, case["ctor"], err)


@pytest.mark.parametrize("name,math_mode", FALLBACK)
def test_fallback_gives_the_pytorch_loop(name, math_mode, monkeypatch):
    t0 = time.perf_counter()
    monkeypatch.setenv("CDS_MATH", math_mode)
    case = bs.CASES[name]
    net = bs.build(case).to(DEV)
    results = []
    for backend in ("auto", "torch"):
        monkeypatch.setenv("CDS_BACKEND", backend)
        agent = bs.agent(case, net, DEV, STEPS)
        calls, falls = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
        try:
            with torch.no_grad():
                results.append(bs.sample(agent, case, BATCH, STEPS, DEV))
        except Exception as e:            # a module that cannot run raises in the PyTorch loop, on either path
            results.append(type(e))
        assert runtime.STATS["engine_calls"] == calls and not agent._engine_plans
        if backend == "auto":
            assert runtime.STATS["fallbacks"] == falls + 1
            reason = runtime.STATS["last_fallback_reason"]
            if case["want"] == "refused":
                assert reason.startswith("libcds error -3"), reason
            else:
                assert case["want"][len("unsupported: "):] in reason, reason
    a, b = results
    if isinstance(a, torch.Tensor):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6)
    else:
        assert a is b
    COST["fallbacks"] = COST.get("fallbacks", 0.0) + time.perf_counter() - t0


def test_new_instantiations_are_reached():
    """conv_tc with 7 taps, conv_simt + GroupNorm at L_out 64 and 128, the CUDA-core attention at head_dim 16 and 64"""
    if len(WORST) == 0:
        pytest.skip("runs after the served cases of this module")
    REACHED = {inst for _, inst in WORST}
    assert any(f.startswith("conv tc") and " taps 7" in f for f in REACHED), sorted(REACHED)
    for L in (64, 128):
        assert any(f.startswith("conv simt") and f.endswith(f" gn L {L}") for f in REACHED), (L, sorted(REACHED))
    for hd in (16, 64):
        assert any(f.startswith(f"attn f32 {hd} ") for f in REACHED), (hd, sorted(REACHED))
