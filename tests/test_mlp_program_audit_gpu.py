"""Audit of the MLP denoiser programs of the offline-RL and Diffusion-BC pipelines (tests/mlp_programs.py) at the batches
those pipelines sample with, in fp32, tf32 and bf16 (tests/program_audit.py does the per-operator work):

- every operator of every iteration (loops of 10 steps or fewer; DBC's 58: iterations 0, 1, the middle one and the last),
  reached by graph replay, run alone and checked against fp64 under its kernel family's bound and for stray writes;
- one iteration is one launch per operator plus the counter advance;
- ``min(12, n_iters - 1)`` whole iterations from iteration 1 give the same bits operator by operator (a synchronisation
  after each), by graph replay and by direct launches;
- the forms these programs exist to reach are reached: conv_simt storing TF32 / bf16 (SfBCUNet, PearceMlp), LNMOD with one
  modulation row for the whole batch (IDQLMlp), SfBCUNet's first block with both CFG row maps;
- the lowered denoiser against the fp64 module (mlp_programs.denoiser_check): what the per-operator audit cannot see.

The module prints the largest error as a fraction of the bound per (program, kernel instantiation), the lowering errors,
and the wall time and peak device memory each audit adds to its program."""
import time

import pytest
import torch

import emulator
import mlp_programs as mp
import program_audit as pa

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODES = ["fp32", "tf32", "bf16"]
WORST, COST, LOWERING = {}, {}, {}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    WORST.clear()
    COST.clear()
    LOWERING.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n[mlp audit] {torch.cuda.get_device_name(0)}: largest error as a fraction of the bound")
        for line in pa.report_lines(WORST):
            print("[mlp audit] " + line)
        for k, errs in sorted(LOWERING.items()):
            print(f"[mlp lowering] {k}: " + ", ".join(f"{n} {e:.2e}" for n, e in errs.items()))
        for k, (sec, extra, base) in sorted(COST.items()):
            print(f"[mlp audit] {k}: {sec:.1f} s, peak {extra / 2 ** 30:.2f} GB on top of the program's {base / 2 ** 30:.2f} GB")


@pytest.fixture(autouse=True)
def _engine(monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.delenv("CDS_BRANCHES", raising=False)
    torch.backends.cuda.matmul.allow_tf32 = False


def _build(name, math_mode, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math_mode)
    agent, plan = mp.sample(name, DEV)
    torch.cuda.synchronize()
    return agent, plan


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.mark.parametrize("math_mode", MODES)
@pytest.mark.parametrize("name", list(mp.PROGRAMS))
def test_every_operator_matches_fp64(name, math_mode, monkeypatch):
    agent, plan = _build(name, math_mode, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    if name.startswith("dbc"):
        assert n == mp.PROGRAMS[name][1] + mp.DBC_EXTRA
    its = sorted({0, 1, n // 2, n - 1}) if n > 10 else list(range(n))
    prog = f"{name}-{math_mode}"
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    aud = pa.Auditor(prog, ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    g = torch.Generator(device=DEV).manual_seed(7)
    plan.x.copy_(torch.randn(plan.x.shape, generator=g, device=DEV))
    aud.audit_once(0)
    nxt = 0
    for it in its:
        if it > nxt:
            plan.handle.run(nxt, it - nxt, st, True)         # graph replay up to the audited iteration
            torch.cuda.synchronize()
        aud.audit_iteration(it)
        nxt = it + 1
    torch.cuda.synchronize()
    COST[f"{prog} per-operator audit ({len(its)} iterations)"] = (time.perf_counter() - t0,
                                                                   torch.cuda.max_memory_allocated() - base, base)
    for inst, (frac, where) in aud.worst.items():
        WORST[(prog, inst)] = (frac, where)
    assert not aud.failures, "\n".join(aud.failures[:20])
    assert plan.handle.launches_per_iter() == pa.launches_per_iter(ops)

    mp.check_forms(name, math_mode, plan)


@pytest.mark.parametrize("math_mode", MODES)
@pytest.mark.parametrize("name", list(mp.PROGRAMS))
def test_lowered_denoiser_matches_the_fp64_module(name, math_mode, monkeypatch):
    agent, plan = _build(name, math_mode, monkeypatch)
    err = mp.denoiser_check(name, agent, plan, stream=_stream(), sync=torch.cuda.synchronize)
    LOWERING[f"{name}-{math_mode}"] = err
    assert max(err.values()) <= mp.LOWERING_TOL[math_mode], err


@pytest.mark.parametrize("math_mode", MODES)
@pytest.mark.parametrize("name", list(mp.PROGRAMS))
def test_replay_gives_the_bits_of_operator_by_operator_runs(name, math_mode, monkeypatch):
    agent, plan = _build(name, math_mode, monkeypatch)
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    f = 1
    K = min(12, n - f)
    mem = emulator.Owned(pa.plan_owners(plan))
    written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(f, f + K))]
    g = torch.Generator(device=DEV).manual_seed(7)
    plan.x.copy_(torch.randn(plan.x.shape, generator=g, device=DEV))
    plan.handle.run(0, f, st, True)
    torch.cuda.synchronize()
    snap = [t.clone() for t in written]
    outs = None
    for mode in ("op by op", "graph", "direct"):
        for t, s in zip(written, snap):
            t.copy_(s)
        if mode == "op by op":
            pa.run_op_by_op(plan.handle, ops, f, K, st, torch.cuda.synchronize)
        else:
            plan.handle.run(f, K, st, mode == "graph")
        torch.cuda.synchronize()
        if outs is None:
            outs = [t.clone() for t in written]
            continue
        diff = [f"{tuple(t.shape)} {t.dtype}" for t, o in zip(written, outs) if not pa.same_bits(t, o)]
        assert not diff, f"{mode}: {len(diff)} buffers differ from the operator-by-operator run: {diff[:8]}"
    assert torch.isfinite(plan.x).all()
    assert any(t.data_ptr() == plan.x.data_ptr() for t in written)
