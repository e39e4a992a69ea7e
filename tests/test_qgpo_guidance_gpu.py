"""QGPO's classifier guidance inside the replayed loop on the H100: CDS_OP_DGRAD / CDS_OP_STASH with SiLU (tests/grad_ref.py)
and CDS_OP_HEAD_GRAD (tests/cg_ref.py) against fp64, QGPONNClassifier's lowered input gradient against fp64 autograd at the
D4RL MuJoCo shapes, QGPO-shaped sample() calls against the host-callback path and the goldens, graph replay /
reproducibility, and an operator-by-operator audit of the guided iteration (tests/program_audit.py)."""
import numpy as np
import pytest
import torch

import cg_ref
import emulator
import grad_ref
import make_golden_qgpo as mg
import program_audit as pa
import qgpo_ref
from common import load_golden, tape_of
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape, load_synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}
ROWS = [50, 333, 800]              # QGPO's batches (50 envs; 800 = 50 x 16 candidates) and one that is no multiple of 32
WIDTHS = [64, 192, 256]            # the classifier's embedding, its first Linear's input, its hidden width


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _run(op, it=0):
    cabi.run_op(0, op, it, _stream())
    torch.cuda.synchronize()


def _frac(got, want, bound):
    err = np.abs(got.cpu().numpy().astype(np.float64) - want)
    return float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), np.where(err > 0, np.inf, 0.0))))


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("N", WIDTHS)
@pytest.mark.parametrize("K", WIDTHS)
def test_dgrad_silu_matches_fp64(rows, N, K):
    """out = (dz W) silu'(z) under grad_ref.dgrad_bound, and bitwise equal over two runs"""
    g = torch.Generator().manual_seed(rows + 7 * N + K)
    dz, w, z = torch.randn(rows, N, generator=g), torch.randn(N, K, generator=g) / N ** 0.5, 3 * torch.randn(2, rows, K, generator=g)
    dz, w, z = dz.to(DEV), w.to(DEV), z.to(DEV)
    out = torch.full((rows, K), 7.0, device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_DGRAD
    d = op.u.dgrad
    d.rows, d.N, d.K, d.dz, d.ldz, d.w, d.ldw = rows, N, K, dz.data_ptr(), N, w.data_ptr(), K
    d.z, d.z_iter_stride, d.act = z.data_ptr(), rows * K, cabi.ACT_SILU
    d.out, d.ldo = out.data_ptr(), K
    _run(op, 1)                                             # iteration 1: the second slot of z
    first = out.clone()
    args = (dz.cpu().numpy(), w.cpu().numpy(), z[1].cpu().numpy(), cabi.ACT_SILU)
    frac = _frac(out, grad_ref.dgrad(*args), grad_ref.dgrad_bound(*args))
    assert frac <= 1.0, frac
    _run(op, 1)
    assert torch.equal(out, first)
    print(f"[qgpo] dgrad silu rows={rows} N={N} K={K}: {frac:.3g} of the bound")


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("K,act", [(256, cabi.ACT_SILU), (64, cabi.ACT_SILU), (100, cabi.ACT_NONE)])
def test_head_grad_matches_fp64(rows, K, act):
    g = torch.Generator().manual_seed(rows + K)
    ldh = K + 4
    h = (4 * torch.randn(rows, ldh, generator=g)).to(DEV)
    w, b = (torch.randn(K, generator=g) / 4).to(DEV), torch.randn(1, generator=g).to(DEV)
    seed = torch.full((rows + 3,), 7.0, device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_HEAD_GRAD
    q = op.u.head_grad
    q.rows, q.K, q.h, q.ldh, q.act = rows, K, h.data_ptr(), ldh, act
    q.w, q.b, q.scale, q.seed = w.data_ptr(), b.data_ptr(), 10.0, seed.data_ptr()
    _run(op)
    first = seed.clone()
    hh, ww, bb = h[:, :K].cpu().numpy(), w.cpu().numpy(), b.cpu().numpy()
    z, want = cg_ref.head_grad(hh, ww, bb, 10.0, act)
    frac = _frac(seed[:rows], want, cg_ref.head_grad_bound(hh, ww, bb, 10.0, act))
    assert frac <= 1.0, frac
    assert bool((seed[rows:] == 7.0).all()), "HEAD_GRAD wrote past its rows"
    assert np.abs(z).max() > 10, "the cases should reach the tanh's saturation"
    _run(op)
    assert torch.equal(seed, first)
    print(f"[qgpo] head_grad rows={rows} K={K} act={act}: {frac:.3g} of the bound")


@pytest.mark.parametrize("n", [50 * 256, 333 * 192, 800 * 64 + 5])
def test_stash_silu_without_slot(n):
    g = torch.Generator().manual_seed(n)
    src = (8 * torch.randn(n, generator=g)).to(DEV)
    src[:4] = torch.tensor([-100.0, -88.5, 0.0, 100.0])
    out = torch.full((n + 3,), 7.0, device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_STASH
    s = op.u.stash
    s.n, s.act, s.src, s.act_out = n, cabi.ACT_SILU, src.data_ptr(), out.data_ptr()
    _run(op)
    x = src.cpu().numpy()
    frac = _frac(out[:n], grad_ref.act(cabi.ACT_SILU, x), grad_ref.silu_bound(x))
    assert frac <= 1.0, frac
    assert bool((out[n:] == 7.0).all())


def _handle(ops, n, owners):
    return runtime._make_handle(torch.device(DEV), ops, n)


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("batch", [50, 800, 5000])
@pytest.mark.parametrize("name", list(qgpo_ref.PIPELINES))
def test_input_gradient_matches_fp64_autograd(name, batch, math):
    kw = qgpo_ref.PIPELINES[name]
    clf = qgpo_ref.make_classifier(kw, 31, DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(batch, kw["act_dim"], generator=g).clamp(-1, 1).to(DEV)
    obs = torch.randn(batch, kw["obs_dim"], generator=g).to(DEV)
    t = torch.tensor([0.9, 0.3], device=DEV)
    got, _ = cg_ref.lowered_gradient(clf, x, t, 1, MATHS[math], DEV, cond=obs, handle=_handle)
    torch.cuda.synchronize()
    want = qgpo_ref.input_gradient_fp64(clf, x, t[1].expand(batch), obs)
    rel = float((got.double() - want).norm() / want.norm())
    # fp32: summation order only (measured 5e-7 to 7e-7 on an H100).  TF32: the 256-wide hidden Linears read 10-bit mantissas
    # (measured 3.4e-4 to 5.4e-4); a wrong column block of W_1 or a missing SiLU' gives rel ~ 1
    print(f"[qgpo] input gradient {name} B={batch} {math}: rel {rel:.3g}")
    assert rel < (1e-5 if math == "fp32" else 1e-2), rel


class _Wrapped:
    """the same classifier behind a class the lowering does not recognise: the host-callback path"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


def qgpo_agent(obs_dim, act_dim, device=DEV):
    """QGPO's actor (ContinuousDiffusionSDE over SfBCUNet with MLPCondition, clip to [-1, 1]) and classifier, synthetic weights"""
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE
    from cleandiffuser_b200.nn_condition import MLPCondition
    from cleandiffuser_b200.nn_diffusion import SfBCUNet
    net = load_synth(SfBCUNet(act_dim), seed=41)
    cond = load_synth(MLPCondition(obs_dim, 64, [64], torch.nn.SiLU()), seed=42)
    agent = ContinuousDiffusionSDE(net, cond, x_max=torch.ones(act_dim), x_min=-torch.ones(act_dim), device=device)
    agent.classifier = qgpo_ref.make_classifier(dict(obs_dim=obs_dim, act_dim=act_dim), 31, device)
    agent.eval()
    return agent


def qgpo_call(agent, obs, steps, w_cg, tape):
    with tape.active():
        x0, log = agent.sample(torch.zeros(obs.shape[0], agent.model["diffusion"].out_layer.out_features, device=obs.device),
                               "ddpm", n_samples=obs.shape[0], sample_steps=steps, sample_step_schedule="quad_continuous",
                               condition_cfg=obs, w_cfg=1.0, condition_cg=obs, w_cg=w_cg)
    torch.cuda.synchronize()
    return x0, log


def _obs(batch, obs_dim, seed=1):
    return torch.randn(batch, obs_dim, generator=torch.Generator().manual_seed(seed)).to(DEV)


# QGPO's calls: halfcheetah (50 envs, 5 steps) and hopper-medium-replay (50 envs x 16 candidates, 10 steps)
CALLS = {"halfcheetah": (17, 6, 50, 5), "hopper-mr": (11, 3, 800, 10)}


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("call", list(CALLS))
def test_qgpo_call_graph_against_callback(call, math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    obs_dim, act_dim, batch, steps = CALLS[call]
    agent = qgpo_agent(obs_dim, act_dim)
    clf = agent.classifier
    obs = _obs(batch, obs_dim)
    tape = NoiseTape()
    x_graph, log = qgpo_call(agent, obs, steps, 3.0, tape)
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    print(f"[qgpo] {call} math={math}: {runtime.STATS['launches']} launches per call")
    agent.classifier = _Wrapped(clf)
    x_cb, log_cb = qgpo_call(agent, obs, steps, 3.0, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "callback"
    err = (x_graph - x_cb).abs()
    print(f"[qgpo] {call} math={math}: x0 graph vs callback max {float(err.max()):.3g} mean {float(err.mean()):.3g}")
    # log_p is the classifier's PyTorch logp of x0 after the loop on both paths
    if math == "fp32":
        assert err.max() < 1e-4, float(err.max())
        torch.testing.assert_close(log["log_p"], log_cb["log_p"], rtol=1e-4, atol=1e-4)
    else:
        # the engine's classifier reads TF32 in its 256-wide Linears where the callback's PyTorch Linears are fp32 (cuBLAS
        # TF32 is off by default): the gradients differ by ~1e-3 of their norm (input-gradient test), which a guidance weight
        # of 3 carries into x0 through the clip: measured 0.014 max / 1.4e-4 mean (hopper-mr) on an H100 80GB HBM3 at 700 W.
        # A wrong gradient moves x0 by O(1)
        assert err.max() < 2e-2 and err.mean() < 2e-3, (float(err.max()), float(err.mean()))
        torch.testing.assert_close(log["log_p"], log_cb["log_p"], rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_goldens_on_the_gpu(name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "fp32")
    G = load_golden("qgpo")
    agent, prior, kw = qgpo_ref.make_sample_agent(name, device=DEV)

    def refuse(*a, **k):
        raise AssertionError("classifier.gradients called: guidance left the program")
    monkeypatch.setattr(agent.classifier, "gradients", refuse)
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = agent.sample(prior, **kw)
    assert runtime.STATS["guidance_path"] == "graph"
    assert np.abs(x0.cpu().numpy() - G[f"sample/{name}/x0"]).max() < 1e-3
    np.testing.assert_allclose(log["log_p"].cpu().numpy(), G[f"sample/{name}/log_p"], rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("math", list(MATHS))
def test_graph_replay_equals_direct_launches_and_repeats_bitwise(math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent = qgpo_agent(11, 3)
    obs = _obs(800, 11)
    tape = NoiseTape()
    a, la = qgpo_call(agent, obs, 10, 3.0, tape)
    b, lb = qgpo_call(agent, obs, 10, 3.0, NoiseTape(tape.draws))
    monkeypatch.setenv("CDS_GRAPH", "0")
    c, _ = qgpo_call(agent, obs, 10, 3.0, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "graph"
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(la["log_p"], lb["log_p"])


@pytest.mark.parametrize("math", list(MATHS))
def test_every_operator_of_the_qgpo_iteration_matches_fp64(math, monkeypatch):
    """tests/program_audit.py over every iteration of the hopper-medium-replay call: each operator within its bound, nothing
    written outside its declared outputs; then whole iterations by graph replay give the operator-by-operator bits"""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent = qgpo_agent(11, 3)
    obs = _obs(800, 11)
    qgpo_call(agent, obs, 10, 3.0, NoiseTape())
    assert len(agent._engine_plans) == 1
    plan = next(iter(agent._engine_plans.values()))
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    assert {cabi.OP_HEAD_GRAD, cabi.OP_GUIDE} <= {op.kind for op in ops}
    torch.cuda.synchronize()
    start = torch.rand(plan.x.shape, generator=torch.Generator().manual_seed(7)).to(DEV) * 2 - 1
    plan.x.copy_(start)
    aud = pa.Auditor(f"qgpo-{math}", ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    aud.audit_once(0)
    for it in range(n):
        aud.audit_iteration(it)
    for line in pa.report_lines({(aud.name, k): v for k, v in aud.worst.items()}):
        print("[qgpo audit]", line)
    assert not aud.failures, "\n".join(aud.failures[:20])
    assert plan.handle.launches_per_iter() == pa.launches_per_iter(ops)

    mem = emulator.Owned(pa.plan_owners(plan))
    written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(n))]
    outs = {}
    for mode in ("op by op", "graph"):
        plan.x.copy_(start)
        torch.cuda.synchronize()
        if mode == "op by op":
            pa.run_op_by_op(plan.handle, ops, 0, n, st, torch.cuda.synchronize)
        else:
            plan.handle.run(0, n, st, True)
        torch.cuda.synchronize()
        outs[mode] = [t.clone() for t in written]
    assert all(pa.same_bits(a, b) for a, b in zip(outs["op by op"], outs["graph"]))
