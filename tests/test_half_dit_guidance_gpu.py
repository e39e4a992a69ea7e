"""Classifier guidance with HalfDiT1d inside the replayed loop on the H100: the backward modes of CDS_OP_ATTN, CDS_OP_LNMOD and
CDS_OP_STASH against fp64 (tests/dit_grad_ref.py), the lowered input gradient against fp64 autograd, the graph path against
the host-callback path, the goldens, graph replay / reproducibility, and an operator-by-operator audit of the guided iteration
(tests/program_audit.py)."""
import numpy as np
import pytest
import torch

import cg_ref
import dit_grad_ref as dr
import emulator
import make_golden_half_dit as mg
import program_audit as pa
from common import load_golden, tape_of
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}
DTS = {"f32": cabi.F32, "tf32": cabi.TF32}


@pytest.fixture(autouse=True)
def gelu_semantics(monkeypatch):
    dr.register(monkeypatch)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _run(op):
    cabi.run_op(0, op, 0, _stream())
    torch.cuda.synchronize()


def _frac(got, ref, bound):
    err = (got.double() - ref).abs()
    return float(torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, np.inf, 0.0)).max())


@pytest.mark.parametrize("dt", list(DTS))
@pytest.mark.parametrize("batch,L,heads,hd", [(3, 1, 1, 16), (50, 10, 2, 16), (7, 32, 8, 32), (333, 64, 8, 32),
                                              (5, 33, 6, 64), (64, 128, 6, 64), (2, 128, 1, 16), (9, 100, 3, 32)])
def test_attn_bwd_matches_fp64(batch, L, heads, hd, dt):
    C = heads * hd
    g = torch.Generator().manual_seed(batch * L + hd)
    qkv = (torch.randn(batch, L, 3 * C, generator=g) * 2).to(DEV)
    dout = torch.randn(batch, L, C, generator=g).to(DEV)
    dqkv = torch.full((batch, L, 3 * C), float("nan"), device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_ATTN
    a = op.u.attn
    a.batch, a.L, a.C, a.heads, a.qkv, a.qkv_dtype = batch, L, C, heads, qkv.data_ptr(), cabi.F32
    a.dout, a.out, a.out_dtype = dout.data_ptr(), dqkv.data_ptr(), DTS[dt]
    _run(op)
    ref = dr.attn_bwd(qkv, dout, heads)
    frac = _frac(dqkv, ref, dr.bound(ref, dr.ATTN_TOL, DTS[dt]))
    print(f"[half-dit] attn_bwd B={batch} L={L} heads={heads} hd={hd} {dt}: {frac:.3g} of the bound")
    assert frac <= 1.0
    again = torch.zeros_like(dqkv)
    a.out = again.data_ptr()
    _run(op)
    assert torch.equal(again.view(torch.int32), dqkv.view(torch.int32))          # no atomics: bitwise repeatable


@pytest.mark.parametrize("dt", list(DTS))
@pytest.mark.parametrize("batch,L,C,form", [(50, 10, 64, "block"), (333, 64, 384, "block"), (800, 1, 192, "affine"),
                                            (7, 32, 96, "bcast"), (3200, 32, 256, "block"), (5, 3, 1000, "block")])
def test_lnmod_bwd_matches_fp64(batch, L, C, form, dt):
    g = torch.Generator().manual_seed(batch + C)
    x = (torch.randn(batch, L, C, generator=g) * 3 + 1).to(DEV)
    rows = 1 if form == "affine" else batch
    mod = (torch.randn(rows, 3 * C, generator=g) * 0.5).to(DEV)              # [scale | gate | unused]
    dout = torch.randn(batch, 1 if form == "bcast" else L, C, generator=g).to(DEV)
    res = torch.randn(batch, L, C, generator=g).to(DEV) if form == "block" else None
    dx, gated = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
    op = cabi.Op()
    op.kind = cabi.OP_LNMOD
    m = op.u.lnmod
    m.batch, m.L, m.C, m.eps, m.in_ = batch, L, C, 1e-6, x.data_ptr()
    m.scale, m.mod_bstride = mod.data_ptr(), 0 if form == "affine" else 3 * C
    m.dout, m.dout_bstride, m.dout_lstride = dout.data_ptr(), dout.shape[1] * C, 0 if form == "bcast" else C
    m.res = res.data_ptr() if res is not None else None
    m.out, m.out_dtype = dx.data_ptr(), DTS[dt]
    m.gate, m.gate_bstride, m.gated, m.gated_dtype = mod.data_ptr() + 4 * C, m.mod_bstride, gated.data_ptr(), DTS[dt]
    _run(op)
    sc, gt = mod[:, :C].expand(batch, C), mod[:, C:2 * C].expand(batch, C)
    rdx, rg = dr.lnmod_bwd(x, sc, dout, 1e-6, res, gt)
    for got, ref in ((dx, rdx), (gated, rg)):
        frac = _frac(got, ref, dr.bound(ref, dr.LN_TOL, DTS[dt]))
        print(f"[half-dit] lnmod_bwd B={batch} L={L} C={C} {form} {dt}: {frac:.3g} of the bound")
        assert frac <= 1.0


@pytest.mark.parametrize("act", [cabi.ACT_GELU_TANH, cabi.ACT_SILU, cabi.ACT_MISH])
@pytest.mark.parametrize("n", [1, 1000, 3200 * 64 * 4 * 32 + 3])
def test_act_bwd_matches_fp64(n, act):
    g = torch.Generator().manual_seed(n)
    z = (torch.randn(n, generator=g) * 4).to(DEV)
    dh = torch.randn(n, generator=g).to(DEV)
    dz = torch.full_like(z, float("nan"))
    op = cabi.Op()
    op.kind = cabi.OP_STASH
    a = op.u.stash
    a.n, a.act, a.src, a.grad, a.act_out = n, act, z.data_ptr(), dh.data_ptr(), dz.data_ptr()
    _run(op)
    ref = dr.act_bwd(z, dh, act)
    assert _frac(dz, ref, dr.act_bwd_bound(z, dh, ref, act, cabi.F32)) <= 1.0


def _handle(ops, n, owners):
    return runtime._make_handle(torch.device(DEV), ops, n)


# the DiT planner shape of bench.py's cfg4 family (d_model 256, 8 heads, depth 2, horizon 32) and the reference default
# (d_model 384, 6 heads, depth 12), shortened to depth 2 to keep the fp64 reference quick
GRAD_CASES = {"planner": dict(in_dim=14, out_dim=1, emb_dim=64, d_model=256, n_heads=8, depth=2, horizon=32),
              "default": dict(in_dim=11, out_dim=3, emb_dim=64, d_model=384, n_heads=6, depth=2, horizon=20)}


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("batch", [50, 800, 3200])
@pytest.mark.parametrize("case", list(GRAD_CASES))
def test_input_gradient_matches_fp64_autograd(case, batch, math):
    kw = GRAD_CASES[case]
    clf = dr.make_classifier(kw, 31, DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(batch, kw["horizon"], kw["in_dim"], generator=g).to(DEV)
    t = torch.tensor([40, 7], device=DEV)
    got, _ = cg_ref.lowered_gradient(clf, x, t, 1, MATHS[math], DEV, handle=_handle)
    torch.cuda.synchronize()
    want = torch.cat([dr.input_gradient_fp64(clf, xc, t[1].expand(len(xc))) for xc in x.split(400)])
    rel = float((got.double() - want).norm() / want.norm())
    # fp32: summation order only (measured 1e-7 .. 1e-6 on the interpreter).  TF32: six token GEMMs per block read 10-bit
    # mantissas (2^-11 each), summing over up to 4 d_model terms: the interpreter measures 1e-3 at depth 2; 1e-2 leaves room
    # for the kernels' own summation order.  A wrong weight transpose, gate or missing derivative gives rel ~ 1
    print(f"[half-dit] input gradient {case} B={batch} {math}: rel {rel:.3g}")
    assert rel < (1e-5 if math == "fp32" else 1e-2), rel


class _Wrapped:
    """the same classifier behind a class the lowering does not recognise: the host-callback path"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


def planner_agent(horizon=32, batch=800):
    """ContinuousDiffusionSDE over a DiT1d planner (d_model 256, 8 heads, depth 2) guided by a HalfDiT1d of the same shape"""
    from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE
    from cleandiffuser_b200.nn_diffusion import DiT1d
    from cleandiffuser_b200.testing import load_synth
    clf = dr.make_classifier(dict(in_dim=14, out_dim=1, emb_dim=64, d_model=256, n_heads=8, depth=2), 31, DEV)
    net = load_synth(DiT1d(14, emb_dim=64, d_model=256, n_heads=8, depth=2), seed=41)
    mask = torch.zeros(horizon, 14)
    mask[0] = 1.
    agent = ContinuousDiffusionSDE(net, fix_mask=mask, classifier=clf, predict_noise=False, device=DEV)
    agent.eval()
    prior = torch.zeros(batch, horizon, 14)
    prior[:, 0] = torch.randn(batch, 14, generator=torch.Generator().manual_seed(3))
    return agent, prior.to(DEV)


def planner_call(agent, prior, tape, w_cg=0.1, steps=5):
    with tape.active():
        x0, log = agent.sample(prior, solver="ddpm", n_samples=prior.shape[0], sample_steps=steps, w_cg=w_cg,
                               sample_step_schedule="uniform_continuous")
    torch.cuda.synchronize()
    return x0, log


@pytest.mark.parametrize("math", list(MATHS))
def test_graph_path_against_callback(math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior = planner_agent()
    clf = agent.classifier
    monkeypatch.setattr(clf, "gradients", lambda *a, **k: (_ for _ in ()).throw(AssertionError("callback")))
    tape = NoiseTape()
    x_graph, log = planner_call(agent, prior, tape)
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    monkeypatch.undo()
    dr.register(monkeypatch)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent.classifier = _Wrapped(clf)
    x_cb, log_cb = planner_call(agent, prior, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "callback"
    agent.classifier = clf
    x_free, _ = planner_call(agent, prior, NoiseTape(tape.draws), w_cg=0.0)
    err, effect = float((x_graph - x_cb).abs().max()), float((x_cb - x_free).abs().max())
    # both paths run the same denoiser program; only the classifier gradient differs (the program's operators against PyTorch's
    # fp32 autograd).  To first order a gradient with relative error eps moves x0 by eps times the guidance's effect on x0, D;
    # eps = 1e-5 (fp32) / 1e-2 (TF32) is what test_input_gradient_matches_fp64_autograd holds the gradient to, and twice that
    # covers the second-order terms.  Under TF32 a moved x_t also re-rolls the denoiser's own TF32 rounding in every later step,
    # so the two runs may differ by up to twice the TF32 denoiser's error against fp32, F (measured here with w_cg = 0)
    floor = 1e-5
    if math == "tf32":
        monkeypatch.setenv("CDS_MATH", "fp32")
        x_fp32, _ = planner_call(agent, prior, NoiseTape(tape.draws), w_cg=0.0)
        floor = 2 * float((x_free - x_fp32).abs().max())
    bound = 2 * (1e-5 if math == "fp32" else 1e-2) * effect + floor
    print(f"[half-dit] planner {math}: x0 graph vs callback {err:.3g}, guidance effect {effect:.3g}, bound {bound:.3g}")
    assert effect > 1e-3, "the guidance does not move x0: the comparison shows nothing"
    assert err < bound, (err, bound)
    torch.testing.assert_close(log["log_p"], log_cb["log_p"], rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_goldens_on_the_gpu(name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "fp32")
    G = load_golden("half_dit")
    agent, prior, kw = dr.make_sample_agent(name, device=DEV)
    monkeypatch.setattr(agent.classifier, "gradients", lambda *a, **k: (_ for _ in ()).throw(AssertionError("callback")))
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
    agent, prior = planner_agent(batch=333)
    tape = NoiseTape()
    a, la = planner_call(agent, prior, tape, steps=10)
    b, lb = planner_call(agent, prior, NoiseTape(tape.draws), steps=10)
    monkeypatch.setenv("CDS_GRAPH", "0")
    d, _ = planner_call(agent, prior, NoiseTape(tape.draws), steps=10)
    assert runtime.STATS["guidance_path"] == "graph"
    assert torch.equal(a, b) and torch.equal(a, d) and torch.equal(la["log_p"], lb["log_p"])


@pytest.mark.parametrize("math", list(MATHS))
def test_every_operator_of_the_guided_iteration_matches_fp64(math, monkeypatch):
    """tests/program_audit.py over every iteration of the guided call: each operator within its bound, nothing written outside
    its declared outputs; then whole iterations by graph replay give the operator-by-operator bits"""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent, prior = planner_agent(batch=333)
    planner_call(agent, prior, NoiseTape(), steps=3)
    plan = next(iter(agent._engine_plans.values()))
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    torch.cuda.synchronize()
    start = plan.x.clone()
    aud = pa.Auditor(f"half-dit-{math}", ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    aud.audit_once(0)
    for it in range(n):
        aud.audit_iteration(it)
    for line in pa.report_lines({(aud.name, k): v for k, v in aud.worst.items()}):
        print("[half-dit audit]", line)
    assert not aud.failures, "\n".join(aud.failures[:20])
    assert any(k.startswith("attn_bwd hd 32") for k in aud.worst) and "lnmod_bwd +res +gated" in aud.worst

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
