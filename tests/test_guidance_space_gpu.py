"""The constructor space of the gradient programs (tests/guidance_space.py) on the H100, in fp32 and TF32.

Every lowered classifier case is built at a ragged batch of 333 (partial 32-row DGRAD / WGRAD tiles, partial 8-warp GN
CTAs, two row tiles in every conv_tc launch) and checked three ways:

- every operator of the input-gradient program alone against fp64 under its kernel family's bound, and for writes outside
  its outputs (tests/program_audit.py);
- graph replay and direct launches give the operator-by-operator bits;
- the whole fp32 input gradient against fp64 autograd of this package's module under the per-element bound (GPU_TOL).

Every served ``sample(requires_grad=True)`` case gives its whole fp32 gradients within the per-element bound of fp64
autograd of the PyTorch loop.  Declined classifiers keep the host callback and give its result.  Then
the operator-level forms the lowerings cannot reach: UPDATE_BWD with per-element bounds (min > max, ties), DGRAD / WGRAD
with row strides wider than their operands (NaN gaps), accumulate 0 / 1 and a bias column opening a new 32-column tile, and
GN / GN_BWD with groups of over 1,000 elements, act = NONE and a per-trajectory row.  The module prints the largest error as
a fraction of the bound per (math mode, instantiation) and its wall time."""
import time

import numpy as np
import pytest
import torch

import cg_ref
import emulator
import grad_ref
import guidance_space as gs
import program_audit as pa
import relu_ref
import test_guidance_space_cpu as tc
from cleandiffuser_b200.engine import cabi, lower, runtime
from cleandiffuser_b200.engine.lower import Program, View, lower_classifier_grad
from cleandiffuser_b200.engine.runtime import _Ctx
from cleandiffuser_b200.testing import NoiseTape

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BATCH = 333
MATHS = tc.MATHS
WORST, WHOLE, START = {}, {}, [time.perf_counter()]
LOWERED = [(n, m) for n in tc.LOWERED for m in MATHS]
RUNNABLE_DECLINED = [n for n in tc.DECLINED if gs.CLASSIFIERS[n]["runs"]]
# Per-element tolerance of the whole gradients on the device (guidance_space.per_element_frac).  The kernels sum in other
# orders than the interpreter (which evaluates every operator in fp64 and rounds its stores), and a HalfJannerUNet1d that
# reaches L = 1 early normalises GroupNorm groups of 4 to 32 elements, whose rstd amplifies those differences: 3.8e-4 of
# the gradient's scale at worst in fp32 on an H100.  Under TF32 the same groups amplify the 10-bit operand rounding to the
# order of the gradient itself (0.98 of |ref| + s at worst, HalfJanner horizon 8 over four stages), so the TF32 bound only
# catches a non-finite or grossly wrong gradient; every TF32 operator is held to its own bound by the audit.
GPU_TOL = {"fp32": 1e-3, "tf32": 2.0}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    START[0] = time.perf_counter()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n[guidance space] {torch.cuda.get_device_name(0)}: largest error as a fraction of the bound")
        for line in pa.report_lines(WORST):
            print("[guidance space] " + line)
        worst = sorted(WHOLE.items(), key=lambda kv: -kv[1])[:10]
        print("[guidance space] largest whole-gradient fractions: " + ", ".join(f"{n}-{m} {f:.3f}" for (n, m), f in worst))
        print(f"[guidance space] wall time {time.perf_counter() - START[0]:.1f} s")


@pytest.fixture(autouse=True)
def _engine(monkeypatch):
    relu_ref.register(monkeypatch)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.delenv("CDS_BRANCHES", raising=False)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _stream():
    return torch.cuda.current_stream().cuda_stream


_instantiation = pa.instantiation


def _form(op):
    """the kernel instantiation of ``op`` and, for convolutions, taps / stride / phases and L_in; GN with its group size"""
    inst = _instantiation(op)
    if op.kind == cabi.OP_CONV:
        c = op.u.conv
        inst += f" taps {c.taps} s{c.stride} ph{c.phases} L_in {c.L_in}"
    elif op.kind in (cabi.OP_GN, cabi.OP_GN_BWD):
        g = op.u.gn if op.kind == cabi.OP_GN else op.u.gn_bwd
        inst += " group > 1000" if g.L * g.C // g.groups > 1000 else ""
    return inst


def _record(math, worst, label):
    for inst, (frac, where) in worst.items():
        key = (math, inst)
        if frac > WORST.get(key, (-1.0, ""))[0]:
            WORST[key] = (frac, f"{label} {where}")


@pytest.mark.parametrize("name,math", LOWERED)
def test_lowered_classifier_gradient(name, math, monkeypatch):
    case = gs.CLASSIFIERS[name]
    clf = gs.build_classifier(case, device=DEV)
    x, c = gs.classifier_inputs(case, BATCH, device=DEV)
    assert lower.guidable(clf, case["x"], c) is None
    t_all = tc.T_ALL.to(DEV)
    B, H, D = x.shape if x.dim() == 3 else (x.shape[0], 1, x.shape[1])
    p = Program(torch.device(DEV), B, len(t_all), MATHS[math])
    xb = p.buf(*x.shape)
    xb.copy_(x)
    g = lower_classifier_grad(p, clf, View(xb, H, D))
    with torch.no_grad():
        for fn in p.per_call:
            fn(_Ctx(t_all, None, c))
    handle = runtime._make_handle(torch.device(DEV), p.ops, len(t_all))
    st = _stream()
    torch.cuda.synchronize()

    # every operator of iteration 1 against fp64, and no write outside its outputs
    monkeypatch.setattr(pa, "instantiation", _form)
    aud = pa.Auditor(f"{name}-{math}", p.ops, handle, list(p.keep), st, torch.cuda.synchronize)
    aud.audit_iteration(1)
    _record(math, aud.worst, name)
    assert not aud.failures, "\n".join(aud.failures[:20])

    # the whole gradient of iteration 1 (the audit ran it operator by operator) against fp64 autograd
    got = g.t.view(B, H, -1)[..., :D].reshape(x.shape).clone()
    want = gs.input_gradient_fp64(clf, case, x, t_all[1].expand(B), c).to(DEV)
    frac, where = gs.per_element_frac(got, want, math, GPU_TOL)
    WHOLE[(name, math)] = frac
    assert frac <= 1.0, (name, case["ctor"], frac, where)

    # graph replay and direct launches give the operator-by-operator bits
    mem = emulator.Owned(list(p.keep))
    written = [mem.owners[i] for i in pa.written_owners(mem, p.ops, [1])]
    outs = None
    for mode in ("op by op", "graph", "direct"):
        for t in written:
            t.fill_(float("nan"))
        torch.cuda.synchronize()
        if mode == "op by op":
            pa.run_op_by_op(handle, p.ops, 1, 1, st, torch.cuda.synchronize)
        else:
            handle.run(1, 1, st, mode == "graph")
        torch.cuda.synchronize()
        if outs is None:
            outs = [t.clone() for t in written]
            continue
        diff = [f"{tuple(t.shape)}" for t, o in zip(written, outs) if not pa.same_bits(t, o)]
        assert not diff, f"{mode}: {len(diff)} buffers differ from the operator-by-operator run: {diff[:8]}"


@pytest.mark.parametrize("name,math", [(n, m) for n in tc.LOWERED if gs.CLASSIFIERS[n]["runs"] for m in MATHS])
def test_guided_iteration(name, math, monkeypatch):
    """a guided sample() with the case's classifier inside the replayed loop: every operator of one whole iteration (the
    denoiser, the classifier's input gradient, CDS_OP_GUIDE and the update) against fp64, writes outside the outputs
    included"""
    case = gs.CLASSIFIERS[name]
    monkeypatch.setenv("CDS_MATH", math)
    clf = gs.build_classifier(case, device=DEV)
    _, c = gs.classifier_inputs(case, BATCH, device=DEV)
    agent, obs = tc.guided_agent(case, clf, DEV)
    torch.manual_seed(5)
    tc.guided_sample(agent, obs, BATCH, c, NoiseTape(), DEV, x_shape=case["x"])
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    (plan,) = agent._engine_plans.values()
    ops, st = plan.program.ops, _stream()
    assert cabi.OP_GUIDE in {op.kind for op in ops}
    torch.cuda.synchronize()
    monkeypatch.setattr(pa, "instantiation", _form)
    aud = pa.Auditor(f"{name}-{math} guided", ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    plan.x.copy_(torch.randn(plan.x.shape, generator=torch.Generator().manual_seed(7)).to(DEV).clamp(-1, 1))
    aud.audit_once(0)
    aud.audit_iteration(0)
    _record(math, aud.worst, name)
    assert not aud.failures, "\n".join(aud.failures[:20])


@pytest.mark.parametrize("name", RUNNABLE_DECLINED)
def test_declined_classifier_keeps_the_callback(name, monkeypatch):
    case = gs.CLASSIFIERS[name]
    monkeypatch.setenv("CDS_MATH", "fp32")
    clf = gs.build_classifier(case, device=DEV)
    _, c = gs.classifier_inputs(case, BATCH, device=DEV)
    agent, obs = tc.guided_agent(case, clf, DEV)
    tape = NoiseTape()
    got = tc.guided_sample(agent, obs, BATCH, c, tape, DEV, x_shape=case["x"])
    assert runtime.STATS["guidance_path"] == "callback" and runtime.STATS["guidance_reason"] == case["want"]
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want = tc.guided_sample(agent, obs, BATCH, c, NoiseTape(tape.draws), DEV, x_shape=case["x"])
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)


def test_more_than_one_chain_takes_the_pytorch_loop(monkeypatch):
    """CDS_BRANCHES = 2 splits the batch into two sub-batch chains: the classifier is not lowered (its reason is recorded),
    and the host callback needs a single chain, so the guided call takes the PyTorch loop and gives its result"""
    monkeypatch.setenv("CDS_MATH", "fp32")
    monkeypatch.setenv("CDS_BACKEND", "auto")
    monkeypatch.setenv("CDS_BRANCHES", "2")
    monkeypatch.setenv("CDS_BRANCH_MIN_BATCH", "1")
    case, _ = tc._request_agent()
    clf = gs.build_classifier(case, device=DEV)
    _, c = gs.classifier_inputs(case, 8, device=DEV)
    agent, obs = tc.guided_agent(case, clf, DEV)
    calls, tape = runtime.STATS["engine_calls"], NoiseTape()
    got = tc.guided_sample(agent, obs, 8, c, tape, DEV, x_shape=case["x"])
    assert runtime.STATS["guidance_reason"] == gs.REQUESTS["branches"] and runtime.STATS["engine_calls"] == calls
    assert runtime.STATS["last_fallback_reason"] == "guided sampling needs a single-branch program with a dense prediction buffer"
    monkeypatch.setenv("CDS_BACKEND", "torch")
    want = tc.guided_sample(agent, obs, 8, c, NoiseTape(tape.draws), DEV, x_shape=case["x"])
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name,math", [(n, m) for n in tc.GRAD_SERVED for m in MATHS])
def test_grad_sampling(name, math, monkeypatch):
    """the whole gradients against fp64 autograd of the PyTorch loop; then every operator of every forward and backward
    iteration of the plan that served the call (program audit, writes outside the outputs included), and both programs'
    whole iterations give the operator-by-operator bits by graph replay and by direct launches"""
    fracs, agent = tc.check_grad_case(name, math, DEV, BATCH, monkeypatch, GPU_TOL)
    worst = max(fracs, key=fracs.get)
    WHOLE[(name, math)] = fracs[worst]
    assert fracs[worst] <= 1.0, (name, gs.GRADS[name], worst, fracs[worst])

    (plan,) = agent._engine_plans.values()
    st = _stream()
    torch.cuda.synchronize()
    monkeypatch.setattr(pa, "instantiation", _form)
    fa, ba = pa.audit_grad_plan(f"{name}-{math}", plan, plan.handle, plan.back_handle, st, torch.cuda.synchronize)
    _record(math, fa.worst, name)
    _record(math, ba.worst, name)
    assert not fa.failures and not ba.failures, "\n".join((fa.failures + ba.failures)[:20])

    n = plan.n_iters
    mem = emulator.Owned(pa.plan_owners(plan))
    start = torch.randn(plan.x.shape, generator=torch.Generator().manual_seed(17)).to(DEV)
    for ops, handle, forward in ((plan.program.ops, plan.handle, True), (plan.back.ops, plan.back_handle, False)):
        written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(n))]
        if forward:
            plan.x.copy_(start)
        else:
            pa.seed_backward(plan, 3)
        torch.cuda.synchronize()
        snap = [t.clone() for t in written]
        outs = None
        for mode in ("op by op", "graph", "direct"):
            for t, s_ in zip(written, snap):
                t.copy_(s_)
            if mode == "op by op":
                pa.run_op_by_op(handle, ops, 0, n, st, torch.cuda.synchronize)
            else:
                handle.run(0, n, st, mode == "graph")
            torch.cuda.synchronize()
            if outs is None:
                outs = [t.clone() for t in written]
                continue
            diff = [f"{tuple(t.shape)}" for t, o in zip(written, outs) if not pa.same_bits(t, o)]
            assert not diff, f"{'forward' if forward else 'backward'} {mode}: {len(diff)} buffers differ: {diff[:8]}"


@pytest.mark.parametrize("name", tc.GRAD_DECLINED)
def test_declined_grad_request_takes_the_pytorch_loop(name, monkeypatch):
    tc.check_grad_decline(name, DEV, BATCH, monkeypatch)


# ================================================================================ operator forms the lowerings cannot reach
def _run(op, it=0):
    cabi.run_op(0, op, it, _stream())
    torch.cuda.synchronize()


def _frac(got, want, bound):
    err = np.abs(np.asarray(got, np.float64) - want)
    return float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), np.where(err > 0, np.inf, 0.0))))


def _note(inst, frac):
    key = ("fp32", inst)
    if frac > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (frac, "operator test")


@pytest.mark.parametrize("predict_noise", [True, False])
@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_update_bwd_per_element_bounds(kind, predict_noise):
    """per-element, non-uniform x_min / x_max / mask with min > max in two elements and exact ties, 333 rows, against fp64
    autograd of torch.clip with tensor bounds"""
    B, A = 333, 7
    g = torch.Generator().manual_seed(11 + kind)
    x = torch.randn(B, A, generator=g, dtype=torch.float64).float()
    pred = (torch.randn(B, A, generator=g) * 2)
    gx = torch.randn(B, A, generator=g)
    x_min = torch.tensor([-0.9, -0.5, 0.1, -1.2, 0.4, -0.3, -0.7])
    x_max = torch.tensor([0.8, 0.2, 0.6, 1.1, -0.1, 0.9, -0.8])        # elements 4 and 6: min > max
    mask = torch.tensor([0., 1., 0., 0., 1., 0., 0.])
    alpha, sigma, k0, k1 = 0.7, 0.55, 1.2, 0.35
    a32, s32 = torch.tensor(alpha, dtype=torch.float32), torch.tensor(sigma, dtype=torch.float32)
    if predict_noise:                       # fp32 as the kernel evaluates the bounds
        lo, hi = (x - a32 * x_max) / s32, (x - a32 * x_min) / s32
    else:
        lo, hi = x_min.expand(B, A), x_max.expand(B, A)
    pred[:40] = lo[:40]
    pred[40:80] = hi[40:80]                 # exact ties with either bound
    coef = torch.zeros(1, cabi.ROW_FLOATS)
    coef[0, :4] = torch.tensor([alpha, sigma, k0, k1])
    coef[0, 7] = float(kind)
    d = {k: v.to(DEV).contiguous() for k, v in dict(gx=gx.clone(), gp=torch.zeros_like(gx), x=x, p=pred, m=mask, lo=x_min,
                                                      hi=x_max, c=coef).items()}
    op = cabi.Op()
    op.kind = cabi.OP_UPDATE_BWD
    u = op.u.update_bwd
    u.batch, u.row, u.gx, u.gpred, u.x, u.pred = B, A, d["gx"].data_ptr(), d["gp"].data_ptr(), d["x"].data_ptr(), d["p"].data_ptr()
    u.mask, u.x_min, u.x_max, u.coef, u.predict_noise = (d["m"].data_ptr(), d["lo"].data_ptr(), d["hi"].data_ptr(),
                                                         d["c"].data_ptr(), int(predict_noise))
    _run(op)

    # fp64 autograd of the update with torch.clip(pred, lo, hi) (tensor bounds, evaluated as the kernel takes its decisions)
    x64, p64 = x.double().requires_grad_(True), pred.double().requires_grad_(True)
    if predict_noise:
        lo_t, hi_t = (x64 - alpha * x_max.double()) / sigma, (x64 - alpha * x_min.double()) / sigma
        lo_t = lo_t + (lo.double() - lo_t).detach()           # the decisions on the fp32 bounds, the gradient through x
        hi_t = hi_t + (hi.double() - hi_t).detach()
        eps = p64.clip(lo_t, hi_t)
        xhat = (x64 - sigma * eps) / alpha
    else:
        xhat = p64.clip(x_min.double(), x_max.double())
        eps = (x64 - alpha * xhat) / sigma
    out = [k0 * (x64 - sigma * eps) + k1 * eps, k0 * (x64 - sigma * eps) / alpha + k1 * eps, k0 * x64 - k1 * eps,
           k0 * x64 - k1 * xhat][kind]
    (out * (gx.double() * (1 - mask.double()))).sum().backward()
    bound = grad_ref.update_bwd_bound(gx.numpy(), alpha, sigma, k0, k1)
    fp = _frac(d["gp"].cpu().numpy(), p64.grad.numpy(), bound)
    fx = _frac(d["gx"].cpu().numpy(), x64.grad.numpy(), bound)
    _note("update_bwd per-element bounds", max(fp, fx))
    assert fp <= 1.0 and fx <= 1.0, (fp, fx)


def _gapped(rows, cols, ld, g, scale=1.0):
    """(rows + 1, ld) fp32 with NaN in the gap columns and the extra row; the (rows, cols) operand in front"""
    t = torch.full((rows + 1, ld), float("nan"))
    t[:rows, :cols] = torch.randn(rows, cols, generator=g) * scale
    return t


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("act", ["none", "relu", "silu", "mish"])
@pytest.mark.parametrize("rows,N,K", [(333, 33, 64), (61, 100, 7), (32, 256, 96)])
def test_dgrad_strided_operands(rows, N, K, act, accumulate):
    """out = (dz W) act'(z) [+ out] with ldz, ldw, ldo wider than the operands: every gap and the row after the output
    stay NaN"""
    g = torch.Generator().manual_seed(rows + N + K)
    a = {"none": cabi.ACT_NONE, "relu": cabi.ACT_RELU, "silu": cabi.ACT_SILU, "mish": cabi.ACT_MISH}[act]
    dz, w = _gapped(rows, N, N + 5, g), _gapped(N, K, K + 3, g, 1 / np.sqrt(N))
    out = _gapped(rows, K, K + 9, g)
    z = torch.randn(rows, K, generator=g) * 2
    before = out.clone()
    d = {k: v.to(DEV) for k, v in dict(dz=dz, w=w, out=out, z=z).items()}
    op = cabi.Op()
    op.kind = cabi.OP_DGRAD
    q = op.u.dgrad
    q.rows, q.N, q.K, q.dz, q.ldz, q.w, q.ldw = rows, N, K, d["dz"].data_ptr(), N + 5, d["w"].data_ptr(), K + 3
    if a != cabi.ACT_NONE:
        q.z, q.z_iter_stride, q.act = d["z"].data_ptr(), 0, a
    q.accumulate, q.out, q.ldo = accumulate, d["out"].data_ptr(), K + 9
    _run(op)
    res = d["out"].cpu()
    zz = z.double().numpy() if a != cabi.ACT_NONE else None
    y = grad_ref.dgrad(dz[:rows, :N].numpy(), w[:N, :K].numpy(), zz, a)
    prev = before[:rows, :K].double().numpy() if accumulate else None
    want = y if prev is None else prev + y
    bound = grad_ref.dgrad_bound(dz[:rows, :N].numpy(), w[:N, :K].numpy(), zz, a, prev)
    f = _frac(res[:rows, :K].numpy(), want, bound)
    _note(f"dgrad {act} strided", f)
    assert f <= 1.0, f
    assert torch.isnan(res[:rows, K:]).all() and torch.isnan(res[rows]).all(), "dgrad wrote into a gap"


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("rows,N,K", [(333, 33, 64), (61, 100, 7), (1000, 32, 32)])
def test_wgrad_strided_operands(rows, N, K, bias, accumulate):
    """dw [+]= dz^T act(h), db [+]= sum dz with ldz, ldh, lddw wider than the operands (K = 32 and 64: the bias column, in
    the same row of dw's buffer layout as the weights' K columns, opens a new 32-column tile); gaps and the row after dw stay
    NaN"""
    g = torch.Generator().manual_seed(rows * 3 + N + K)
    dz, h = _gapped(rows, N, N + 4, g), _gapped(rows, K, K + 6, g)
    dw = _gapped(N, K, K + 8, g)
    db = torch.full((N + 1,), float("nan"))
    db[:N] = torch.randn(N, generator=g)
    w0, b0 = dw.clone(), db.clone()
    d = {k: v.to(DEV) for k, v in dict(dz=dz, h=h, dw=dw, db=db).items()}
    op = cabi.Op()
    op.kind = cabi.OP_WGRAD
    q = op.u.wgrad
    q.rows, q.N, q.K, q.dz, q.ldz = rows, N, K, d["dz"].data_ptr(), N + 4
    q.h, q.h_iter_stride, q.ldh, q.act = d["h"].data_ptr(), 0, K + 6, cabi.ACT_MISH
    q.dw, q.lddw, q.accumulate = d["dw"].data_ptr(), K + 8, accumulate
    if bias:
        q.db, q.db_iter_stride = d["db"].data_ptr(), 0
    _run(op)
    gw, gb = grad_ref.wgrad(dz[:rows, :N].numpy(), h[:rows, :K].numpy(), cabi.ACT_MISH)
    pw = w0[:N, :K].double().numpy() if accumulate else None
    pb = b0[:N].double().numpy() if accumulate else None
    bw, bb = grad_ref.wgrad_bound(dz[:rows, :N].numpy(), h[:rows, :K].numpy(), cabi.ACT_MISH, pw, pb)
    res, rb = d["dw"].cpu(), d["db"].cpu()
    f = _frac(res[:N, :K].numpy(), gw if pw is None else pw + gw, bw)
    _note(f"wgrad mish strided{' + bias' if bias else ''}", f)
    assert f <= 1.0, f
    assert torch.isnan(res[:N, K:]).all() and torch.isnan(res[N]).all(), "wgrad wrote into a gap"
    if bias:
        fb = _frac(rb[:N].numpy(), gb if pb is None else pb + gb, bb)
        _note("wgrad bias column", fb)
        assert fb <= 1.0, fb
    else:
        assert torch.equal(rb[:N], b0[:N]), "wgrad wrote a bias row it was not given"
    assert torch.isnan(rb[N]), "wgrad wrote past the bias row"


@pytest.mark.parametrize("act", [cabi.ACT_MISH, cabi.ACT_NONE])
@pytest.mark.parametrize("L,C", [(256, 32), (128, 64), (5, 12)])
def test_gn_large_groups_and_sample_rows(L, C, act):
    """GN with a per-trajectory vec row and GN_BWD, groups of L C / groups elements (256 x 32 / 8 = 1024), act NONE and Mish,
    333 trajectories, against cg_ref.gn / gn_bwd under their bounds"""
    B, groups = 333, min(8, C // 4)
    g = torch.Generator().manual_seed(L * C + act)
    h = torch.randn(B, L, C, generator=g) * 1.5 + 0.3
    gamma, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    row = torch.randn(B, C, generator=g)
    dout = torch.randn(B, L, C, generator=g)
    d = {k: v.to(DEV) for k, v in dict(h=h, gamma=gamma, beta=beta, row=row, dout=dout, out=torch.zeros(B, L, C),
                                       dh=torch.zeros(B, L, C)).items()}
    op = cabi.Op()
    op.kind = cabi.OP_GN
    q = op.u.gn
    q.batch, q.L, q.C, q.groups, q.eps, q.act = B, L, C, groups, 1e-5, act
    q.h, q.h_bstride, q.h_lstride = d["h"].data_ptr(), L * C, C
    q.gamma, q.beta = d["gamma"].data_ptr(), d["beta"].data_ptr()
    q.vec = cabi_vec(d["row"])
    q.out, q.out_bstride, q.out_lstride, q.out_dtype = d["out"].data_ptr(), L * C, C, cabi.F32
    _run(op)
    ref = cg_ref.gn(h, gamma, beta, groups, 1e-5, act, vec=row)
    bound = cg_ref.gn_bound(h, gamma, beta, groups, 1e-5, ref, act, vec=row)
    f = _frac(d["out"].cpu().numpy(), ref.numpy(), bound.numpy())
    big = " group > 1000" if L * C // groups > 1000 else ""
    _note(f"gn act {act} + sample row{big}", f)
    assert f <= 1.0, f
    op = cabi.Op()
    op.kind = cabi.OP_GN_BWD
    q = op.u.gn_bwd
    q.batch, q.L, q.C, q.groups, q.eps, q.act = B, L, C, groups, 1e-5, act
    q.h, q.h_bstride, q.h_lstride = d["h"].data_ptr(), L * C, C
    q.gamma, q.beta = d["gamma"].data_ptr(), d["beta"].data_ptr()
    q.dout, q.dout_bstride, q.dout_lstride = d["dout"].data_ptr(), L * C, C
    q.dh, q.dh_bstride, q.dh_lstride, q.dh_dtype = d["dh"].data_ptr(), L * C, C, cabi.F32
    _run(op)
    ref = cg_ref.gn_bwd(h, gamma, beta, dout, groups, 1e-5, act)
    bound = cg_ref.gn_bwd_bound(h, gamma, beta, dout, groups, 1e-5, ref, act)
    f = _frac(d["dh"].cpu().numpy(), ref.numpy(), bound.numpy())
    _note(f"gn_bwd act {act}{big}", f)
    assert f <= 1.0, f


def cabi_vec(sample_rows):
    """a cabi.Vec of one (batch, C) per-trajectory row"""
    from cleandiffuser_b200.engine.lower import _vec
    return _vec(sample=sample_rows)
