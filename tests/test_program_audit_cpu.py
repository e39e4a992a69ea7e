"""The machinery of tests/test_program_audit_gpu.py without a GPU: the same auditor drives the interpreter's handle
(tests/emulator.py) over programs lowered for CPU tensors, at small batches.  The interpreter computes what the fp64
reference computes, so every operator must pass with a fraction at most the half unit of the stored rounding; injected
faults must be caught and pinned on the right operator.  The faults of the classifier-guided and differentiable programs
are subtly wrong kernels run in place of one operator."""
import pytest
import torch

import cg_ref
import chi_cases as cc
import emulator
import grad_ref
import opref
import program_audit as pa
from cleandiffuser_b200 import workloads
from cleandiffuser_b200.diffusion import DDPM
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import ChiTransformer
from cleandiffuser_b200.testing import synth_state_dict

# the interpreter stores the rounding of the exact value: half a unit of TF32 (bound 2^-10 |ref|) at most
PASS_FRAC = 0.5 + 1e-3


@pytest.fixture(autouse=True)
def _emulate(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "tf32")


def _cfg2_plan(monkeypatch, branches=1):
    monkeypatch.setenv("CDS_BRANCHES", str(branches))
    monkeypatch.setenv("CDS_BRANCH_MIN_BATCH", "1")
    w = workloads.cfg2("cpu", batch=8, steps=3)
    with torch.no_grad():
        w.sample("cpu")
    plan = next(iter(w.agent._engine_plans.values()))
    assert plan.n_branches == branches
    return plan


def _chi_plan():
    ctor = dict(cc.NETS["kitchen"], d_model=192, nhead=1, num_layers=2)      # kitchen's head_dim 192, CPU-sized
    net = ChiTransformer(**ctor)
    net.load_state_dict(cc.weights(net.state_dict(), synth_state_dict))
    x_max = torch.ones((1, ctor["Ta"], ctor["act_dim"]))
    agent = DDPM(net.eval(), IdentityCondition(dropout=0.0), x_max=x_max, x_min=-x_max, diffusion_steps=3, device="cpu")
    g = torch.Generator().manual_seed(5)
    cond = torch.randn(3, ctor["To"], ctor["obs_dim"], generator=g)
    with torch.no_grad():
        agent.sample(torch.zeros(3, ctor["Ta"], ctor["act_dim"]), n_samples=3, sample_steps=3, condition_cfg=cond, w_cfg=1.0)
    return next(iter(agent._engine_plans.values()))


def _audit(plan, handle=None, iters=(0, 1)):
    aud = pa.Auditor("cpu", plan.program.ops, handle or plan.handle, pa.plan_owners(plan))
    plan.x.copy_(torch.randn(plan.x.shape, generator=torch.Generator().manual_seed(0)))
    aud.audit_once(0)
    for it in iters:
        aud.audit_iteration(it)
    return aud


class _Faulty:
    """the plan's handle, with ``fault(op, it)`` applied right after operator ``j`` ran, or run in its place (``replace``: a
    wrong kernel)"""

    def __init__(self, inner, ops, j, fault, replace=False):
        self.inner, self.ops, self.j, self.fault, self.replace = inner, ops, j, fault, replace

    def run(self, *a):
        self.inner.run(*a)

    def run_range(self, it, i, n, stream):
        if not (i <= self.j < i + n):
            self.inner.run_range(it, i, n, stream)
            return
        if not self.replace:
            self.inner.run_range(it, i, n, stream)
            self.fault(self.ops[self.j], it)
            return
        if self.j > i:
            self.inner.run_range(it, i, self.j - i, stream)
        self.fault(self.ops[self.j], it)
        if i + n > self.j + 1:
            self.inner.run_range(it, self.j + 1, i + n - self.j - 1, stream)

    def launches_per_iter(self):
        return self.inner.launches_per_iter()


@pytest.mark.parametrize("which", ["cfg2", "chi"])
def test_every_operator_passes(which, monkeypatch):
    plan = _cfg2_plan(monkeypatch) if which == "cfg2" else _chi_plan()
    aud = _audit(plan)
    assert not aud.failures, aud.failures[:5]
    kinds = {op.kind for op in plan.program.ops}
    assert {cabi.OP_CONV, cabi.OP_UPDATE} <= kinds and (which == "cfg2" or {cabi.OP_MHA, cabi.OP_LNMOD} <= kinds)
    assert aud.worst and max(f for f, _ in aud.worst.values()) <= PASS_FRAC, aud.worst


def test_a_corrupted_element_is_pinned_on_its_operator(monkeypatch):
    plan = _chi_plan()
    ops = plan.program.ops
    j = [i for i, op in enumerate(ops) if op.kind == cabi.OP_MHA][-1]
    mem = emulator.Owned(pa.plan_owners(plan))

    def corrupt(op, it):
        out = emulator.view(mem, *pa.declared_outputs(op, it)[0])
        # an error of 2|y| + 1: 2^11 times the 2^-10 |ref| rounding term of the TF32 output, and, with these O(1) values, far
        # above the accumulation terms of the bound; finite, so that the operators downstream see an ordinary input
        out[-1, 3, 5] = -out[-1, 3, 5] - 1
    aud = _audit(plan, _Faulty(plan.handle, ops, j, corrupt), iters=(1,))
    assert aud.failures and all(f"op {j} " in m for m in aud.failures), aud.failures[:5]
    assert min(frac for frac, where in aud.worst.values() if f"op {j} " in where) > 100, aud.worst


def test_a_write_one_row_past_the_output_is_flagged(monkeypatch):
    plan = _cfg2_plan(monkeypatch, branches=2)
    ops = plan.program.ops
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_UPDATE)        # branch 0's update: x rows [0, 4)
    mem = emulator.Owned(pa.plan_owners(plan))

    def past(op, it):
        u = op.u.update
        row_past = emulator.view(mem, u.x + 4 * u.batch * u.row, (u.row,), (1,), cabi.F32)   # branch 1's first row
        row_past += 1.0
    aud = _audit(plan, _Faulty(plan.handle, ops, j, past), iters=(0,))
    assert aud.failures and all(f"op {j} " in m and "outside the declared outputs" in m for m in aud.failures), \
        aud.failures[:5]


def test_the_extent_check_rejects_a_stride_past_the_owner(monkeypatch):
    plan = _cfg2_plan(monkeypatch)
    mem = emulator.Owned(pa.plan_owners(plan))
    op = next(op for op in plan.program.ops if op.kind == cabi.OP_CONV)
    emulator.conv_operands(op.u.conv, 0, mem)
    bad = cabi.Op.from_buffer_copy(op)
    bad.u.conv.out_bstride += bad.u.conv.L_out * bad.u.conv.phases * bad.u.conv.C_out    # one row per trajectory too far
    with pytest.raises(AssertionError, match="past its owner"):
        emulator.conv_operands(bad.u.conv, 0, mem)


# ---- classifier guidance and differentiable sampling (tests/cg_ref.py, tests/grad_ref.py) -----------------------------------
def _guided_plan(monkeypatch, math_mode):
    """a guided sample() of tests/golden/make_golden_classifier.py (horizon 8, batch 8, 5 DDPM steps), classifier lowered"""
    monkeypatch.setenv("CDS_MATH", math_mode)
    agent, prior, kw = cg_ref.make_sample_agent("discrete_ddpm_eps")
    agent.sample(prior, **kw)
    assert runtime.STATS["guidance_path"] == "graph"
    (plan,) = agent._engine_plans.values()
    return plan


def _grad_plan(monkeypatch, case, math_mode="tf32", batch=16):
    monkeypatch.setenv("CDS_MATH", math_mode)
    agent, kw = grad_ref.grad_agent(case, "cpu")
    g = torch.Generator().manual_seed(2)
    obs, act = grad_ref.GRAD_CASES[case]["net"]["obs_dim"], grad_ref.GRAD_CASES[case]["net"]["act_dim"]
    agent.sample(torch.randn(batch, act, generator=g), n_samples=batch, condition_cfg=torch.randn(batch, obs, generator=g), **kw)
    (plan,) = agent._engine_plans.values()
    assert isinstance(plan, runtime.GradSamplerPlan) and plan.n_iters == 5
    return plan


def _grad_audit(plan, back=None):
    plan.x.copy_(torch.randn(plan.x.shape, generator=torch.Generator().manual_seed(0)))
    return pa.audit_grad_plan("cpu", plan, plan.handle, back or plan.back_handle)


@pytest.mark.parametrize("math_mode", ["fp32", "tf32"])
def test_guided_program_every_operator_passes(math_mode, monkeypatch):
    plan = _guided_plan(monkeypatch, math_mode)
    aud = _audit(plan, iters=(0, 1, plan.n_iters - 1))
    assert not aud.failures, aud.failures[:5]
    kinds = {op.kind for op in plan.program.ops}
    assert {cabi.OP_GN, cabi.OP_GN_BWD, cabi.OP_GUIDE, cabi.OP_DGRAD} <= kinds
    names = set(aud.worst)
    assert {"guide", "dgrad", "dgrad mish", f"gn +vec -> {math_mode[:4].replace('fp32', 'f32')}"} <= names, names
    assert aud.worst and max(f for f, _ in aud.worst.values()) <= PASS_FRAC, aud.worst


@pytest.mark.parametrize("case", list(grad_ref.GRAD_CASES))
@pytest.mark.parametrize("math_mode", ["fp32", "tf32"])
def test_grad_programs_every_operator_passes(case, math_mode, monkeypatch):
    plan = _grad_plan(monkeypatch, case, math_mode)
    fa, ba = _grad_audit(plan)
    assert not fa.failures and not ba.failures, (fa.failures + ba.failures)[:5]
    assert {"stash", "stash +act"} <= set(fa.worst), fa.worst
    assert {"wgrad +bias", "wgrad mish +bias", "dgrad +=", "dgrad mish", "dgrad mish +out_sum"} <= set(ba.worst), ba.worst
    assert any(n.startswith("update_bwd") for n in ba.worst)
    worst = list(fa.worst.values()) + list(ba.worst.values())
    assert max(f for f, _ in worst) <= PASS_FRAC, (fa.worst, ba.worst)


def _pinned(failures, j, tag=""):
    return failures and all(f"op {j} " in m and tag in m for m in failures)


def test_gn_variance_over_n_minus_1_is_caught(monkeypatch):
    plan = _guided_plan(monkeypatch, "fp32")
    ops, mem = plan.program.ops, plan.handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_GN)
    stats = cg_ref._stats

    def stats_unbiased(h, groups, eps):
        g, mean, _ = stats(h, groups, eps)
        n = g.shape[1] * g.shape[3]
        var = ((g - mean) ** 2).sum(dim=(1, 3), keepdim=True) / (n - 1)
        return g, mean, 1.0 / torch.sqrt(var + eps)

    def gn_unbiased(op, it):
        with monkeypatch.context() as m:
            m.setattr(cg_ref, "_stats", stats_unbiased)
            emulator.run_gn(op.u.gn, it, mem)
    aud = _audit(plan, _Faulty(plan.handle, ops, j, gn_unbiased, replace=True), iters=(1,))
    assert _pinned(aud.failures, j), aud.failures[:5]


def test_gn_time_row_of_iteration_0_is_caught(monkeypatch):
    plan = _guided_plan(monkeypatch, "tf32")
    ops, mem = plan.program.ops, plan.handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_GN and op.u.gn.vec.step)
    aud = _audit(plan, _Faulty(plan.handle, ops, j, lambda op, it: emulator.run_gn(op.u.gn, 0, mem), replace=True), iters=(0, 1))
    assert _pinned(aud.failures, j) and all(m.startswith("cpu it 1 ") for m in aud.failures), aud.failures[:5]


def test_downsample_data_gradient_with_a_circular_halo_is_caught(monkeypatch):
    """dx[2m+1] = W2^T d[m] + W0^T d[m+1]: at the last position d[m+1] is past the end (zero); a circular halo reads d[0]"""
    plan = _guided_plan(monkeypatch, "tf32")
    ops, mem = plan.program.ops, plan.handle.mem
    first_gn = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_GN)
    j = max(i for i, op in enumerate(ops) if op.kind == cabi.OP_CONV and op.u.conv.phases == 2)
    assert j > first_gn and ops[j].u.conv.L_out >= 2                   # the classifier's, not the denoiser's up-sampling

    def wrap(op, it):
        c = op.u.conv
        emulator.run_conv(c, it, mem)
        x, w, _, out = emulator.conv_operands(c, it, mem)             # w: (taps, C_in, C_out * phases)
        halo = (x[:, 0].double() @ w[2].double()).reshape(c.batch, c.phases, c.C_out)
        out[:, -c.phases:] = opref.store(out[:, -c.phases:].double() + halo, c.out_dtype).to(out.dtype)
    aud = _audit(plan, _Faulty(plan.handle, ops, j, wrap, replace=True), iters=(1,))
    assert _pinned(aud.failures, j), aud.failures[:5]


def test_dgrad_reading_the_forward_slot_of_its_own_index_is_caught(monkeypatch):
    """backward iteration m must read the stash of forward iteration n_iters - 1 - m"""
    plan = _grad_plan(monkeypatch, "dql-eps")
    ops, mem = plan.back.ops, plan.back_handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_DGRAD and op.u.dgrad.z)

    def forward_order(op, it):
        bad = cabi.Op.from_buffer_copy(op)
        d = bad.u.dgrad
        d.z, d.z_iter_stride = d.z + 4 * (plan.n_iters - 1) * d.z_iter_stride, -d.z_iter_stride
        emulator.run_dgrad(d, it, mem)
    fa, ba = _grad_audit(plan, _Faulty(plan.back_handle, ops, j, forward_order, replace=True))
    assert not fa.failures and _pinned(ba.failures, j, "bwd"), (fa.failures + ba.failures)[:5]
    # the middle iteration reads its own slot either way (at the last one, forward iteration 0, the clip to [-1, 1] at
    # alpha ~ 0 sends the whole gradient to x_t: d pred = 0)
    its = {m.split(" op ")[0] for m in ba.failures}
    assert {"cpu bwd it 0", "cpu bwd it 1", "cpu bwd it 3"} <= its and "cpu bwd it 2" not in its, its


def test_wgrad_bias_into_the_neighbouring_row_is_flagged(monkeypatch):
    plan = _grad_plan(monkeypatch, "dql-x0")
    ops, mem = plan.back.ops, plan.back_handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_WGRAD and op.u.wgrad.db_iter_stride)

    def neighbour(op, it):
        bad = cabi.Op.from_buffer_copy(op)
        g = bad.u.wgrad
        g.db += 4 * (1 if it < plan.n_iters - 1 else -1) * g.db_iter_stride
        emulator.run_wgrad(g, it, mem)
    fa, ba = _grad_audit(plan, _Faulty(plan.back_handle, ops, j, neighbour, replace=True))
    assert not fa.failures and _pinned(ba.failures, j, "bwd"), (fa.failures + ba.failures)[:5]
    assert any("outside the declared outputs" in m for m in ba.failures), ba.failures[:5]
