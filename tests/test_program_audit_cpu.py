"""The machinery of tests/test_program_audit_gpu.py without a GPU: the same auditor drives the interpreter's handle
(tests/emulator.py, tests/mha_ref.py) over programs lowered for CPU tensors, at small batches.  The interpreter computes
what the fp64 reference computes, so every operator must pass with a fraction at most the half unit of the stored rounding;
three injected faults must be caught and pinned on the right operator."""
import pytest
import torch

import chi_cases as cc
import emulator
import mha_ref
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
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: mha_ref.Handle(ops, n, owners()))
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
    """the plan's handle, with ``fault(op)`` applied right after operator ``j`` ran"""

    def __init__(self, inner, ops, j, fault):
        self.inner, self.ops, self.j, self.fault = inner, ops, j, fault

    def run(self, *a):
        self.inner.run(*a)

    def run_range(self, it, i, n, stream):
        self.inner.run_range(it, i, n, stream)
        if i <= self.j < i + n:
            self.fault(self.ops[self.j])

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

    def corrupt(op):
        out = emulator.view(mem, *pa.declared_outputs(op)[0])
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

    def past(op):
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
