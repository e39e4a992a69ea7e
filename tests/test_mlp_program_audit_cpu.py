"""The MLP denoiser programs of tests/mlp_programs.py at CPU sizes on the interpreter (tests/emulator.py): every operator
passes the per-operator audit, the lowered denoiser matches the fp64 module, and four injected faults -- three in an
operator, one in the lowering -- are each caught by the check meant for them and pinned on the right operator."""
import pytest
import torch

import emulator
import mlp_programs as mp
import opref
import program_audit as pa
from cleandiffuser_b200.engine import cabi, lower

# The interpreter stores the rounding of the exact value: at most half a unit of the output type, 2^-11 2^e for TF32 and
# 2^-8 2^e for bf16 (e: the exponent of |ref|, so 2^e <= |ref|), against the bound's 2^-10 |ref| and 2^-8 |ref|
PASS_FRAC = {"tf32": 0.5 + 1e-3, "bf16": 1.0}
NAMES = ["idql", "dql", "veteran50", "sfbc", "sfbc-cfg", "dbc10"]


@pytest.fixture(autouse=True)
def _emulate(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.delenv("CDS_BRANCHES", raising=False)


def _plan(name, math_mode, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math_mode)
    return mp.sample(name, "cpu", small=True)


class _Faulty:
    """the plan's handle with operator ``j`` replaced by ``fault(op, it)``"""

    def __init__(self, inner, j, fault):
        self.inner, self.j, self.fault = inner, j, fault

    def run(self, *a):
        self.inner.run(*a)

    def run_range(self, it, i, n, stream):
        for k in range(i, i + n):
            if k == self.j:
                self.fault(self.inner.ops[k], it)
            else:
                self.inner.run_range(it, k, 1, stream)


def _audit(plan, handle=None, iters=(0, 1)):
    aud = pa.Auditor("cpu", plan.program.ops, handle or plan.handle, pa.plan_owners(plan))
    plan.x.copy_(torch.randn(plan.x.shape, generator=torch.Generator().manual_seed(0)))
    aud.audit_once(0)
    for it in iters:
        aud.audit_iteration(it)
    return aud


def _pinned(failures, j):
    return bool(failures) and all(f"op {j} " in m for m in failures)


def _first_on(failures, j):
    """the first failure is operator j's (the NaN it stores then fails every operator downstream as well)"""
    return bool(failures) and f"op {j} " in failures[0]


@pytest.mark.parametrize("math_mode", ["tf32", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_every_operator_passes(name, math_mode, monkeypatch):
    agent, plan = _plan(name, math_mode, monkeypatch)
    aud = _audit(plan)
    assert not aud.failures, aud.failures[:5]
    assert aud.worst and max(f for f, _ in aud.worst.values()) <= PASS_FRAC[math_mode], aud.worst
    mp.check_forms(name, math_mode, plan)


@pytest.mark.parametrize("math_mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_lowered_denoiser_matches_the_fp64_module(name, math_mode, monkeypatch):
    agent, plan = _plan(name, math_mode, monkeypatch)
    err = mp.denoiser_check(name, agent, plan)
    print(f"[lowering] {name}-{math_mode}: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert max(err.values()) <= mp.LOWERING_TOL[math_mode], err


def _fail_with_nan(op, it, mem):
    """what a kernel that read past its operand would store, for the auditor to see"""
    emulator.view(mem, *pa.declared_outputs(op, it)[0]).fill_(float("nan"))


def test_simt_bf16_store_by_truncation_is_caught(monkeypatch):
    agent, plan = _plan("dbc10", "bf16", monkeypatch)
    ops, mem = plan.program.ops, plan.handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_CONV and op.u.conv.out_dtype == cabi.BF16 and
             cabi.conv_choice(op.u.conv)["family"] == "simt")

    def truncating(op, it):
        c = op.u.conv
        x, w, kw, out = emulator.conv_operands(c, it, mem)
        y = opref.conv(x, w, **kw).to(torch.float32).contiguous()
        out.copy_((y.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16))    # round toward zero
    aud = _audit(plan, _Faulty(plan.handle, j, truncating), iters=(1,))
    assert _pinned(aud.failures, j), aud.failures[:5]


def test_lnmod_broadcast_row_read_per_row_is_caught(monkeypatch):
    """IDQLMlp's LayerNorm affine is one row for the whole batch (mod_bstride 0); a kernel taking the stride as C reads
    past the table"""
    agent, plan = _plan("idql", "tf32", monkeypatch)
    ops, mem = plan.program.ops, plan.handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_LNMOD)
    assert ops[j].u.lnmod.mod_bstride == 0
    past = []

    def per_row(op, it):
        bad = cabi.Op.from_buffer_copy(op)
        bad.u.lnmod.mod_bstride = bad.u.lnmod.C
        try:
            emulator.run_lnmod(bad.u.lnmod, it, mem)
        except AssertionError as e:
            past.append(str(e))
            _fail_with_nan(op, it, mem)
    aud = _audit(plan, _Faulty(plan.handle, j, per_row), iters=(1,))
    assert past and "past its owner" in past[0], past
    assert _first_on(aud.failures, j), aud.failures[:5]


def test_cfg_shortcut_read_at_row_b_is_caught(monkeypatch):
    """SfBCUNet's first block with two CFG branches: the shortcut reads x_t at row b % res_batch_mod"""
    agent, plan = _plan("sfbc-cfg", "tf32", monkeypatch)
    ops, mem = plan.program.ops, plan.handle.mem
    j = next(i for i, op in enumerate(ops) if op.kind == cabi.OP_CONV and op.u.conv.res_batch_mod > 0)
    past = []

    def no_mod(op, it):
        bad = cabi.Op.from_buffer_copy(op)
        bad.u.conv.res_batch_mod = 0
        try:
            emulator.run_conv(bad.u.conv, it, mem)
        except AssertionError as e:
            past.append(str(e))
            _fail_with_nan(op, it, mem)
    aud = _audit(plan, _Faulty(plan.handle, j, no_mod), iters=(1,))
    assert past and "past its owner" in past[0], past
    assert _first_on(aud.failures, j), aud.failures[:5]


def test_sfbc_shift_of_the_wrong_block_is_caught_by_the_lowering_check_only(monkeypatch):
    """the first block's post-activation shift read one block to the right in the per-call tables: every operator is
    still what its descriptor says, so the audit passes and only the whole-network check can see it"""
    vec = lower._vec
    first_width = []

    def shifted(step=None, sample=None, col=0):
        if col == 0 and first_width:
            col = first_width[0]
        return vec(step, sample, col)
    orig = lower.lower_sfbc

    def lower_sfbc(p, net, x, has_cond, in_batch_mod):
        first_width.append(net.down_blocks[0].linear1[0].out_features)
        return orig(p, net, x, has_cond, in_batch_mod)
    monkeypatch.setattr(lower, "_vec", shifted)
    monkeypatch.setattr(lower, "lower_sfbc", lower_sfbc)
    agent, plan = _plan("sfbc", "tf32", monkeypatch)
    aud = _audit(plan)
    assert not aud.failures, aud.failures[:5]
    err = mp.denoiser_check("sfbc", agent, plan)
    assert err["pred"] > 100 * mp.LOWERING_TOL["tf32"], err
