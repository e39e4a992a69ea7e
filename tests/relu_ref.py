"""TEST INFRASTRUCTURE: CDS_ACT_RELU for the shared operator references.  tests/opref.py, tests/grad_ref.py and
tests/program_audit.py describe the activations the other operators use; ``register(monkeypatch)`` adds ReLU to them for the
duration of one test, so that the interpreter (tests/emulator.py), the error bounds and the program audit read CDS_OP_STASH
and CDS_OP_DGRAD with ReLU like every other activation:
  - opref.act: relu(x) = x where x > 0, else 0;
  - grad_ref.ACT_BOUND / ACT_GRAD: ReLU and its derivative (1 where x > 0, else 0, so 0 at x == 0: ATen's threshold_backward)
    are selects, exact in fp32, so their own error bound is 0;
  - program_audit.instantiation: "stash relu", "stash relu (no slot)" and "dgrad relu" name the kernel instantiations."""
import numpy as np
import torch

import grad_ref
import opref
import program_audit
from cleandiffuser_b200.engine import cabi


def relu_grad(x):
    """d/dx relu(x) (ATen's threshold_backward: 1 where x > 0, else 0, so 0 at x == 0)"""
    return (np.asarray(x, np.float64) > 0).astype(np.float64)


def exact_bound(z):
    """ReLU and its derivative are exact in fp32 (a select): no error of their own"""
    return np.zeros_like(np.asarray(z, np.float64))


def register(monkeypatch):
    """ReLU in opref.act, grad_ref.ACT_BOUND / ACT_GRAD and program_audit.instantiation until the test ends"""
    act, instantiation = opref.act, program_audit.instantiation

    def act_with_relu(kind, x):
        if kind == cabi.ACT_RELU:
            return torch.where(x > 0, x, torch.zeros_like(x))
        return act(kind, x)

    def instantiation_with_relu(op):
        if op.kind == cabi.OP_STASH and op.u.stash.act == cabi.ACT_RELU:
            return "stash relu" + ("" if op.u.stash.dst else " (no slot)")
        if op.kind == cabi.OP_DGRAD and op.u.dgrad.act == cabi.ACT_RELU:
            d = op.u.dgrad
            return f"dgrad relu{' +=' if d.accumulate else ''}{' +out_sum' if d.out_sum else ''}"
        return instantiation(op)

    monkeypatch.setattr(opref, "act", act_with_relu)
    monkeypatch.setattr(program_audit, "instantiation", instantiation_with_relu)
    monkeypatch.setitem(grad_ref.ACT_BOUND, cabi.ACT_RELU, exact_bound)
    monkeypatch.setitem(grad_ref.ACT_GRAD, cabi.ACT_RELU, (relu_grad, exact_bound))
