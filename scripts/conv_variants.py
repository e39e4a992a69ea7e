"""Which conv kernel instantiations does the test-suite reach?  Prints a markdown table on the CPU (needs the built libcds.so,
no GPU): for every instantiation of CDS_TC_VARIANTS / CDS_PS_VARIANTS and conv_simt, the convs that reach it

  * "nets / workloads": every cases.NETS entry (at the batch of the net-level tests) and every workloads config (at its
    benchmark batch), lowered in each math mode, each conv passed through cds_conv_choice;
  * "operator cases": the cases of tests/conv_cases.py.

python scripts/conv_variants.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

import torch  # noqa: E402

import cases  # noqa: E402
import conv_cases as cc  # noqa: E402
from common import product_net  # noqa: E402
from test_conv_dispatch_cpu import _instantiations  # noqa: E402
from cleandiffuser_b200 import workloads  # noqa: E402
from cleandiffuser_b200.engine import cabi  # noqa: E402
from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser  # noqa: E402

LOWER_ROWS = 256         # lowering batch; the descriptors are then scaled to the real batch (only m_tiles depends on it)


def _lowered(net, x_shape, rows, has_cond, cfg_branches):
    """cds_conv_choice keys of the convs of ``net`` lowered for ``rows`` trajectories, in every math mode"""
    out = []
    L, D = x_shape if len(x_shape) == 2 else (1, x_shape[-1])
    sub = LOWER_ROWS
    for math in (cabi.MATH_TF32_TC, cabi.MATH_BF16_TC, cabi.MATH_FP32):
        p = Program(torch.device("cpu"), sub * cfg_branches, 1, math)
        lower_denoiser(p, net, View(p.buf(sub * cfg_branches, L, D), L, D), x_shape, has_cond,
                       sub if cfg_branches == 2 else 0)
        for op in p.ops:
            if op.kind != cabi.OP_CONV:
                continue
            c = cabi.ConvOp.from_buffer_copy(op.u.conv)
            f = rows / sub
            c.batch = int(round(c.batch * f))
            if c.in_batch_mod:
                c.in_batch_mod = int(round(c.in_batch_mod * f))
            out.append(cc.choice_key(cabi.conv_choice(c)))
    return out


def before():
    reached = {}
    for name, case in cases.NETS.items():
        net, _ = product_net(case)
        for k in _lowered(net, case["x"], cases.NET_BATCH, case["cond"] is not None, 1):
            reached.setdefault(k, set()).add(name)
    for name, build in workloads.BUILDERS.items():
        wl = build("cpu", steps=1) if name != "cfg3" else build("cpu", steps=2)
        model = wl.agent.model_ema if hasattr(wl.agent, "model_ema") else wl.agent.model
        two = float(wl.kwargs.get("w_cfg", 1.0)) not in (0.0, 1.0)
        for k in _lowered(model["diffusion"], tuple(wl.prior.shape[1:]), wl.prior.shape[0], wl.cond is not None,
                          2 if two else 1):
            reached.setdefault(k, set()).add(name)
    return reached


def main():
    torch.set_grad_enabled(False)
    inst = sorted(_instantiations() | {cc.simt(32), cc.simt(64), cc.simt(128)}, key=str)
    old = before()
    new = {}
    for c in cc.CASES.values():
        new.setdefault(c["want"], []).append(c["name"])
    print("| instantiation | nets / workloads | operator cases |")
    print("|---|---|---|")
    for k in inst:
        print(f"| {k} | {', '.join(sorted(old.get(k, []))) or '-'} | {len(new.get(k, []))} |")
    print(f"\n{len(inst)} instantiations: the nets / workloads reach {sum(1 for k in inst if k in old)}, the operator cases "
          f"{sum(1 for k in inst if k in new)}")


if __name__ == "__main__":
    main()
