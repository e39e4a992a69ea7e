"""TEST INFRASTRUCTURE: CDS_OP_MHA (include/cds.h) as plain torch fp64 code, and the numpy interpreter of tests/emulator.py
extended with that operator.

``mha`` is the one fp64 reference of the operator: the GPU tests run it next to the kernel (tests/mha_cases.py), and
``Handle`` executes lowered ChiTransformer programs on the CPU with it, every other operator going through tests/emulator.py.
Never imported by the product.
"""
import math

import numpy as np
import torch

import emulator
import opref
from cleandiffuser_b200.engine import cabi

F64 = torch.float64


def mha(q, kv, heads, diag=None):
    """CDS_OP_MHA in fp64: q (batch, Lq, C), kv (batch, Lk, 2C) with [k | v] column blocks (the step + sample sum), both read
    as stored; key j is visible to query i iff j <= i + diag (diag None: every key).  (batch, Lq, C); a query row without a
    visible key is zeros."""
    B, Lq, C = q.shape
    Lk, hd = kv.shape[1], C // heads
    q = q.to(F64).reshape(B, Lq, heads, hd).transpose(1, 2)                                      # (B, heads, Lq, hd)
    k, v = (t.to(F64).reshape(B, Lk, heads, hd).transpose(1, 2) for t in kv.split(C, dim=-1))
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    if diag is not None:
        vis = torch.arange(Lk, device=q.device)[None, :] <= torch.arange(Lq, device=q.device)[:, None] + diag
        s = s.masked_fill(~vis, float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
    return (p @ v).transpose(1, 2).reshape(B, Lq, C)


def mha_operands(m, it, mem=emulator.HOST):
    """(q view as stored, k|v as the fp32 sum step + sample (the kernel's adds of the widened parts), output view, whether both
    k|v parts are present) of a CDS_OP_MHA descriptor"""
    esize = 2 if m.in_dtype == cabi.BF16 else 4
    q = emulator.view(mem, m.q, (m.batch, m.Lq, m.C), (m.q_bstride, m.q_lstride, 1), m.in_dtype)
    kv = None
    if m.kv_step:
        kv = emulator.view(mem, m.kv_step + esize * it * m.kv_step_stride, (m.Lk, 2 * m.C), (m.kv_step_lstride, 1),
                           m.in_dtype).float()[None].expand(m.batch, m.Lk, 2 * m.C)
    if m.kv_sample:
        s = emulator.view(mem, m.kv_sample, (m.batch, m.Lk, 2 * m.C), (m.kv_sample_bstride, m.kv_sample_lstride, 1),
                          m.in_dtype).float()
        kv = s if kv is None else s + kv
    out = emulator.view(mem, m.out, (m.batch, m.Lq, m.C), (m.out_bstride, m.out_lstride, 1), m.out_dtype)
    return q, kv, out, bool(m.kv_step and m.kv_sample)


def run_mha(m, it, mem=emulator.HOST):
    """CDS_OP_MHA: q and the k|v sum through ``mha``"""
    q, kv, out, _ = mha_operands(m, it, mem)
    out.copy_(opref.store(mha(q, kv, m.heads, m.diag if m.masked else None), m.out_dtype).to(out.dtype))


def run_program(ops, n_iters, first=0, mem=emulator.HOST):
    """emulator.run_program with CDS_OP_MHA: same order, the other operators run one at a time by tests/emulator.py"""
    emulator.run_program([op for op in ops if op.flags & cabi.OPF_ONCE], 0, first, mem)
    body = [op for op in ops if not op.flags & cabi.OPF_ONCE]
    for it in range(first, first + n_iters):
        for op in body:
            if op.kind == cabi.OP_MHA:
                run_mha(op.u.mha, it, mem)
            else:
                emulator.run_program([op], 1, it, mem)


class Handle(emulator.Handle):
    """emulator.Handle for programs that contain CDS_OP_MHA"""

    def run(self, first, count, stream, use_graph=True):
        run_program(self.ops, count, first, self.mem)

    def run_range(self, it, op_first, op_count, stream):
        keep = [op for op in self.ops[op_first:op_first + op_count] if not (op.flags & cabi.OPF_ONCE)]
        run_program(keep, 1, it, self.mem)
