"""TEST INFRASTRUCTURE: CDS_OP_MHA (include/cds.h) as plain torch fp64 code.

``mha`` is the one fp64 reference of the operator: the GPU tests run it next to the kernel (tests/mha_cases.py), and
tests/emulator.py executes lowered ChiTransformer programs on the CPU with it.  Never imported by the product.
"""
import math

import torch

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
