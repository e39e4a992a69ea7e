"""Time CDS_OP_ATTN alone at a DiT1d shape (default: cfg4's 4096 x 100 tokens, 10 heads of 32) through cds_run_op.
usage: python scripts/attn_bench.py [batch] [L] [heads] [reps]"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from cleandiffuser_b200.engine import cabi, lower  # noqa: E402

B, L, H, reps = (int(a) for a in (sys.argv[1:5] + ["4096", "100", "10", "20"][len(sys.argv) - 1:]))
Cd = 32 * H
qkv = lower.round_tf32(torch.randn(B, L, 3 * Cd)).cuda()
out = torch.empty(B, L, Cd, device="cuda")
op = cabi.Op()
op.kind = cabi.OP_ATTN
a = op.u.attn
a.batch, a.L, a.C, a.heads = B, L, Cd, H
a.qkv = qkv.data_ptr()
a.out = out.data_ptr()
a.out_dtype, a.qkv_dtype = cabi.TF32, cabi.TF32
st = torch.cuda.current_stream().cuda_stream
for _ in range(3):
    cabi.run_op(0, op, 0, st)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    cabi.run_op(0, op, 0, st)
e1.record()
torch.cuda.synchronize()
us = e0.elapsed_time(e1) / reps * 1e3
flop = 4.0 * B * H * L * L * 32
byt = 4.0 * B * L * Cd * 4
print(f"attn B={B} L={L} heads={H}: {us:.1f} us  {flop / us / 1e6:.1f} TFLOP/s  {byt / us / 1e3:.0f} GB/s (algorithmic)")
