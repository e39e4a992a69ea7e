"""DiT1d's gated Linear -> LayerNorm + modulate pair as the lowering emits it, run as a two-operator plan: conv_tc's gated
and table epilogue lanes followed by LNMOD.  Both outputs -- X, the Linear's result, and Y, the modulated LayerNorm of X --
are checked against tests/opref.py in fp64 at row counts from fewer 128-row tiles than an H100 has SMs to several tiles
per persistent CTA, with a ragged last tile and with the CFG halves sharing their input rows."""
import pytest
import torch

import opref
from cleandiffuser_b200.engine import cabi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C_IN, C = 128, 256
ATOL, R_TF32 = 1e-4, 2.0 ** -10
SPARE = 128

# (form, tokens per trajectory L, trajectories, CFG halves share their input rows, X dtype)
PLANS = [
    ("gated", 100, 37, False, cabi.F32),        # 3700 rows: fewer row tiles than SMs
    ("table", 32, 1064, True, cabi.F32),        # 34048 rows
    ("gated", 32, 2000, True, cabi.TF32),       # 64000 rows
    ("table", 100, 617, False, cabi.F32),       # 61700 rows: ragged last tile
]


def _plan(form, L, B, shared, x_dtype):
    g = torch.Generator().manual_seed(L * 7 + B)
    rows = B * L
    in_rows = rows // 2 if shared else rows
    assert not shared or in_rows % 128 == 0
    d = {"x": opref.tf32_round(torch.randn(in_rows, C_IN, generator=g)).to(DEV),
         "w": opref.tf32_round(torch.randn(C, C_IN, generator=g) / C_IN ** 0.5).to(DEV),
         "bias": (0.1 * torch.randn(2, C, generator=g)).to(DEV),
         "gate": (1 + 0.3 * torch.randn(B, C + 4, generator=g)).to(DEV),
         "res": torch.randn(L if form == "table" else rows, C, generator=g).to(DEV),
         "mod": (0.3 * torch.randn(B, 2 * C + 4, generator=g)).to(DEV),
         # one spare 128-row tile of NaN after X and Y: a write past the (ragged) last tile shows up there
         "Xbuf": torch.full((rows + SPARE, C), float("nan"), device=DEV),
         "Ybuf": torch.full((rows + SPARE, C), float("nan"), device=DEV)}
    d["X"], d["Y"] = d["Xbuf"][:rows], d["Ybuf"][:rows]
    lin = cabi.Op()
    lin.kind = cabi.OP_CONV
    c = lin.u.conv
    c.batch, c.L_in, c.L_out, c.C_in, c.C_out, c.taps, c.stride, c.pad, c.phases = rows, 1, 1, C_IN, C, 1, 1, 0, 1
    c.in_batch_mod = in_rows if shared else 0
    c.in_, c.in_bstride, c.in_lstride, c.in_dtype = d["x"].data_ptr(), C_IN, C_IN, cabi.TF32
    c.w, c.math = d["w"].data_ptr(), cabi.MATH_TF32_TC
    c.bias = cabi.Vec(d["bias"].data_ptr(), C, 0, 0)
    if form == "gated":
        c.scale = cabi.Vec(0, 0, d["gate"].data_ptr(), C + 4)
    c.res, c.res_bstride, c.res_lstride, c.res_dtype = d["res"].data_ptr(), C, C, cabi.F32
    c.res_batch_mod = L if form == "table" else 0
    c.sample_row_div = L
    c.out, c.out_bstride, c.out_lstride, c.out_dtype = d["X"].data_ptr(), C, C, x_dtype
    ln = cabi.Op()
    ln.kind = cabi.OP_LNMOD
    m = ln.u.lnmod
    m.batch, m.L, m.C, m.eps = B, L, C, 1e-6
    m.in_, m.out, m.out_dtype = d["X"].data_ptr(), d["Y"].data_ptr(), cabi.TF32
    m.shift, m.scale, m.mod_bstride = d["mod"].data_ptr(), d["mod"].data_ptr() + 4 * C, 2 * C + 4
    return [lin, ln], d


def _reference_x(form, L, B, d):
    rows = B * L
    return opref.conv(d["x"][:, None], d["w"].t()[None], batch=rows, L_out=1, math_mode=cabi.MATH_TF32_TC,
                      bias=d["bias"][1], scale=d["gate"][:, :C] if form == "gated" else None, res=d["res"][:, None],
                      sample_row_div=L)[:, 0]


def _check(y, ref, r):
    s = max(1.0, ref.abs().mean().item())
    frac = ((y.double() - ref).abs() / (ATOL * s + r * ref.abs())).max().item()
    assert torch.isfinite(y).all()
    return frac


@pytest.mark.parametrize("form,L,B,shared,x_dtype", PLANS)
def test_linear_layernorm_plan_matches_fp64(form, L, B, shared, x_dtype):
    st = torch.cuda.current_stream().cuda_stream
    ops, d = _plan(form, L, B, shared, x_dtype)
    plan = cabi.Plan(0)
    plan.append(ops)
    plan.finalize(2)
    assert plan.launches_per_iter() == 3                      # the two operators and the iteration-counter advance
    runs = []
    for _ in range(2):
        d["Xbuf"].fill_(float("nan"))
        d["Ybuf"].fill_(float("nan"))
        plan.run(1, 1, st, use_graph=False)
        torch.cuda.synchronize()
        assert torch.isnan(d["Xbuf"][B * L:]).all() and torch.isnan(d["Ybuf"][B * L:]).all(), "a write past the last row"
        runs.append((d["X"].clone(), d["Y"].clone()))
    plan.close()
    X, Y = runs[0]
    assert torch.equal(X.view(torch.int32), runs[1][0].view(torch.int32))
    assert torch.equal(Y.view(torch.int32), runs[1][1].view(torch.int32))
    fx = _check(X, _reference_x(form, L, B, d), R_TF32 if x_dtype == cabi.TF32 else 0.0)
    # Y against the LayerNorm of the X the kernel stored: X's own rounding is checked above
    fy = _check(Y, opref.lnmod(X, d["mod"][:, :C], d["mod"][:, C:2 * C], 1e-6, L=L), R_TF32)
    assert int((Y.view(torch.int32) & 0x1FFF).abs().max()) == 0
    print(f"[linear+layernorm] {form} L={L} rows={B * L}: X {fx:.3f}, Y {fy:.3f} of the bound")
    assert fx <= 1 and fy <= 1, (fx, fy)
