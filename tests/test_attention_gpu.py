"""Operator-level parity of CDS_OP_ATTN against softmax(q k^T / sqrt(d)) v in fp64 on the same q / k / v.

Every case of tests/attn_cases.py -- every kernel and all 20 instantiations -- runs through ``cds_run_op`` with each
value pattern of attn_cases.MODES and each output dtype it supports, and is checked against tests/opref.py with the
bound of attn_cases.check.  Each case also checks that NaN sentinels around the output stay untouched, that two runs give
the same bits, that TF32 / bf16 outputs are exactly the rounding of the kernel's fp32 output, and that a sub-batch at a
trajectory offset gives the same bits.  At the end the module prints each kernel's largest error as a fraction of its bound.

Reference behaviour: nn.MultiheadAttention's core inside DiTBlock (cleandiffuser/nn_diffusion/dit.py:10-36)."""
import numpy as np
import pytest
import torch

import attn_cases as ac
import opref
from cleandiffuser_b200.engine import cabi, lower

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SPARE = 4096            # NaN elements after the output
WORST = {}              # kernel family -> (largest error / bound, case)


def _run_attn(qkv, heads, out_dtype):
    B, L, C3 = qkv.shape
    out = torch.full((B, L, C3 // 3), float("nan"), device=qkv.device, dtype=torch.float32)
    op = cabi.Op()
    op.kind = cabi.OP_ATTN
    a = op.u.attn
    a.batch, a.L, a.C, a.heads = B, L, C3 // 3, heads
    a.qkv = qkv.data_ptr()
    a.out = out.data_ptr()
    a.out_dtype, a.qkv_dtype = out_dtype, cabi.TF32
    cabi.run_op(qkv.device.index or 0, op, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B,L,heads", [(3, 100, 10), (2, 128, 4), (5, 17, 2), (1, 7, 1), (4, 96, 3), (700, 100, 10), (2, 113, 5)])
def test_tf32_attention_matches_fp64(B, L, heads):
    g = torch.Generator().manual_seed(100 * B + L)
    C_ = 32 * heads
    qkv = torch.randn(B, L, 3 * C_, generator=g) * 1.5
    qkv = lower.round_tf32(qkv).cuda()
    out = _run_attn(qkv, heads, cabi.F32)
    q, k, v = (t.reshape(B, L, heads, 32).permute(0, 2, 1, 3).double() for t in qkv.split(C_, dim=-1))
    ref = torch.softmax(q @ k.transpose(-1, -2) / np.sqrt(32.0), dim=-1) @ v
    ref = ref.permute(0, 2, 1, 3).reshape(B, L, C_)
    err = (out.double() - ref).abs()
    assert torch.isfinite(out).all()
    # P is rounded to TF32 (10 mantissa bits) before P V: |err| <= 2^-11 * sum_j P_j |v_j| <= ~5e-4 * max|v|
    assert err.max().item() < 4e-3, err.max().item()
    assert err.mean().item() < 3e-4, err.mean().item()


def test_tf32_attention_rounded_output_and_repeatability():
    g = torch.Generator().manual_seed(7)
    qkv = lower.round_tf32(torch.randn(64, 100, 960, generator=g)).cuda()
    a = _run_attn(qkv, 10, cabi.TF32)
    b = _run_attn(qkv, 10, cabi.TF32)
    assert torch.equal(a, b)
    bits = a.view(torch.int32)
    assert int((bits & 0x1FFF).abs().max()) == 0          # stored values are TF32-representable
    c = _run_attn(qkv, 10, cabi.F32)
    assert (a - c).abs().max().item() < 2e-3


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    """after the module: the largest error of each kernel as a fraction of its bound, over every checked run"""
    WORST.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print()
        for fam, (frac, name) in sorted(WORST.items()):
            print(f"[attn] {fam}: largest error = {frac:.3f} of the bound ({name})")


def _record(fam, frac, name):
    if frac > WORST.get(fam, (0.0, ""))[0]:
        WORST[fam] = (frac, name)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _launch(c, qkv, out_dtype, first=0):
    """run the case on trajectories [first, B) of qkv into a fresh NaN-filled buffer: returns (buffer, output view of all B
    trajectories, descriptor)"""
    B, L, C3 = qkv.shape
    n = B * L * (C3 // 3)
    off = c["out_off"]
    buf = torch.full((off + n + SPARE,), float("nan"), dtype=ac.TORCH_DT[out_dtype], device=DEV)
    out = buf[off:off + n].view(B, L, C3 // 3)
    op = ac.descriptor(c, qkv[first:].data_ptr(), out[first:].data_ptr(), out_dtype, B=B - first)
    cabi.run_op(0, op, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return buf, out, op


def _sentinels_untouched(c, buf, qkv):
    n = qkv.shape[0] * qkv.shape[1] * qkv.shape[2] // 3
    return bool(torch.isnan(buf[:c["out_off"]]).all() and torch.isnan(buf[c["out_off"] + n:]).all())


@pytest.mark.parametrize("name", list(ac.CASES))
def test_attention_case_matches_fp64(name):
    c = ac.CASES[name]
    fam = c["want"][0]
    if fam == "tma":         # the grid regime the case was sized for (attn_cases.SMS) holds on this device
        grid = 2 * cabi.load().cds_device_sm_count(0)
        work = c["B"] * c["heads"]
        assert work >= 3 * grid if name.endswith("_ring") else work < grid, (work, grid)
    for mode in ac.MODES:
        qkv = ac.make(c, mode, DEV)
        ref = opref.attn(qkv, c["heads"], c["qkv_dtype"])
        y32 = None
        for od in c["outs"]:
            buf, out, op = _launch(c, qkv, od)
            assert ac.choice_key(cabi.attn_choice(op.u.attn)) == c["want"]
            assert _sentinels_untouched(c, buf, qkv), f"{mode}: a write outside the output"
            y = out.float()
            ok, frac, msg = ac.check(c, y, qkv, ref, od)
            _record(fam, frac, f"{name} {mode} out={od}")
            assert ok, f"{mode} out={od}: {msg}"
            if od == cabi.F32:
                y32 = y
            elif y32 is not None:
                assert torch.equal(_bits(opref.store(y32, od)), _bits(y)), \
                    f"{mode}: out={od} is not the rounding of the kernel's fp32 output"
        if mode != "n0.5":
            continue
        od = c["outs"][0]
        full = _launch(c, qkv, od)[1]
        again = _launch(c, qkv, od)[1]
        assert torch.equal(_bits(again), _bits(full)), "two runs differ"
        buf, sub, op = _launch(c, qkv, od, first=1)
        assert ac.choice_key(cabi.attn_choice(op.u.attn)) == c["want"]
        assert torch.isnan(sub[0].float()).all() and _sentinels_untouched(c, buf, qkv)
        assert torch.equal(_bits(sub[1:]), _bits(full[1:])), "a sub-batch at a trajectory offset differs"
