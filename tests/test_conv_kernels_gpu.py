"""Operator-level parity of CDS_OP_CONV: every case of tests/conv_cases.py runs through ``cds_run_op`` and is checked
against tests/opref.py's fp64 reference on the same GPU, with the bound of conv_cases.check.  Each case also checks
that the gaps of every buffer (NaN) are neither read nor written, that the result is deterministic and does not depend
on the TMA store / residual-prefetch path, on the position of the batch in its tiles, or (CDS_TF32 outputs, and every
TF32 / bf16 output of conv_simt) on anything but the round-to-nearest of the kernel's fp32 value."""
import pytest
import torch

import conv_cases as cc
import opref
from cleandiffuser_b200.engine import cabi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}          # kernel family -> (largest error / bound, case)


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    """after the module: the largest error of each kernel family as a fraction of its bound, over every checked run"""
    WORST.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print()
        for fam, (frac, name) in sorted(WORST.items()):
            print(f"[conv] {fam}: largest error = {frac:.3f} of the bound ({name})")


def _record(fam, frac, name):
    if frac > WORST.get(fam, (0.0, ""))[0]:
        WORST[fam] = (frac, name)


def _run(c, op):
    """run the op once at iteration 1: through cds_run_op, or -- ``one_cta`` cases -- inside a plan with a second, trivial
    branch, where every conv_tc launch is capped at one CTA per SM"""
    st = torch.cuda.current_stream().cuda_stream
    if not c.get("one_cta"):
        cabi.run_op(0, op, 1, st)
        torch.cuda.synchronize()
        return
    src = torch.zeros(1, 1, 2, device=DEV)
    dst = torch.zeros(1, 1, 2, device=DEV)
    side = cabi.Op()
    side.kind, side.flags = cabi.OP_CAST, 1 << cabi.OPF_BRANCH_SHIFT
    k = side.u.cast
    k.batch, k.L, k.C_in, k.C_out, k.in_, k.out, k.out_dtype = 1, 1, 2, 2, src.data_ptr(), dst.data_ptr(), cabi.F32
    plan = cabi.Plan(0)
    plan.append([op, side])
    plan.finalize(2)
    plan.run(1, 1, st, use_graph=False)
    torch.cuda.synchronize()
    plan.close()


def _fresh_out(d):
    d["buf/out"].fill_(float("nan"))


def _gaps_untouched(c, d):
    rows, Lv, C, dt = cc.geometry(c)["out"]
    buf, off = d["buf/out"], d["off/out"]
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    mask[:rows, :Lv, off:off + C] = False
    ibits = torch.int16 if buf.dtype == torch.bfloat16 else torch.int32
    nan = torch.full((1,), float("nan"), dtype=buf.dtype).view(ibits).item()
    return bool((buf.view(ibits)[mask] == nan).all())


def _shifted(c, d, k):
    """the op over trajectories [k, B) of the same buffers"""
    op = cc.descriptor(dict(c, B=c["B"] - k), d)
    o = op.u.conv
    geo = cc.geometry(c)
    for name, field in (("in", "in_"), ("out", "out"), ("res", "res"), ("res_in", "res_in")):
        if name in geo:
            es = 2 if geo[name][3] == cabi.BF16 else 4
            setattr(o, field, getattr(o, field) + k * getattr(o, (field.rstrip("_") + "_bstride")) * es)
    for v in (o.bias, o.scale, o.shift):
        if v.sample:
            v.sample += 4 * k * v.sample_stride
    return op


def _fast_lane(c):
    """is the layer served by conv_tc_kernel's GroupNorm + Mish lane (fast_ok: also needs out_dtype == the operand type)?"""
    return bool(c["groups"] and c["act"] == cabi.ACT_MISH and c["film"] not in ("traj", "gate") and c["bias"] in ("step", None))


def _on_tma_store_lane(c):
    """is the layer served by an epilogue lane of conv_tc_kernel that exists only with a TMA-store target?"""
    fast = _fast_lane(c)
    gated = c["film"] == "gate" and c["res"] == "id" and c["act"] == cabi.ACT_NONE
    table = c["res"] == "id" and c["res_mod"] > 0 and c["film"] is None and c["groups"] == 0
    return bool(fast or gated or table)


@pytest.mark.parametrize("name", list(cc.CASES))
def test_conv_case_matches_fp64(name, monkeypatch):
    for var in ("CDS_NO_TMA_STORE", "CDS_NO_TMA_RES", "CDS_PS"):
        monkeypatch.delenv(var, raising=False)
    c = cc.CASES[name]
    d = cc.make(c, DEV)
    op = cc.descriptor(c, d)
    assert cc.choice_key(cabi.conv_choice(op.u.conv)) == c["want"]
    ref = cc.reference(c, d)
    extra = cc.gn_offset_atol(cc.pre_norm(c, d), c["groups"], d["gamma"]) if c["offset"] else 0.0
    _run(c, op)
    y = d["view/out"].float().clone()
    ok, frac, msg = cc.check(c, y, ref, extra)
    fam = c["want"][0]
    _record(fam, frac, name)
    assert ok, msg
    assert _gaps_untouched(c, d), "a write outside the output view"
    bits = d["buf/out"].clone()

    _fresh_out(d)
    _run(c, op)
    assert torch.equal(d["buf/out"].view(torch.int16 if bits.dtype == torch.bfloat16 else torch.int32),
                       bits.view(torch.int16 if bits.dtype == torch.bfloat16 else torch.int32)), "two runs differ"

    # the identity residual's TMA prefetch is a fetch path only: the same bits
    monkeypatch.setenv("CDS_NO_TMA_RES", "1")
    _fresh_out(d)
    _run(c, cc.descriptor(c, d))
    assert torch.equal(d["view/out"].float(), y), "the residual-fetch path changed the result"
    # Without the TMA store, the layers of the specialised epilogue lanes that require it (conv_tc_kernel: fast_ok,
    # gated_ok, table_ok) run on the generic lane, whose arithmetic rounds differently (GroupNorm as (v - mean) * rstd
    # instead of fma(v, rstd, -mean * rstd), Mish and the gate in another order): those agree within the bound, every
    # other layer bit for bit.
    monkeypatch.setenv("CDS_NO_TMA_STORE", "1")
    _fresh_out(d)
    _run(c, cc.descriptor(c, d))
    if fam == "tc" and _on_tma_store_lane(c):
        ok, frac, msg = cc.check(c, d["view/out"].float(), ref, extra)
        _record(fam, frac, name + " (CDS_NO_TMA_STORE=1)")
        assert ok, "CDS_NO_TMA_STORE=1: " + msg
    else:
        assert torch.equal(d["view/out"].float(), y), "the store path changed the result"
    assert _gaps_untouched(c, d)
    monkeypatch.delenv("CDS_NO_TMA_STORE")
    monkeypatch.delenv("CDS_NO_TMA_RES")

    if not (c["in_mod"] or c["res_mod"] or c["srd"] > 1):
        T = 128 // c["L"]                       # trajectories per 128-row tile
        k = T // 2 + 1 if T > 1 else 1
        sub = _shifted(c, d, k)
        if k < c["B"] and cc.choice_key(cabi.conv_choice(sub.u.conv)) == c["want"]:
            _fresh_out(d)
            _run(c, sub)
            assert torch.equal(d["view/out"][k:].float(), y[k:]), "a sub-batch at a tile-unaligned offset differs"

    # (a GroupNorm + Mish layer with fp32 output leaves the fast lane, whose rounding differs: there the low bits and the
    # bound above are the check)
    if c["out_dtype"] == cabi.TF32 and fam == "tc" and not _fast_lane(c):
        c32 = dict(c, out_dtype=cabi.F32)
        d32 = cc.make(c32, DEV)
        _run(c32, cc.descriptor(c32, d32))
        assert torch.equal(opref.tf32_round(d32["view/out"]).view(torch.int32), y.view(torch.int32)), \
            "CDS_TF32 store is not the round-to-nearest (ties away) of the kernel's fp32 value"

    if fam == "simt" and c["out_dtype"] != cabi.F32:
        _simt_store_is_the_rounding_of_fp32(c, d, y)

    if fam == "ps":
        monkeypatch.setenv("CDS_PS", "0")
        op_tc = cc.descriptor(c, d)
        assert cabi.conv_choice(op_tc.u.conv)["family"] == "tc"
        _fresh_out(d)
        _run(c, op_tc)
        ok, frac, msg = cc.check(c, d["view/out"].float(), ref, extra)
        _record("tc", frac, name + " (CDS_PS=0)")
        assert ok, "CDS_PS=0 (conv_tc): " + msg
        assert _gaps_untouched(c, d)


def _simt_store_is_the_rounding_of_fp32(c, d, y):
    """conv_gemm_f32_kernel reads out_dtype only in st_act, at the store: everything before it is the same arithmetic for
    every output type.  So the same op with an fp32 output, into a separate buffer, gives the kernel's fp32 value, and a
    TF32 / bf16 output must be exactly its round-to-nearest -- a check no bound can make, since one TF32 ulp is within
    the 2^-10 |ref| of conv_cases.check."""
    c32 = dict(c, out_dtype=cabi.F32)
    d32 = cc.make(c32, DEV)
    for name in cc.geometry(c):                         # the same operands, bit for bit
        if name != "out":
            assert torch.equal(d32["buf/" + name].float().nan_to_num(7.0), d["buf/" + name].float().nan_to_num(7.0)), name
    _run(c32, cc.descriptor(c32, d32))
    y32 = d32["view/out"]
    want = opref.tf32_round(y32) if c["out_dtype"] == cabi.TF32 else y32.to(torch.bfloat16).float()
    assert torch.equal(want.view(torch.int32), y.view(torch.int32)), \
        f"conv_simt's {'CDS_TF32' if c['out_dtype'] == cabi.TF32 else 'bf16'} store is not the round-to-nearest of its fp32 value"
