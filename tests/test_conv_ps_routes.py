"""The two L = 4 layer shapes that conv_ps serves through runtime parameters of existing instantiations:

* the 256-wide GroupNorm + Mish layer with a 1x1 shortcut conv on ps(32, shortcut): one GroupNorm group per CTA tile, whose
  statistics the two epilogue column slices combine;
* the two-phase transposed conv (the UNets' L = 4 -> 8 upsample, C_out >= 128) on ps(64, no shortcut): bias only, column c of
  phase ph at output position l stored at position 2 l + ph.

The CPU tests pin the routes (cds_conv_choice, host logic only), including those of cfg2's operators; the GPU tests check
the kernel against tests/opref.py's fp64 reference with the bound of conv_cases.check, and the conv_tc route (CDS_PS=0)
against the same bound."""
import pytest
import torch

import conv_cases as cc
import emulator
from cleandiffuser_b200 import workloads
from cleandiffuser_b200.engine import cabi
from test_conv_kernels_gpu import _fresh_out, _gaps_untouched, _run, _shifted

GN = cc.GN
DEV = "cuda:0"

CASES = {c["name"]: c for c in [
    # 256-wide layer + shortcut conv: ragged batch, an additive time row, a strided output view
    cc.case("ps_tf32_c256_k5_shortcut", "tf32", 300, 4, 256, 256, cc.ps(32, 1, 1), taps=5, **GN, res="conv", res_C=128,
            film="shift", strided=True),
    cc.case("ps_tf32_c256_k3_shortcut_mods", "tf32", 512, 4, 128, 256, cc.ps(32, 1, 1), taps=3, **GN, res="conv", res_C=64,
            in_mod=256, res_mod=128),
    cc.case("ps_bf16_c256_k5_shortcut", "bf16", 300, 4, 256, 256, cc.ps(32, 1, 0), taps=5, **GN, res="conv", res_C=128,
            strided=True),
    # two-phase transposed conv, bias only
    cc.case("ps_tf32_convT_c128", "tf32", 300, 4, 128, 128, cc.ps(64, 0, 1), taps=3, phases=2, strided=True),
    cc.case("ps_tf32_convT_c256", "tf32", 300, 4, 256, 256, cc.ps(64, 0, 1), taps=3, phases=2),
    cc.case("ps_tf32_convT_c128_mod", "tf32", 512, 4, 128, 128, cc.ps(64, 0, 1), taps=3, phases=2, in_mod=256, bias=None),
    cc.case("ps_bf16_convT_c128", "bf16", 300, 4, 128, 128, cc.ps(64, 0, 0), taps=3, phases=2, strided=True),
]}


@pytest.mark.parametrize("name", list(CASES))
def test_route(name, monkeypatch):
    monkeypatch.delenv("CDS_PS", raising=False)
    c = CASES[name]
    op = cc.descriptor(c)
    assert cc.choice_key(cabi.conv_choice(op.u.conv)) == c["want"]
    monkeypatch.setenv("CDS_PS", "0")
    assert cabi.conv_choice(op.u.conv)["family"] == "tc"


def test_upsample_routes():
    """the 64-wide upsample, a time row or GroupNorm on the upsample, and the other resolutions stay on conv_tc"""
    up = cc.case("up", "tf32", 300, 4, 128, 128, None, taps=3, phases=2)
    assert cabi.conv_choice(cc.descriptor(up).u.conv)["family"] == "ps"
    for kw in (dict(C_in=64, C_out=64), dict(film="shift"), dict(act=cabi.ACT_MISH), dict(L=8), dict(L=2)):
        assert cabi.conv_choice(cc.descriptor(dict(up, **kw)).u.conv)["family"] == "tc", kw


def test_cfg2_l4_stage_routes(monkeypatch):
    """every convolution of cfg2's L = 4 stage runs position-sliced: op 17 (256 -> 256 k5 + 1x1 shortcut 128 -> 256) on
    ps(32, shortcut), op 28 (the L = 4 -> 8 upsample, 128 channels) on ps(64)"""
    emulator.emulate(monkeypatch)
    monkeypatch.delenv("CDS_PS", raising=False)
    for k, v in dict(CDS_BACKEND="cuda", CDS_MATH="tf32", CDS_BRANCHES="1", CDS_BRANCH_MIN_BATCH="1").items():
        monkeypatch.setenv(k, v)
    w = workloads.cfg2("cpu", batch=8, steps=1)
    with torch.no_grad():
        w.sample("cpu")
    ops = next(iter(w.agent._engine_plans.values())).program.ops
    convs = {i: op.u.conv for i, op in enumerate(ops) if op.kind == cabi.OP_CONV}
    l4 = {i for i, c in convs.items() if c.L_in == 4 and c.stride == 1}
    assert l4 == set(range(16, 29))
    assert all(cabi.conv_choice(convs[i])["family"] == "ps" for i in l4)
    c17, c28 = convs[17], convs[28]
    assert (c17.C_in, c17.C_out, c17.taps, c17.res_C, bool(c17.res_w)) == (256, 256, 5, 128, True)
    assert cc.choice_key(cabi.conv_choice(c17)) == cc.ps(32, True, True)
    assert (c28.C_in, c28.C_out, c28.taps, c28.phases, c28.groups) == (128, 128, 3, 2, 0)
    assert cc.choice_key(cabi.conv_choice(c28)) == cc.ps(64, False, True)


def _check(c, d, ref):
    ok, frac, msg = cc.check(c, d["view/out"].float(), ref)
    assert ok, msg
    assert _gaps_untouched(c, d), "a write outside the output view"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_matches_fp64(name, monkeypatch):
    for var in ("CDS_NO_TMA_STORE", "CDS_PS"):
        monkeypatch.delenv(var, raising=False)
    c = CASES[name]
    d = cc.make(c, DEV)
    op = cc.descriptor(c, d)
    assert cc.choice_key(cabi.conv_choice(op.u.conv)) == c["want"]
    ref = cc.reference(c, d)
    _run(c, op)
    _check(c, d, ref)
    y = d["view/out"].float().clone()

    # the direct-store fallback: the same bits
    monkeypatch.setenv("CDS_NO_TMA_STORE", "1")
    _fresh_out(d)
    _run(c, cc.descriptor(c, d))
    assert torch.equal(d["view/out"].float(), y), "the store path changed the result"
    assert _gaps_untouched(c, d)
    monkeypatch.delenv("CDS_NO_TMA_STORE")

    # trajectories [17, B): every trajectory tile starts half-way into a 128-trajectory tile of the full batch
    if not (c["in_mod"] or c["res_mod"]):
        _fresh_out(d)
        _run(c, _shifted(c, d, 17))
        assert torch.equal(d["view/out"][17:].float(), y[17:]), "a sub-batch at a tile-unaligned offset differs"

    # the conv_tc route of the same op, against the same bound
    monkeypatch.setenv("CDS_PS", "0")
    op_tc = cc.descriptor(c, d)
    assert cabi.conv_choice(op_tc.u.conv)["family"] == "tc"
    _fresh_out(d)
    _run(c, op_tc)
    _check(c, d, ref)
