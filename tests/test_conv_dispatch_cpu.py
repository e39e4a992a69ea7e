"""CPU checks of the operator-level conv case table (tests/conv_cases.py): every case reaches the kernel instantiation
it names (cds_conv_choice, pure host logic), the table covers every instantiation the dispatcher can select, and the
checker of tests/test_conv_kernels_gpu.py accepts the fp64 reference and rejects three typical kernel faults."""
import os
import re

import pytest
import torch

import conv_cases as cc
import opref
from cleandiffuser_b200.engine import cabi

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cleandiffuser_b200", "csrc")


def _instantiations():
    tc_src = open(os.path.join(CSRC, "conv_tc.cuh")).read()
    ps_src = open(os.path.join(CSRC, "conv_ps.cuh")).read()
    body = lambda src, name: re.search(r"#define %s\(X\)(.*?)\n\n" % name, src, re.S).group(1)
    out = set()
    for kc, n, s, r, tf in re.findall(r"X\((\d+),\s*(\d+),\s*(\d+),\s*([01]),\s*([01])\)", body(tc_src, "CDS_TC_VARIANTS")):
        out.add(cc.tc(int(kc), int(n), int(s), int(r), int(tf)))
    for n, r, tf in re.findall(r"X\((\d+),\s*(true|false),\s*(true|false)\)", body(ps_src, "CDS_PS_VARIANTS")):
        out.add(cc.ps(int(n), r == "true", tf == "true"))
    return out


@pytest.mark.parametrize("name", list(cc.CASES))
def test_case_reaches_its_variant(name):
    c = cc.CASES[name]
    assert cc.choice_key(cabi.conv_choice(cc.descriptor(c).u.conv)) == c["want"]


def test_cases_cover_every_instantiation():
    inst = _instantiations()
    assert len(inst) == 64 + 6
    reached = {c["want"] for c in cc.CASES.values() if c["want"][0] != "simt"}
    assert reached == inst, (sorted(inst - reached), sorted(reached - inst))
    assert {c["want"] for c in cc.CASES.values() if c["want"][0] == "simt"} == {cc.simt(32), cc.simt(64), cc.simt(128)}


def test_every_tc_instantiation_runs_three_tiles_per_cta():
    """the persistent tile loop of conv_tc: for every instantiation some case gives each resident CTA (at most
    2 per SM, or 1 in a plan with parallel branches) three or more tiles, counted from cds_conv_choice's SPLIT / column
    tiles"""
    best = {}
    for c in cc.CASES.values():
        if c["want"][0] != "tc":
            continue
        ch = cabi.conv_choice(cc.descriptor(c).u.conv)
        tiles = -(-c["B"] * c["L"] // 128) * (ch["split"] if ch["split"] > 1 else ch["col_tiles"])
        assert tiles == cc.num_tiles(c), c["name"]
        best[c["want"]] = max(best.get(c["want"], 0), tiles / cc.resident_ctas(c))
    tc_variants = {k for k in _instantiations() if k[0] == "tc"}
    assert set(best) == tc_variants
    assert all(v >= 3 for v in best.values()), sorted((v, k) for k, v in best.items() if v < 3)


def test_conv_choice_reports_refusals():
    c = cc.descriptor(cc.CASES["bf16_c128_k64"]).u.conv
    c.L_out = 3                                     # not a power of two: no tensor-core kernel
    with pytest.raises(cabi.CdsError):
        cabi.conv_choice(c)
    c.math = cabi.MATH_FP32                         # ... and GroupNorm tiles of 128 rows hold whole trajectories only
    with pytest.raises(cabi.CdsError):
        cabi.conv_choice(c)
    c.groups = 0
    assert cabi.conv_choice(c) == {"family": "simt", "bn": 128}


# ---- the checker itself, with the fp64 reference standing in for the kernel (small batches, CPU)
SELF_CHECK = ["bf16_c128_k64", "tf32_c32_gn_k64", "tf32_convT_c64", "ps_tf32_c128_k5", "simt_bn64_cpg8"]


def _small(name):
    return dict(cc.CASES[name], B=5)


def _kernel_like(c, d):
    """what a correct kernel stores: the exact result rounded to fp32, then to the output type"""
    return opref.store(cc.reference(c, d), c["out_dtype"])


@pytest.mark.parametrize("name", SELF_CHECK)
def test_checker_accepts_the_reference(name):
    c = _small(name)
    d = cc.make(c, "cpu")
    ok, frac, msg = cc.check(c, _kernel_like(c, d), cc.reference(c, d))
    assert ok, msg


@pytest.mark.parametrize("name", SELF_CHECK)
def test_checker_rejects_a_tap_shifted_by_one(name):
    c = _small(name)
    d = cc.make(c, "cpu")
    ref = cc.reference(c, d)
    if c["taps"] == 1:
        pytest.skip("1x1 conv")
    bad = opref.store(opref.conv(d["view/in"], d["w"], batch=c["B"], L_out=c["L"], taps=c["taps"], stride=c["stride"],
                                 pad=c["taps"] // 2 - 1, phases=c["phases"], math_mode=cc.MATH[c["math"]], bias=d["bias"],
                                 groups=c["groups"], gamma=d.get("gamma"), beta=d.get("beta"), act_kind=c["act"],
                                 scale=d["scale"], shift=d["shift"], res=d.get("view/res"), res_in=d.get("view/res_in"),
                                 res_w=d.get("res_w"), res_bias=d.get("res_bias")), c["out_dtype"])
    assert not cc.check(c, bad, ref)[0]


@pytest.mark.parametrize("name", [n for n in SELF_CHECK if cc.CASES[n]["groups"]])
def test_checker_rejects_gamma_of_the_wrong_column_tile(name):
    c = _small(name)
    d = cc.make(c, "cpu")
    ref = cc.reference(c, d)
    tile = {"tc": lambda w: w[2], "ps": lambda w: w[1], "simt": lambda w: w[1]}[c["want"][0]](c["want"])   # CTA tile width
    d["gamma"] = torch.roll(d["gamma"], tile % c["C_out"] or c["C_out"] // 2)
    assert not cc.check(c, opref.store(cc.reference(c, d), c["out_dtype"]), ref)[0]


@pytest.mark.parametrize("name", [n for n in SELF_CHECK if cc.CASES[n]["out_dtype"] == cabi.TF32])
def test_checker_rejects_a_dropped_tf32_store_rounding(name):
    c = _small(name)
    d = cc.make(c, "cpu")
    ref = cc.reference(c, d)
    assert not cc.check(c, ref.to(torch.float32), ref)[0]
