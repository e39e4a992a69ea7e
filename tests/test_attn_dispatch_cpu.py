"""CPU checks of the operator-level attention case table (tests/attn_cases.py): every case reaches the kernel instantiation
it names (cds_attn_choice, pure host logic), the table covers all 20 instantiations, the refusals hold, and the checker of
tests/test_attention_gpu.py accepts the fp64 reference and rejects three typical kernel faults."""
import math
import os
import re

import pytest
import torch

import attn_cases as ac
import opref
from cleandiffuser_b200.engine import cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cleandiffuser_b200", "csrc")


def _instantiations():
    f32 = re.findall(r"CDS_ATTN_CASE\((\d+)\)\n", open(os.path.join(CSRC, "attention.cuh")).read())
    nt = re.findall(r"CDS_ATTN_NT\((\d+)\)", open(os.path.join(CSRC, "attention_tma.cuh")).read())
    return {ac.key("f32", int(h)) for h in f32} | {ac.key("tma", int(n)) for n in nt} | {ac.key("bf16_mma")}


@pytest.mark.parametrize("name", list(ac.CASES))
def test_case_reaches_its_instantiation(name):
    c = ac.CASES[name]
    for od in c["outs"]:
        assert ac.choice_key(cabi.attn_choice(ac.fake_descriptor(c, od).u.attn)) == c["want"], od


def test_cases_cover_every_instantiation():
    inst = _instantiations()
    assert len(inst) == 20
    assert {c["want"] for c in ac.CASES.values()} == inst


def test_tma_cases_cover_every_residue_and_both_grid_regimes():
    tma = [c for c in ac.CASES.values() if c["want"][0] == "tma"]
    assert {c["L"] % 16 for c in tma} == set(range(16))
    assert {c["L"] for c in tma} >= set(range(113, 129))
    assert any(c["B"] * c["heads"] < 2 * ac.SMS for c in tma)
    assert any(c["B"] * c["heads"] >= 3 * 2 * ac.SMS for c in tma)


def test_fp32_kernel_cases_exceed_48kb_of_shared_memory():
    for hd in (16, 32, 64):
        smem = [cabi.attn_choice(ac.fake_descriptor(c).u.attn)["smem"] for c in ac.CASES.values() if c["want"] == ac.key("f32", hd)]
        assert max(smem) > 48 * 1024 and min(smem) < 48 * 1024, (hd, smem)


def _refused(c, **kw):
    op = ac.fake_descriptor(c)
    for k, v in kw.items():
        setattr(op.u.attn, k, v)
    with pytest.raises(cabi.CdsError) as e:
        cabi.attn_choice(op.u.attn)
    return e.value.code


def test_refusals():
    f32 = ac.CASES["f32_hd16_L100_f32"]
    bf16 = ac.CASES["bf16mma_L100"]
    for hd in (8, 128):
        assert _refused(f32, C=hd * f32["heads"]) == ERR_UNSUPPORTED
    for hd, L in ac.MAX_L.items():
        c = dict(f32, hd=hd, L=L)
        assert cabi.attn_choice(ac.fake_descriptor(c).u.attn) == {"family": "f32", "param": hd, "hd": hd, "smem": 200 * 1024}
        assert _refused(c, L=L + 1) == ERR_UNSUPPORTED
    assert _refused(bf16, L=129) == ERR_UNSUPPORTED
    assert _refused(bf16, C=64 * bf16["heads"]) == ERR_UNSUPPORTED
    assert _refused(bf16, qkv=(1 << 20) + 8) == ERR_UNSUPPORTED
    assert _refused(f32, heads=0) == ERR_INVALID
    assert _refused(f32, C=16 * f32["heads"] + 1) == ERR_INVALID


ERR_INVALID, ERR_UNSUPPORTED = -1, -3      # cds_status


# ---- the checker itself, with the fp64 reference standing in for the kernel (one trajectory, CPU)
def _ref(c, qkv):
    return opref.attn(qkv, c["heads"], c["qkv_dtype"])


def _padded_keys_as_zero(c, qkv):
    """softmax over ceil16(L) keys, the padding keys with score 0 and v = 0"""
    pad = -c["L"] % 16
    B, L, C3 = qkv.shape
    z = torch.zeros(B, pad, C3, dtype=qkv.dtype)
    return _ref(c, torch.cat([qkv, z], 1))[:, :L]


def _scale_of_hd32(c, qkv):
    return _ref(c, torch.cat([qkv[..., :c["heads"] * 64] * math.sqrt(64 / 32), qkv[..., c["heads"] * 64:]], -1))


def _next_heads_v(c, qkv):
    C = c["heads"] * c["hd"]
    v = qkv[..., 2 * C:]
    return _ref(c, torch.cat([qkv[..., :2 * C], torch.roll(v, -c["hd"], dims=-1)], -1))


FAULTS = {"padded keys counted with score 0": _padded_keys_as_zero, "1/sqrt(32) scale for head_dim 64": _scale_of_hd32,
          "one head reads the next head's V": _next_heads_v}


@pytest.mark.parametrize("name", list(ac.CASES))
def test_checker_accepts_the_reference_and_rejects_faults(name):
    """each fault that changes the result at the case's shape is rejected in at least one of the value patterns the GPU
    test runs (a lone padding key among 128 shifts a zero-mean output by less than the bf16 P rounding: v100 shows it)"""
    c = ac.CASES[name]
    applies = {"padded keys counted with score 0": c["L"] % 16 != 0,
               "1/sqrt(32) scale for head_dim 64": c["hd"] == 64 and c["L"] > 1,
               "one head reads the next head's V": c["heads"] > 1}
    caught = {f: [] for f, a in applies.items() if a}
    for mode in ac.MODES:
        qkv = ac.make(c, mode, "cpu", B=1)
        ref = _ref(c, qkv)
        for od in c["outs"]:
            ok, frac, msg = ac.check(c, opref.store(ref, od), qkv, ref, od)
            assert ok, f"{mode}: {msg}"
        for fault in caught:
            ok, frac, msg = ac.check(c, opref.store(FAULTS[fault](c, qkv), c["outs"][0]), qkv, ref, c["outs"][0])
            if not ok:
                caught[fault].append(mode)
    assert all(caught.values()), caught
