"""The constructor space of the lowered backbones (tests/backbone_space.py) on the interpreter (tests/emulator.py): every
case the lowering serves matches the float64 module within mlp_programs.LOWERING_TOL in fp32, TF32 and bf16, the library's
host-side queries refuse exactly the cases labelled "refused", and every case the module cannot run or the lowering
declines raises ``Unsupported`` and sends ``sample()`` to the PyTorch loop."""
import inspect
import re

import pytest
import torch

import backbone_space as bs
import emulator
import mlp_programs as mp
from cleandiffuser_b200.engine import cabi, lower, runtime

BATCH = 16
LOWERED = [n for n, c in bs.CASES.items() if not c["want"].startswith("unsupported")]
DECLINED = [n for n, c in bs.CASES.items() if c["want"].startswith("unsupported")]


@pytest.fixture
def programs(monkeypatch):
    """runs every program on the interpreter; the operator lists handed to it, in order"""
    emulator.emulate(monkeypatch)
    monkeypatch.delenv("CDS_BRANCHES", raising=False)
    made, inner = [], runtime._make_handle
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: made.append(list(ops)) or inner(device, ops, n))
    return made


@pytest.mark.parametrize("math_mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("name", LOWERED)
def test_lowered_backbone_matches_the_fp64_module(name, math_mode, programs, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math_mode)
    case = bs.CASES[name]
    net = bs.build(case)
    x, t, cond = bs.inputs(case, BATCH)
    y = runtime.engine_forward(net, x, t, cond)
    err = bs.rel_err(y, bs.reference(net, case, x, t, cond))
    assert err <= mp.LOWERING_TOL[math_mode], (name, case["ctor"], err)
    assert bs.library_outcome(programs[-1]) == case["want"], (name, case["ctor"])


def _raise_line(exc):
    tb = exc.__traceback__
    while tb.tb_next is not None:
        tb = tb.tb_next
    return tb.tb_frame.f_code.co_filename, tb.tb_lineno


@pytest.mark.parametrize("name", DECLINED)
def test_declined_backbone_raises_unsupported_and_sample_falls_back(name, programs, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "fp32")
    monkeypatch.delenv("CDS_BACKEND", raising=False)
    case = bs.CASES[name]
    text = case["want"][len("unsupported: "):]
    net = bs.build(case)
    x, t, cond = bs.inputs(case, BATCH)
    with pytest.raises(lower.Unsupported, match=re.escape(text)):
        runtime.engine_forward(net, x, t, cond)
    a = bs.agent(case, net, "cpu", 4)
    calls, falls = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
    try:
        with torch.no_grad():
            bs.sample(a, case, BATCH, 2, "cpu")
    except Exception:                        # the PyTorch loop of a module that cannot run raises its own error
        pass
    assert runtime.STATS["engine_calls"] == calls
    assert runtime.STATS["fallbacks"] == falls + 1 and text in runtime.STATS["last_fallback_reason"]
    assert not programs


def _backbone_raises():
    """(file, line) of every ``raise Unsupported`` in lower_denoiser and the backbone lowerings it dispatches to"""
    fns = [lower._lower_conv_block, lower._unet_body, lower.lower_janner, lower.lower_chi, lower.lower_dql,
           lower.lower_idql, lower.lower_sfbc, lower.lower_pearce, lower.lower_dit, lower.lower_chitransformer,
           lower.lower_denoiser]
    out = set()
    for fn in fns:
        src, first = inspect.getsourcelines(fn)
        out |= {(inspect.getsourcefile(fn), first + i) for i, line in enumerate(src) if "raise Unsupported(" in line}
    return out


def test_every_unsupported_reason_is_reached():
    reached = set()
    for name in DECLINED:
        case = bs.CASES[name]
        net = bs.build(case)
        p = lower.Program(torch.device("cpu"), BATCH, 1, cabi.MATH_FP32)
        L = case["x"][0] if len(case["x"]) == 2 else 1
        with pytest.raises(lower.Unsupported) as e:
            lower.lower_denoiser(p, net, lower.View(p.buf(BATCH, *case["x"]), L, case["x"][-1]), case["x"],
                                 case["cond"] is not None, 0)
        reached.add(_raise_line(e.value))
    want = _backbone_raises()
    assert len(want) >= 18
    assert want <= reached, sorted(want - reached)


def test_the_table_reaches_the_new_axes():
    """the values the case table exists for: every timestep embedding, taps 3 / 5 / 7, one to four UNet stages, GroupNorm
    widths below 32 channels (conv_simt in every math mode), horizons up to 256, DiT1d's head_dim 16 / 32 / 64 on both sides
    of L = 128, x_t widths on and off the 16 / 32 channel grid"""
    served = [c for c in bs.CASES.values() if c["want"] == "served"]
    unets = [c for c in served if c["kind"] in ("JannerUNet1d", "ChiUNet1d")]
    assert {c["ctor"]["kernel_size"] for c in unets} == {3, 5, 7}
    assert {len(c["ctor"]["dim_mult"]) for c in unets} == {1, 2, 3, 4}
    assert {c["ctor"]["model_dim"] for c in unets} >= {8, 16, 24, 32}
    assert {c["x"][0] for c in unets if c["kind"] == "JannerUNet1d"} >= {4, 8, 32, 64, 128}
    assert {c["x"][0] for c in bs.CASES.values() if c["kind"] in ("JannerUNet1d", "ChiUNet1d")} >= {256}
    assert {c["x"][-1] % 32 == 0 for c in unets} == {True, False} and {c["x"][-1] % 16 for c in unets} > {0}
    assert {(c["cond"] is None, c["ctor"].get("cond_predict_scale")) for c in unets} >= {(True, None), (False, True),
                                                                                         (False, False)}
    dits = {(c["ctor"]["d_model"] // c["ctor"]["n_heads"], c["x"][0] > 128) for c in served if c["kind"] == "DiT1d"}
    assert dits == {(hd, long) for hd in (16, 32, 64) for long in (False, True)}
    assert {c["ctor"].get("timestep_emb_type") for c in served} - {None} == set(bs.EMB_TYPES)
    assert {c["t"] for c in served} == {"int", "float"}
    assert {c["ctor"]["n_blocks"] for c in served if c["kind"] == "IDQLMlp"} == {1, 2, 3, 5}
    assert len({c["ctor"]["hidden_dims"] for c in served if c["kind"] == "SfBCUNet"}) == 5
    assert {c["ctor"]["To"] for c in served if c["kind"] == "PearceMlp"} == {1, 2, 3}
    chit = [c for c in served if c["kind"] == "ChiTransformer"]
    assert {c["ctor"]["Ta"] for c in chit} >= {1, 16, 33} and {c["ctor"]["To"] for c in chit} >= {1, 8}
    assert {c["ctor"]["d_model"] // c["ctor"]["nhead"] for c in chit} == {32, 64}
    assert 150 <= len(bs.CASES) <= 300
