"""ChiTransformer without a GPU: the module against the reference's goldens (tests/golden/chitransformer.npz), the lowered
program executed by the numpy interpreter of the C ABI (tests/emulator.py, with CDS_OP_MHA from tests/mha_ref.py), the cases the lowering declines, and the host
side of CDS_OP_MHA (which instantiation each case of tests/mha_cases.py reaches, the refusals, and that the error bound
rejects typical kernel faults)."""
import os

import numpy as np
import pytest
import torch

import chi_cases as cc
import emulator
import mha_cases as mc
import mha_ref
from cleandiffuser_b200.diffusion import DDPM, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.engine.lower import Program, Unsupported, View, lower_denoiser
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import ChiTransformer
from cleandiffuser_b200.testing import NoiseTape, synth_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "chitransformer.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN, allow_pickle=False)


def _net(ctor):
    net = ChiTransformer(**ctor)
    net.load_state_dict(cc.weights(net.state_dict(), synth_state_dict))
    return net.eval()


def _scale(want):
    return max(1.0, float(np.abs(want).mean()))


@pytest.mark.parametrize("name", list(cc.NETS))
def test_state_dict_matches_reference(gold, name):
    sd = ChiTransformer(**cc.NETS[name]).state_dict()
    got = ["%s|%s" % (k, ",".join(map(str, v.shape))) for k, v in sd.items()]
    assert got == list(gold[name + "/keys"])


@pytest.mark.parametrize("name", list(cc.NETS))
def test_module_forward_matches_reference(gold, name):
    net = _net(cc.NETS[name])
    x, t, cond = cc.net_inputs(cc.NETS[name])
    with torch.no_grad():
        y, y0 = net(x, t, cond), net(x, t, None)
    for got, key in ((y, "/y"), (y0, "/y_uncond")):
        want = gold[name + key]
        np.testing.assert_allclose(got.numpy(), want, rtol=0, atol=1e-5 * _scale(want))


@pytest.fixture
def emulate(monkeypatch):
    monkeypatch.setattr(runtime, "_device_ok", lambda device: True)
    owners = emulator.record_owners(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setattr(runtime, "_make_handle", lambda device, ops, n: mha_ref.Handle(ops, n, owners()))
    monkeypatch.setenv("CDS_BACKEND", "cuda")       # any fallback to the PyTorch loop is a failure here


# (max, mean) of |engine - golden| relative to the output scale; fp32 programs are exact up to summation order, TF32 / bf16
# programs are held to the bounds of the other lowered transformers (tests/test_lowering_cpu.py)
EMU_TOL = {"fp32": (2e-5, 2e-6), "tf32": (2e-2, 2e-3), "bf16": (0.08, 0.015)}


@pytest.mark.parametrize("math", list(EMU_TOL))
@pytest.mark.parametrize("name", list(cc.NETS))
def test_lowered_forward_matches_reference(gold, emulate, monkeypatch, name, math):
    monkeypatch.setenv("CDS_MATH", math)
    net = _net(cc.NETS[name])
    x, t, cond = cc.net_inputs(cc.NETS[name])
    for i in range(cc.BATCH):
        for c, key in ((cond, "/y"), (None, "/y_uncond")):
            want = gold[name + key][i]
            err = np.abs(runtime.engine_forward(net, x, t[i:i + 1], c)[i].numpy() - want) / _scale(want)
            assert err.max() < EMU_TOL[math][0] and err.mean() < EMU_TOL[math][1], (name, key, i, err.max(), err.mean())


def _agent(spec):
    net = _net(cc.SAMPLE_NET)
    _, _, x_max, x_min = cc.sampler_inputs()
    if spec["kind"] == "legacy":
        agent = DDPM(net, IdentityCondition(dropout=0.0), x_max=x_max, x_min=x_min, diffusion_steps=spec["T"], device="cpu")
        kw = dict(sample_steps=spec["T"])
    else:
        agent = DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), x_max=x_max, x_min=x_min, diffusion_steps=spec["T"],
                                     device="cpu")
        kw = dict(solver=spec["solver"], sample_steps=spec["steps"])
    agent.model_ema.eval()
    return agent, dict(kw, n_samples=cc.SAMPLE_BATCH, use_ema=True, w_cfg=spec["w_cfg"])


@pytest.mark.parametrize("name", list(cc.SAMPLERS))
def test_lowered_sampler_matches_reference(gold, emulate, monkeypatch, name):
    monkeypatch.setenv("CDS_MATH", "fp32")
    agent, kw = _agent(cc.SAMPLERS[name])
    prior, cond, _, _ = cc.sampler_inputs()
    tape = NoiseTape([gold[f"{name}/z{j}"] for j in range(int(gold[name + "/n_draws"]))])
    before = runtime.STATS["engine_calls"]
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(prior, condition_cfg=cond, **kw)
    assert runtime.STATS["engine_calls"] == before + 1 and tape.pos == len(tape.draws)
    np.testing.assert_allclose(x0.numpy(), gold[name + "/x0"], rtol=1e-4, atol=3e-4)


def _lower(net, horizon=None, math=cabi.MATH_FP32):
    L = horizon or net.T
    p = Program(torch.device("cpu"), 2, 1, math)
    xin = p.buf(2, L, net.head.out_features)
    return lower_denoiser(p, net, View(xin, L, net.head.out_features), (L, net.head.out_features), True, 0), p


def test_lowering_declines_what_it_cannot_run():
    ctor = dict(act_dim=2, obs_dim=5, Ta=10, To=2, d_model=64, nhead=2, num_layers=1)
    _lower(ChiTransformer(**ctor).eval())
    with pytest.raises(Unsupported, match="train mode"):
        _lower(ChiTransformer(**ctor).train())
    _lower(ChiTransformer(**dict(ctor, p_drop_attn=0.0)).train())           # no dropout anywhere: train mode computes the same
    with pytest.raises(Unsupported, match="n_cond_layers"):
        _lower(ChiTransformer(**ctor, n_cond_layers=1).eval())
    with pytest.raises(Unsupported, match="masks"):
        _lower(ChiTransformer(**ctor).eval(), horizon=8)
    net = ChiTransformer(**ctor).eval()
    with torch.no_grad():
        net.memory_mask.zero_()
    with pytest.raises(Unsupported, match="masks"):
        _lower(net)


def test_lowering_program_shape():
    """Per layer: 3 LayerNorms, 6 Linears, 2 attentions; the cross-attention reads the per-iteration and per-trajectory k|v
    tables of its own layer, with the memory mask."""
    net = ChiTransformer(act_dim=2, obs_dim=5, Ta=10, To=2, d_model=64, nhead=2, num_layers=3).eval()
    _, p = _lower(net, math=cabi.MATH_TF32_TC)
    kinds = [op.kind for op in p.ops]
    mhas = [op.u.mha for op in p.ops if op.kind == cabi.OP_MHA]
    assert kinds.count(cabi.OP_MHA) == 6 and kinds.count(cabi.OP_LNMOD) == 3 * 3 + 1
    assert all(m.Lq == 10 and m.C == 64 and m.heads == 2 and m.in_dtype == cabi.TF32 for m in mhas)
    self_, cross = mhas[0::2], mhas[1::2]
    assert all(m.Lk == 10 and m.masked and m.diag == 0 and not m.kv_step and m.kv_sample == m.q + 4 * 64 for m in self_)
    assert all(m.Lk == 3 and m.masked and m.diag == 1 and m.kv_step and m.kv_sample for m in cross)
    assert len({m.kv_step for m in cross}) == 3 and all(m.kv_step_stride == 3 * 3 * 128 for m in cross)
    convs = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV]
    assert all(c.math == cabi.MATH_TF32_TC for c in convs) and len(convs) == 1 + 6 * 3 + 1


# ---------------------------------------------------------------------------------------------------------------- CDS_OP_MHA
def test_mha_cases_reach_every_instantiation():
    reached = set()
    for c in mc.CASES.values():
        for dt in mc.IN_DTYPES:
            ch = cabi.mha_choice(mc.descriptor(c, dt, cabi.F32).u.mha)
            assert ch["hpl"] == c["hd"] // 32 and ch["bf16"] == (dt == cabi.BF16), (c["name"], ch)
            reached.add((ch["hpl"], ch["bf16"]))
    assert reached == {(h, b) for h in range(1, 9) for b in (False, True)}


def test_mha_refusals():
    for (B, Lq, Lk, heads, hd), code in mc.REFUSED:
        c = mc.case("refused", B, Lq, Lk, heads, hd, 0, "sample")
        with pytest.raises(cabi.CdsError) as e:
            cabi.mha_choice(mc.descriptor(c, cabi.F32, cabi.F32).u.mha)
        assert e.value.code == code, ((B, Lq, Lk, heads, hd), e.value.code)
    biggest = mc.case("largest", 1, 64, 64, 2, 256, None, "both")
    assert cabi.mha_choice(mc.descriptor(biggest, cabi.BF16, cabi.F32).u.mha) == {"hpl": 8, "bf16": True}


def test_mha_bound_accepts_reference_and_rejects_faults():
    """The checker passes the fp64 reference stored in fp32 and rejects, on every case where the fault changes the result:
    a mask off by one, k and v swapped, and heads read with the wrong stride."""
    n_rejected = {"mask": 0, "swap": 0, "heads": 0}
    for c in mc.CASES.values():
        if c["B"] > 8:
            continue
        inp = mc.make(c, "n0.5", cabi.F32, "cpu")
        q, kv = inp["q"], inp["kv"]
        ref = mc.reference(c, inp)
        ok, _, msg = mc.check(c, ref.to(torch.float32), q, kv, ref, cabi.F32)
        assert ok, msg
        C = q.shape[-1]
        faults = {"swap": mha_ref.mha(q, torch.cat([kv[..., C:], kv[..., :C]], -1), c["heads"], c["diag"]),
                  "heads": _wrong_head_stride(q, kv, c)}
        if c["diag"] is not None:
            faults["mask"] = mha_ref.mha(q, kv, c["heads"], c["diag"] + 1)
        for kind, y in faults.items():
            if torch.equal(y, ref):
                continue
            ok, _, msg = mc.check(c, y.to(torch.float32), q, kv, ref, cabi.F32)
            assert not ok, f"{kind} fault accepted: {msg}"
            n_rejected[kind] += 1
    assert all(n > 0 for n in n_rejected.values()), n_rejected


def _wrong_head_stride(q, kv, c):
    """heads interleaved (channel d of head h at d * heads + h) instead of contiguous (h * hd + d)"""
    B, Lq, C = q.shape
    H, hd = c["heads"], c["hd"]
    perm = torch.arange(C).reshape(hd, H).t().reshape(-1)
    kvp = torch.cat([kv[..., :C][..., perm], kv[..., C:][..., perm]], -1)
    y = mha_ref.mha(q[..., perm], kvp, H, c["diag"])
    out = torch.empty_like(y)
    out[..., perm] = y
    return out


def test_alias_package_exports_chitransformer():
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    snippet = ("from cleandiffuser.nn_diffusion import ChiTransformer\nimport cleandiffuser_b200\n"
               "assert ChiTransformer is cleandiffuser_b200.nn_diffusion.ChiTransformer\nprint('ok')")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(root, "compat"), root]))
    out = subprocess.run([sys.executable, "-c", snippet], env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stderr[-2000:]
