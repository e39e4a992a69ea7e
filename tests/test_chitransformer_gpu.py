"""ChiTransformer on the H100: CDS_OP_MHA against fp64, the lowered network against the fp32 module, and whole sample()
calls against the PyTorch loop.

- Every case of tests/mha_cases.py runs through ``cds_run_op`` with each input dtype, each value pattern and each output
  dtype, under the term-by-term bound of mha_cases.bound; NaN padding around the output stays untouched, two runs give the
  same bits, and a sub-batch starting at trajectory 1 (odd element offsets) gives the same bits.
- ``engine_forward`` at the pipeline shapes and the edge shape in all three math modes, with CDS_FUSE_LN on and off.
- ``sample()`` through the legacy DDPM class (the dp_* pipelines' agent) and DiscreteDiffusionSDE at the three pipeline
  shapes, per-GPU batch 2048 and batch 1, against the PyTorch loop on the same noise; the engine must serve every call.
- A model in train mode with dropout falls back to the PyTorch loop and gives its result.
At the end the module prints each family's largest error as a fraction of its bound."""
import numpy as np
import pytest
import torch

import chi_cases as cc
import mha_cases as mc
import opref
from cleandiffuser_b200.diffusion import DDPM, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import ChiTransformer
from cleandiffuser_b200.testing import NoiseTape, synth_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SPARE = 1024            # NaN elements after the output
WORST = {}              # family -> (largest error / bound, case)
# (max-abs, mean-abs) relative to the output scale max(1, mean |ref|): tests/test_baseline_configs_gpu.py's TOL for the tensor-
# core programs, 1e-4 for fp32 programs
TOL = {"tf32": (2e-2, 2e-3), "bf16": (2.5e-1, 2.5e-2), "fp32": (1e-4, 1e-4)}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    WORST.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print()
        for fam, (frac, name) in sorted(WORST.items()):
            print(f"[chitransformer] {fam}: largest error = {frac:.3f} of the bound ({name})")


def _record(fam, frac, name):
    if frac > WORST.get(fam, (-1.0, ""))[0]:
        WORST[fam] = (frac, name)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


# ---------------------------------------------------------------------------------------------------------------- CDS_OP_MHA
def _launch(c, inp, in_dtype, out_dtype, first=0):
    """run the case on trajectories [first, B) into a fresh NaN-filled output buffer: (buffer, (B, Lq, C) output view)"""
    B, Lq, C = c["B"], c["Lq"], c["heads"] * c["hd"]
    n = B * Lq * (C + 2)
    buf = torch.full((n + SPARE,), float("nan"), dtype=mc.TORCH_DT[out_dtype], device=DEV)
    rows = buf[:n].view(B, Lq, C + 2)
    esz_in = 2 if in_dtype == cabi.BF16 else 4
    esz_out = buf.element_size()
    qb, sb, pb = inp["qbuf"], inp["stepbuf"], inp["sampbuf"]
    ptrs = (qb[first].data_ptr() + esz_in * mc.Q_OFF,
            0 if sb is None else sb.data_ptr(),
            0 if pb is None else pb[first].data_ptr() + esz_in * mc.KV_OFF,
            rows[first].data_ptr() + esz_out * mc.OUT_OFF)
    op = mc.descriptor(c, in_dtype, out_dtype, ptrs, B=B - first)
    cabi.run_op(0, op, mc.ITER, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return buf, rows


def _outside_untouched(buf, rows, C, first=0):
    gap = rows.clone()
    gap[first:, :, mc.OUT_OFF:mc.OUT_OFF + C] = float("nan")
    return bool(torch.isnan(gap.float()).all() and torch.isnan(buf[rows.numel():].float()).all())


@pytest.mark.parametrize("in_dtype", mc.IN_DTYPES, ids=["f32", "tf32", "bf16"])
@pytest.mark.parametrize("name", list(mc.CASES))
def test_mha_case_matches_fp64(name, in_dtype):
    c = mc.CASES[name]
    C = c["heads"] * c["hd"]
    fam = f"mha {'bf16' if in_dtype == cabi.BF16 else 'f32'} in"
    for mode in mc.MODES:
        inp = mc.make(c, mode, in_dtype, DEV)
        ref = mc.reference(c, inp)
        y32 = None
        for od in mc.OUTS:
            buf, rows = _launch(c, inp, in_dtype, od)
            assert _outside_untouched(buf, rows, C), f"{mode} out={od}: a write outside the output"
            y = rows[..., mc.OUT_OFF:mc.OUT_OFF + C].float()
            ok, frac, msg = mc.check(c, y, inp["q"], inp["kv"], ref, od)
            _record(fam, frac, f"{name} {mode} out={od}")
            assert ok, f"{mode} out={od}: {msg}"
            if od == cabi.F32:
                y32 = y
            else:
                assert torch.equal(_bits(opref.store(y32, od).to(mc.TORCH_DT[od])), _bits(y.to(mc.TORCH_DT[od]))), \
                    f"{mode}: out={od} is not the rounding of the kernel's fp32 output"
        if mode != "n0.5":
            continue
        full = _launch(c, inp, in_dtype, cabi.F32)[1]
        again = _launch(c, inp, in_dtype, cabi.F32)[1]
        assert torch.equal(_bits(full), _bits(again)), "two runs differ"
        if c["B"] > 1:
            buf, sub = _launch(c, inp, in_dtype, cabi.F32, first=1)
            assert _outside_untouched(buf, sub, C, first=1) and torch.isnan(sub[0]).all()
            assert torch.equal(_bits(sub[1:]), _bits(full[1:])), "a sub-batch at a trajectory offset differs"


# ---------------------------------------------------------------------------------------------------------------- network
def _net(ctor, seed=0):
    net = ChiTransformer(**ctor)
    net.load_state_dict(cc.weights(net.state_dict(), synth_state_dict, seed=seed))
    return net.eval().to(DEV)


FWD_SHAPES = ["pusht", "kitchen", "edge"]


@pytest.mark.parametrize("fuse", ["1", "0"])
@pytest.mark.parametrize("math", ["tf32", "bf16", "fp32"])
@pytest.mark.parametrize("name", FWD_SHAPES)
def test_engine_forward_matches_module(name, math, fuse, monkeypatch):
    monkeypatch.setenv("CDS_FUSE_LN", fuse)
    torch.backends.cuda.matmul.allow_tf32 = False
    ctor = cc.NETS[name]
    net = _net(ctor)
    B = 37
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, ctor["Ta"], ctor["act_dim"], generator=g).to(DEV)
    cond = torch.randn(B, ctor["To"], ctor["obs_dim"], generator=g).to(DEV)
    t = torch.tensor([17], device=DEV)
    mode = {"tf32": cabi.MATH_TF32_TC, "bf16": cabi.MATH_BF16_TC, "fp32": cabi.MATH_FP32}[math]
    for c in (cond, None):
        with torch.no_grad():
            want = net(x, t.expand(B), c)
        got = runtime.engine_forward(net, x, t, c, math=mode)
        scale = max(1.0, want.abs().mean().item())
        err = (got - want).abs() / scale
        assert torch.isfinite(got).all()
        mx, mean = err.max().item(), err.mean().item()
        _record(f"forward {math}", mx / TOL[math][0], f"{name} fuse={fuse} cond={c is not None}")
        assert mx < TOL[math][0] and mean < TOL[math][1], (mx, mean)


# ---------------------------------------------------------------------------------------------------------------- sample()
SAMPLE_SHAPES = ["pusht", "robomimic", "kitchen"]


def _agent(kind, net, ctor):
    x_max = torch.ones((1, ctor["Ta"], ctor["act_dim"]), device=DEV)
    nc = IdentityCondition(dropout=0.0)
    if kind == "legacy":
        agent = DDPM(net, nc, x_max=x_max, x_min=-x_max, diffusion_steps=10, device=DEV)
        kw = dict(sample_steps=10)
    else:
        agent = DiscreteDiffusionSDE(net, nc, x_max=x_max, x_min=-x_max, diffusion_steps=100, device=DEV)
        kw = dict(solver="ddpm", sample_steps=10)
    agent.model_ema.eval()
    return agent, kw


def _sample(agent, kw, prior, cond, backend, monkeypatch, draws=None, **extra):
    monkeypatch.setenv("CDS_BACKEND", backend)
    tape = NoiseTape(draws)
    with tape.active(), torch.no_grad():
        x, _ = agent.sample(prior, n_samples=prior.shape[0], condition_cfg=cond, w_cfg=1.0, **dict(kw, **extra))
    torch.cuda.synchronize()
    return x, tape.draws


@pytest.mark.parametrize("batch", [2048, 1])
@pytest.mark.parametrize("kind", ["legacy", "sde"])
@pytest.mark.parametrize("name", SAMPLE_SHAPES)
def test_sample_matches_pytorch_loop(name, kind, batch, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "tf32")
    torch.backends.cuda.matmul.allow_tf32 = False
    ctor = cc.NETS[name]
    agent, kw = _agent(kind, _net(ctor, seed=1), ctor)
    g = torch.Generator().manual_seed(batch)
    prior = torch.zeros(batch, ctor["Ta"], ctor["act_dim"], device=DEV)
    cond = torch.randn(batch, ctor["To"], ctor["obs_dim"], generator=g).to(DEV)
    calls, falls = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
    torch.manual_seed(5)
    x, draws = _sample(agent, kw, prior, cond, "cuda", monkeypatch)
    assert runtime.STATS["engine_calls"] == calls + 1 and runtime.STATS["fallbacks"] == falls, runtime.STATS
    ref, _ = _sample(agent, kw, prior, cond, "torch", monkeypatch, draws=draws)
    assert runtime.STATS["engine_calls"] == calls + 1
    err = ((x - ref).abs() / max(1.0, ref.abs().mean().item())).cpu()
    assert torch.isfinite(x).all()
    mx, mean, p99 = err.max().item(), err.mean().item(), float(np.quantile(err.numpy().ravel(), 0.99))
    outliers = float((err > TOL["tf32"][0]).float().mean())
    _record("sample tf32 (p99)", p99 / TOL["tf32"][0], f"{name} {kind} B={batch}")
    # the prediction is clipped to [-1, 1] at every step: an element whose clip decision flips at some step is an isolated
    # outlier (as in test_baseline_configs_gpu.py's cfg3), so the max bound sits on the 99th percentile, at most 0.1 % of the
    # elements may exceed it, and the max gets 0.5 (seen on an H100 at batch 2048: 0.28, with p99 5e-3 and mean 5e-4)
    assert p99 < TOL["tf32"][0] and mean < TOL["tf32"][1] and outliers < 1e-3 and mx < 0.5, (mx, mean, p99, outliers)


def test_train_mode_falls_back_to_pytorch(monkeypatch):
    ctor = cc.NETS["pusht"]
    net = _net(ctor)
    agent, kw = _agent("legacy", net, ctor)
    agent.model.train()
    prior = torch.zeros(16, ctor["Ta"], ctor["act_dim"], device=DEV)
    cond = torch.randn(16, ctor["To"], ctor["obs_dim"], device=DEV)
    falls = runtime.STATS["fallbacks"]
    torch.manual_seed(9)
    x, _ = _sample(agent, kw, prior, cond, "auto", monkeypatch, use_ema=False)
    assert runtime.STATS["fallbacks"] == falls + 1 and "train mode" in runtime.STATS["last_fallback_reason"]
    torch.manual_seed(9)
    ref, _ = _sample(agent, kw, prior, cond, "torch", monkeypatch, use_ema=False)
    assert torch.equal(x, ref)


def test_dp_pusht_call_sequence_is_served(monkeypatch):
    """pipelines/dp_pusht.py with nn=chi_transformer, diffusion=ddpm: the network, agent and sample() call as the pipeline
    writes them (obs_dim 5, action_dim 2, horizon 10, obs_steps 2, sample_steps 5, one environment)."""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    device, horizon, action_dim, obs_dim, obs_steps, sample_steps, num_envs = DEV, 10, 2, 5, 2, 5, 1
    nn_diffusion = ChiTransformer(action_dim, obs_dim, horizon, obs_steps, d_model=256, nhead=4, num_layers=4,
                                  timestep_emb_type="positional").to(device)
    nn_condition = IdentityCondition(dropout=0.0).to(device)
    x_max = torch.ones((1, horizon, action_dim), device=device) * +1.0
    x_min = torch.ones((1, horizon, action_dim), device=device) * -1.0
    agent = DDPM(nn_diffusion=nn_diffusion, nn_condition=nn_condition, device=device, diffusion_steps=sample_steps,
                 x_max=x_max, x_min=x_min, optim_params={"lr": 1e-4})
    agent.eval()
    calls, falls = runtime.STATS["engine_calls"], runtime.STATS["fallbacks"]
    for _ in range(3):
        condition = torch.randn(num_envs, obs_steps, obs_dim, device=device)
        prior = torch.zeros((num_envs, horizon, action_dim), device=device)
        with torch.no_grad():
            naction, _ = agent.sample(prior=prior, n_samples=num_envs, sample_steps=sample_steps, solver=None,
                                      condition_cfg=condition, w_cfg=1.0, use_ema=True)
        assert naction.shape == (num_envs, horizon, action_dim) and torch.isfinite(naction).all()
    assert runtime.STATS["engine_calls"] == calls + 3 and runtime.STATS["fallbacks"] == falls, runtime.STATS
