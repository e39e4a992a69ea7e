"""Parity of the CUDA engine (through the C ABI) against the golden vectors of the reference and the
CPU oracle.  Everything here needs an H100: run with ``-m gpu``."""
import os

import numpy as np
import pytest
import torch

import cases
import oracle.sampler as osamp
from common import oracle_cond_emb, oracle_net, product_net, tape_of
from test_host_golden import build_agent
from cleandiffuser_b200.diffusion import ContinuousConsistencyModel, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import JannerUNet1d
from cleandiffuser_b200.testing import NoiseTape, load_synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# fp32 CUDA-core path: same arithmetic as the fp32 oracle up to summation order / libm rounding
NET_ATOL = 2e-4
SAMPLER_ATOL, SAMPLER_RTOL = 1e-3, 1e-3


@pytest.fixture(autouse=True)
def _force_engine(monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")      # a fallback to PyTorch is a test failure, not a pass
    monkeypatch.setenv("CDS_MATH", "fp32")


def test_library_loaded_from_tree():
    lib = cabi.load()
    assert os.path.samefile(cabi.lib_path(), os.path.join(os.path.dirname(cabi.__file__), "..", "csrc", "libcds.so"))
    assert lib.cds_version() == cabi.ABI_VERSION
    assert lib.cds_device_sm_count(0) > 0


@pytest.mark.parametrize("name", list(cases.NETS))
def test_denoiser_forward_matches_reference(golden, name):
    case = cases.NETS[name]
    net, sd = product_net(case)
    net = net.to(DEV)
    x, t, cond = cases.net_inputs(case)
    cond_emb = None if cond is None else cond.to(DEV)
    want = golden["nets"][name + "/y"]
    for i in range(cases.NET_BATCH):                       # inside sample() t is batch-constant: one run per t
        y = runtime.engine_forward(net, x.to(DEV), t[i:i + 1], cond_emb)
        np.testing.assert_allclose(y[i].cpu().numpy(), want[i], rtol=0, atol=NET_ATOL, err_msg=f"{name} row {i}")


@pytest.mark.parametrize("name", list(cases.sampler_cases()))
def test_sampler_matches_reference(golden, name):
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec, device=DEV)
    for k in ("condition_cfg", "warm_start_reference"):
        if kw.get(k) is not None:
            kw[k] = kw[k].to(DEV)
    before = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["samplers"], name))
    with tape.active(), torch.no_grad():
        x0, log = agent.sample(inp["prior"].to(DEV), **kw)
    assert runtime.STATS["engine_calls"] == before + 1, runtime.STATS
    assert tape.pos == len(tape.draws)
    assert x0.device.type == "cuda" and log["sample_history"] is None
    np.testing.assert_allclose(x0.cpu().numpy(), golden["samplers"][name + "/x0"], rtol=SAMPLER_RTOL, atol=SAMPLER_ATOL)


@pytest.mark.parametrize("steps", [1, 3])
def test_consistency_matches_reference(golden, steps):
    g = golden["consistency"]
    net, _ = product_net(cases.NETS["chi_cm_fourier"])
    cm = ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), x_max=torch.ones(1, 8, 3),
                                    x_min=-torch.ones(1, 8, 3), device=DEV)
    tape = NoiseTape(tape_of(g, f"cm{steps}"))
    before = runtime.STATS["engine_calls"]
    with tape.active(), torch.no_grad():
        x0, _ = cm.sample(torch.zeros(4, 8, 3, device=DEV), n_samples=4, sample_steps=steps,
                          condition_cfg=torch.as_tensor(g[f"cm{steps}/cond"]).to(DEV), w_cfg=1.0)
    assert runtime.STATS["engine_calls"] == before + 1
    np.testing.assert_allclose(x0.cpu().numpy(), g[f"cm{steps}/x0"], rtol=SAMPLER_RTOL, atol=SAMPLER_ATOL)


def _cfg2_agent(T):
    net = load_synth(JannerUNet1d(14, model_dim=32, emb_dim=32, kernel_size=5, dim_mult=[1, 2, 2, 2]), seed=0)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    mask = torch.zeros(32, 14)
    mask[0, :11] = 1.
    return DiscreteDiffusionSDE(net, None, fix_mask=mask, predict_noise=False, diffusion_steps=T, device=DEV), sd, mask


def test_cfg2_full_batch_properties_and_oracle():
    """BASELINE config 2 shapes (B=4096, H=32, d=14; 10 DDPM steps to keep the oracle leg short):
    size-independent properties at full batch + oracle comparison on a slice."""
    T, B = 10, 4096
    agent, sd, mask = _cfg2_agent(T)
    g = torch.Generator().manual_seed(1)
    prior = torch.zeros(B, 32, 14)
    prior[:, 0, :11] = torch.randn(B, 11, generator=g)
    tape = NoiseTape()
    with tape.active(), torch.no_grad():
        x_full, _ = agent.sample(prior.to(DEV), solver="ddpm", n_samples=B, sample_steps=T, temperature=0.5)
    x_full = x_full.cpu()
    assert torch.isfinite(x_full).all()
    # (a) the fixed portion is re-imposed exactly
    assert torch.equal(x_full[:, 0, :11], prior[:, 0, :11])
    # (b) trajectories are independent: a 96-row sub-batch with the same noise gives the same bits
    sub = slice(1000, 1096)
    tape_sub = NoiseTape([z[sub] for z in tape.draws])
    with tape_sub.active(), torch.no_grad():
        x_sub, _ = agent.sample(prior[sub].to(DEV), solver="ddpm", n_samples=96, sample_steps=T, temperature=0.5)
    assert torch.equal(x_sub.cpu(), x_full[sub])
    # (c) oracle on 16 trajectories
    pick = slice(2040, 2056)
    fn = oracle_net(cases.NETS["janner_cfg2"], sd)
    with torch.no_grad():
        x_ref = osamp.sample_discrete(fn, prior[pick], osamp.Tape([z[pick].numpy() for z in tape.draws]), T=T, steps=T,
                                      solver="ddpm", temperature=0.5, fix_mask=mask[None], predict_noise=False)
    np.testing.assert_allclose(x_full[pick].numpy(), x_ref.numpy(), rtol=SAMPLER_RTOL, atol=SAMPLER_ATOL)


def test_weights_refresh_after_training_step():
    """Training mutates parameters behind the plan's back; the packed copies must follow (SURVEY 3.4)."""
    spec = cases.sampler_cases()["disc_dx_ddpm_eps"]
    agent, inp, kw = build_agent(spec, device=DEV)
    kw["condition_cfg"] = kw["condition_cfg"].to(DEV)
    kw["use_ema"] = False
    agent.model.eval()

    def run(backend):
        os.environ["CDS_BACKEND"] = backend
        torch.manual_seed(7)
        with torch.no_grad():
            return agent.sample(inp["prior"].to(DEV), **kw)[0]

    a0 = run("cuda")
    with torch.no_grad():
        for p in agent.model["diffusion"].parameters():
            p.add_(0.01 * torch.randn_like(p))
    a1, t1 = run("cuda"), run("torch")
    assert (a1 - a0).abs().max() > 1e-4
    np.testing.assert_allclose(a1.cpu().numpy(), t1.cpu().numpy(), rtol=SAMPLER_RTOL, atol=SAMPLER_ATOL)


def test_smoke_entry():
    import __graft_entry__ as ge
    ge.smoke()


# ------------------------------------------------------------------------------------------------------------------
# tensor-core programs (CDS_MATH=bf16): bf16 operands / activations, fp32 accumulation and fp32 GN/Mish epilogue.
# Stated tolerance vs the fp32 reference (SURVEY 8c, measured by emulation: ~8e-3 relative per forward, no
# compounding over the reverse steps): max-abs 2e-1, mean-abs 2e-2 on O(1) outputs.
BF16_NETS = ["janner_cfg2", "janner_kitchen_cond", "chi_small", "chi_cm_fourier", "dit_small", "dit_pos_uncond"]


@pytest.mark.parametrize("name", BF16_NETS)
def test_denoiser_forward_bf16_tensor_cores(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "bf16")
    case = cases.NETS[name]
    net, _ = product_net(case)
    net = net.to(DEV)
    x, t, cond = cases.net_inputs(case)
    cond_emb = None if cond is None else cond.to(DEV)
    want = golden["nets"][name + "/y"]
    for i in range(cases.NET_BATCH):
        y = runtime.engine_forward(net, x.to(DEV), t[i:i + 1], cond_emb)
        err = np.abs(y[i].cpu().numpy() - want[i])
        assert err.max() < 0.08 and err.mean() < 0.015, (name, i, float(err.max()), float(err.mean()))


def test_cfg2_bf16_tensor_cores_full_batch(monkeypatch):
    monkeypatch.setenv("CDS_MATH", "bf16")
    T, B = 10, 4096
    agent, sd, mask = _cfg2_agent(T)
    g = torch.Generator().manual_seed(1)
    prior = torch.zeros(B, 32, 14)
    prior[:, 0, :11] = torch.randn(B, 11, generator=g)
    tape = NoiseTape()
    with tape.active(), torch.no_grad():
        x_full, _ = agent.sample(prior.to(DEV), solver="ddpm", n_samples=B, sample_steps=T, temperature=0.5)
    x_full = x_full.cpu()
    assert torch.isfinite(x_full).all()
    assert torch.equal(x_full[:, 0, :11], prior[:, 0, :11])
    sub = slice(1024, 1024 + 128)
    tape_sub = NoiseTape([z[sub] for z in tape.draws])
    with tape_sub.active(), torch.no_grad():
        x_sub, _ = agent.sample(prior[sub].to(DEV), solver="ddpm", n_samples=128, sample_steps=T, temperature=0.5)
    assert torch.equal(x_sub.cpu(), x_full[sub])
    pick = slice(2040, 2056)
    fn = oracle_net(cases.NETS["janner_cfg2"], sd)
    with torch.no_grad():
        x_ref = osamp.sample_discrete(fn, prior[pick], osamp.Tape([z[pick].numpy() for z in tape.draws]), T=T, steps=T,
                                      solver="ddpm", temperature=0.5, fix_mask=mask[None], predict_noise=False)
    err = (x_full[pick] - x_ref).abs()
    assert err.max() < 0.2 and err.mean() < 0.02, (float(err.max()), float(err.mean()))


@pytest.mark.parametrize("name", ["disc_dup_ddpm_x0", "cont_ddim_eps", "cont_sde_dpmsolverpp_2M_x0"])
def test_sampler_bf16_tensor_cores_goldens(golden, name, monkeypatch):
    """Reverse loop on the tensor-core programs (once-cast + update-fused bf16 x_t copy + programmatic dependent launch)
    against the reference goldens, with the stated bf16 tolerance; graph replay and direct launches must give the same bits
    (both chain the kernels with programmatic dependent launch: tests/test_program_audit_gpu.py compares them with runs
    that synchronise after every operator)."""
    monkeypatch.setenv("CDS_MATH", "bf16")
    spec = cases.sampler_cases()[name]
    outs = []
    for graph in ("1", "0"):
        monkeypatch.setenv("CDS_GRAPH", graph)
        agent, inp, kw = build_agent(spec, device=DEV)
        for k in ("condition_cfg", "warm_start_reference"):
            if kw.get(k) is not None:
                kw[k] = kw[k].to(DEV)
        tape = NoiseTape(tape_of(golden["samplers"], name))
        with tape.active(), torch.no_grad():
            x0, _ = agent.sample(inp["prior"].to(DEV), **kw)
        outs.append(x0.cpu())
        err = np.abs(x0.cpu().numpy() - golden["samplers"][name + "/x0"])
        assert err.max() < 0.2 and err.mean() < 0.02, (name, graph, float(err.max()), float(err.mean()))
    assert torch.equal(outs[0], outs[1])         # graph replay == direct launches


@pytest.mark.parametrize("math", ["fp32", "bf16", "tf32"])
def test_parallel_branches_give_the_same_bits(math, monkeypatch):
    """CDS_BRANCHES splits the batch into independent kernel chains on parallel streams / graph branches: trajectories are
    independent, so the result must equal the single-chain run bit for bit (graph replay and direct launches)."""
    monkeypatch.setenv("CDS_MATH", math)
    T, B = 6, 2048
    outs = {}
    for branches, graph in (("1", "1"), ("2", "1"), ("2", "0"), ("4", "1")):
        monkeypatch.setenv("CDS_BRANCHES", branches)
        monkeypatch.setenv("CDS_BRANCH_MIN_BATCH", "256")
        monkeypatch.setenv("CDS_GRAPH", graph)
        agent, sd, mask = _cfg2_agent(T)
        g = torch.Generator().manual_seed(1)
        prior = torch.zeros(B, 32, 14)
        prior[:, 0, :11] = torch.randn(B, 11, generator=g)
        torch.manual_seed(5)
        with torch.no_grad():
            x, _ = agent.sample(prior.to(DEV), solver="ddpm", n_samples=B, sample_steps=T, temperature=0.5)
        plan = next(iter(agent._engine_plans.values()))
        assert plan.n_branches == int(branches)
        outs[(branches, graph)] = x.cpu()
    ref = outs[("1", "1")]
    assert torch.isfinite(ref).all()
    for k, v in outs.items():
        assert torch.equal(v, ref), k


# ------------------------------------------------------------------------------------------------------------------
# TF32 tensor-core programs (CDS_MATH=tf32, the library default and what bench.py measures): fp32 activations and weights in
# memory, wgmma .tf32 (operands read with a 10-bit mantissa), fp32 accumulation and fp32 GN/Mish epilogue -- the
# arithmetic of the reference's own GPU path (cuDNN TF32 convs).  Stated tolerance vs the fp32 reference: max-abs 2e-2,
# mean-abs 2e-3 (per forward and after a full sampler; emulated figures: ~4e-3 / ~9e-4 per forward).
TF32_MAX, TF32_MEAN = 2e-2, 2e-3


@pytest.mark.parametrize("name", list(cases.NETS))
def test_denoiser_forward_tf32_tensor_cores(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "tf32")
    case = cases.NETS[name]
    net, _ = product_net(case)
    net = net.to(DEV)
    x, t, cond = cases.net_inputs(case)
    cond_emb = None if cond is None else cond.to(DEV)
    want = golden["nets"][name + "/y"]
    for i in range(cases.NET_BATCH):
        y = runtime.engine_forward(net, x.to(DEV), t[i:i + 1], cond_emb)
        err = np.abs(y[i].cpu().numpy() - want[i])
        assert err.max() < TF32_MAX and err.mean() < TF32_MEAN, (name, i, float(err.max()), float(err.mean()))


@pytest.mark.parametrize("name", ["disc_dup_ddpm_x0", "disc_dup_ddim_eps", "cont_ddim_eps", "cont_sde_dpmsolverpp_2M_x0",
                                  "cont_cfg2branch_2M", "disc_warm_ddim"])
def test_sampler_tf32_tensor_cores_goldens(golden, name, monkeypatch):
    """Reverse loop on the TF32 programs (once-cast + update-fused fp32 x_t copy + programmatic dependent launch) against the
    reference goldens; graph replay and direct launches must give the same bits."""
    monkeypatch.setenv("CDS_MATH", "tf32")
    spec = cases.sampler_cases()[name]
    outs = []
    for graph in ("1", "0"):
        monkeypatch.setenv("CDS_GRAPH", graph)
        agent, inp, kw = build_agent(spec, device=DEV)
        for k in ("condition_cfg", "warm_start_reference"):
            if kw.get(k) is not None:
                kw[k] = kw[k].to(DEV)
        tape = NoiseTape(tape_of(golden["samplers"], name))
        with tape.active(), torch.no_grad():
            x0, _ = agent.sample(inp["prior"].to(DEV), **kw)
        outs.append(x0.cpu())
        err = np.abs(x0.cpu().numpy() - golden["samplers"][name + "/x0"])
        # two-branch CFG (w_cfg = 2.5) multiplies the rounding of the two predictions by |w| + |1 - w| = 4, and that toy case
        # clips most outputs to x_max: an element crossing the clip boundary at a different iteration is an isolated outlier
        # (toy 8-channel nets with clipping: an isolated element may sit on the other side of a clip decision)
        mx, mean = (0.15, 4 * TF32_MEAN) if "cfg2branch" in name else (3 * TF32_MAX, TF32_MEAN)
        assert err.max() < mx and err.mean() < mean, (name, graph, float(err.max()), float(err.mean()))
    assert torch.equal(outs[0], outs[1])         # graph replay == direct launches


def test_tf32_is_the_default_math_mode(monkeypatch):
    monkeypatch.delenv("CDS_MATH", raising=False)
    assert runtime._math_mode() == cabi.MATH_TF32_TC
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    net, _ = product_net(cases.NETS["janner_cfg2"])
    p = Program(torch.device(DEV), 256, 1, runtime._math_mode())
    lower_denoiser(p, net.to(DEV), View(p.buf(256, 32, 14), 32, 14), (32, 14), False, 0)
    convs = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV]
    assert len(convs) == 40 and all(c.math == cabi.MATH_TF32_TC and c.in_dtype == cabi.TF32 for c in convs)


def test_chiunet_full_size_on_tensor_cores(monkeypatch):
    """cfg3's backbone exactly as the DP pipelines build it (model_dim 256 -> 256/512/1024 channels, 68.9 M parameters): every conv,
    the C_out = 512 / 1024 ones included (2 / 4 CTAs of 256 columns, two-pass GroupNorm), runs on wgmma; checked against the
    module's own fp32 forward on the GPU (TF32 off), bf16 tolerance."""
    monkeypatch.setenv("CDS_MATH", "bf16")
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    from cleandiffuser_b200.nn_diffusion import ChiUNet1d
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    net = load_synth(ChiUNet1d(7, 20, 2, model_dim=256, emb_dim=256, kernel_size=5, dim_mult=[1, 2, 2]), seed=3).eval().to(DEV)
    g = torch.Generator().manual_seed(4)
    B = 160                                                         # 2.5 / 5 / 20 row tiles at L = 4 / 8 / 16 (ragged last tile)
    x, cond = torch.randn(B, 16, 7, generator=g).to(DEV), torch.randn(B, 40, generator=g).to(DEV)
    t = torch.tensor([17], device=DEV)
    with torch.no_grad():
        want = net(x, t.expand(B), cond)
    y = runtime.engine_forward(net, x, t, cond)
    err = (y - want).abs()
    assert torch.isfinite(y).all()
    assert err.max().item() < 0.25 and err.mean().item() < 0.02, (err.max().item(), err.mean().item())
    p = Program(torch.device(DEV), B, 1, cabi.MATH_BF16_TC)
    lower_denoiser(p, net, View(p.buf(B, 16, 7), 16, 7), (16, 7), True, 0)
    convs = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV and op.u.conv.taps > 1]
    assert len(convs) >= 28 and all(c.math == cabi.MATH_BF16_TC for c in convs), [(c.C_in, c.C_out, c.math) for c in convs]


def test_dit_full_size_on_tensor_cores(monkeypatch):
    """cfg4's backbone as the DD pipeline builds it (d_model 320, 10 heads of 32, depth 2, L = 100 tokens -- not a multiple of
    the 16-row MMA tile: padded keys are masked, padded queries dropped): Linear layers on wgmma over the flattened token
    stream, attention on mma.sync, checked against the module's own fp32 forward on the GPU."""
    monkeypatch.setenv("CDS_MATH", "bf16")
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    from cleandiffuser_b200.nn_diffusion import DiT1d
    torch.backends.cuda.matmul.allow_tf32 = False
    net = load_synth(DiT1d(29, emb_dim=128, d_model=320, n_heads=10, depth=2, timestep_emb_type="fourier"), seed=0).eval().to(DEV)
    g = torch.Generator().manual_seed(2)
    B, L = 37, 100                                                  # 3700 token rows: ragged last 128-row tile
    x, cond = torch.randn(B, L, 29, generator=g).to(DEV), torch.randn(B, 128, generator=g).to(DEV)
    t = torch.tensor([0.37], device=DEV)
    with torch.no_grad():
        want = net(x, t.expand(B), cond)
    y = runtime.engine_forward(net, x, t, cond)
    err = (y - want).abs()
    assert torch.isfinite(y).all()
    assert err.max().item() < 0.15 and err.mean().item() < 0.02, (err.max().item(), err.mean().item())
    p = Program(torch.device(DEV), B, 1, cabi.MATH_BF16_TC)
    lower_denoiser(p, net, View(p.buf(B, L, 29), L, 29), (L, 29), True, 0)
    assert sum(1 for op in p.ops if op.kind == cabi.OP_CONV and op.u.conv.math == cabi.MATH_BF16_TC) == 10
    assert all(op.u.attn.qkv_dtype == cabi.BF16 for op in p.ops if op.kind == cabi.OP_ATTN)


@pytest.mark.parametrize("d_model,heads", [(320, 10), (256, 8)])
def test_dit_fused_linear_layernorm_matches_the_two_launch_form(d_model, heads, monkeypatch):
    """TF32 programs fuse `gated Linear -> LayerNorm + modulate` pairs into one launch at plan-finalize time (csrc/linear_ln.cuh);
    CDS_FUSE_LN=0 keeps the two launches.  Same arithmetic up to summation order: the two forms must agree far inside the TF32
    tolerance, and both must match the module's fp32 forward.  37 x 100 = 3700 token rows: ragged last 128-row tile."""
    monkeypatch.setenv("CDS_MATH", "tf32")
    from cleandiffuser_b200.nn_diffusion import DiT1d
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(3)
    B, L = 37, 100
    x, cond = torch.randn(B, L, 29, generator=g).to(DEV), torch.randn(B, 128, generator=g).to(DEV)
    t = torch.tensor([0.37], device=DEV)
    outs, launches = {}, {}
    for fuse in ("1", "0"):
        monkeypatch.setenv("CDS_FUSE_LN", fuse)
        net = load_synth(DiT1d(29, emb_dim=128, d_model=d_model, n_heads=heads, depth=2, timestep_emb_type="fourier"), seed=0).eval().to(DEV)
        with torch.no_grad():
            want = net(x, t.expand(B), cond)
        outs[fuse] = runtime.engine_forward(net, x, t, cond)
        err = (outs[fuse] - want).abs()
        assert torch.isfinite(outs[fuse]).all()
        assert err.max().item() < TF32_MAX and err.mean().item() < TF32_MEAN, (fuse, err.max().item(), err.mean().item())
    d = (outs["1"] - outs["0"]).abs()
    assert d.max().item() < 2e-3, d.max().item()


def test_run_range_splits_a_fused_linear_layernorm_pair(monkeypatch):
    """`cds_plan_run_range` with a boundary BETWEEN a gated Linear and the LayerNorm fused into its launch must run the two
    operators separately (the classifier-guidance interleave may cut a program anywhere); every split point gives the whole
    program's result up to the summation order of the LayerNorm statistics."""
    monkeypatch.setenv("CDS_MATH", "tf32")
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    from cleandiffuser_b200.nn_diffusion import DiT1d
    net = load_synth(DiT1d(9, emb_dim=32, d_model=256, n_heads=8, depth=1, timestep_emb_type="fourier"), seed=1).eval().to(DEV)
    B, L = 5, 64
    g = torch.Generator().manual_seed(4)
    x, cond = torch.randn(B, L, 9, generator=g).to(DEV), torch.randn(B, 32, generator=g).to(DEV)
    p = Program(torch.device(DEV), B, 1, cabi.MATH_TF32_TC)
    xin = p.buf(B, L, 9)
    xin.copy_(x)
    pred = lower_denoiser(p, net, View(xin, L, 9), (L, 9), True, 0)
    handle = runtime._make_handle(torch.device(DEV), p.ops, 1)
    with torch.no_grad():
        ctx = runtime._Ctx(torch.tensor([0.4], device=DEV), cond)
        for fn in p.per_call:
            fn(ctx)
    st = torch.cuda.current_stream().cuda_stream
    n = len(p.ops)
    pairs = [i for i in range(n - 1) if p.ops[i].kind == cabi.OP_CONV and p.ops[i + 1].kind == cabi.OP_LNMOD
             and p.ops[i].u.conv.scale.sample and p.ops[i].u.conv.math == cabi.MATH_TF32_TC]
    assert len(pairs) == 2, pairs                                # out-projection + fc2 of the one block
    assert handle.launches_per_iter() == n + 1 - len(pairs) - sum(1 for op in p.ops if op.flags & 1)   # fused pairs count once
    handle.run(0, 1, st, False)
    torch.cuda.synchronize()
    whole = pred.t.clone()
    for i in pairs:
        pred.t.fill_(float("nan"))
        handle.run_range(0, 0, i + 1, st)                        # ... up to and including the Linear
        handle.run_range(0, i + 1, n - (i + 1), st)              # the LayerNorm onwards
        torch.cuda.synchronize()
        d = (pred.t - whole).abs().max().item()
        assert d < 2e-3, (i, d)
    handle.close()
