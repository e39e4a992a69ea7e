"""Execute the lowered operator programs with the numpy interpreter (tests/emulator.py) on CPU tensors and
compare with the reference goldens: pins ``engine/lower.py`` + ``engine/runtime.py`` (strides, table columns,
phase packing, CFG row doubling, noise slots, coefficient rows) without needing a GPU."""
import numpy as np
import pytest
import torch

import cases
import emulator
from common import product_net, tape_of
from test_host_golden import build_agent
from cleandiffuser_b200.diffusion import ContinuousConsistencyModel
from cleandiffuser_b200.engine import runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.testing import NoiseTape



@pytest.fixture(autouse=True)
def _emulate(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")       # any fallback to the PyTorch loop is a failure here
    monkeypatch.setenv("CDS_MATH", "fp32")


@pytest.mark.parametrize("name", list(cases.NETS))
def test_lowered_denoiser(golden, name):
    case = cases.NETS[name]
    net, _ = product_net(case)
    x, t, cond = cases.net_inputs(case)
    want = golden["nets"][name + "/y"]
    for i in range(cases.NET_BATCH):
        y = runtime.engine_forward(net, x, t[i:i + 1], cond)
        np.testing.assert_allclose(y[i].numpy(), want[i], rtol=0, atol=2e-5, err_msg=f"{name} row {i}")


@pytest.mark.parametrize("name", list(cases.sampler_cases()))
def test_lowered_sampler(golden, name):
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    before = runtime.STATS["engine_calls"]
    tape = NoiseTape(tape_of(golden["samplers"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    assert runtime.STATS["engine_calls"] == before + 1
    assert tape.pos == len(tape.draws)
    np.testing.assert_allclose(x0.numpy(), golden["samplers"][name + "/x0"], rtol=1e-4, atol=3e-4)


@pytest.mark.parametrize("steps", [1, 3])
def test_lowered_consistency(golden, steps):
    g = golden["consistency"]
    net, _ = product_net(cases.NETS["chi_cm_fourier"])
    cm = ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), x_max=torch.ones(1, 8, 3),
                                    x_min=-torch.ones(1, 8, 3), device="cpu")
    tape = NoiseTape(tape_of(g, f"cm{steps}"))
    before = runtime.STATS["engine_calls"]
    with tape.active(), torch.no_grad():
        x0, _ = cm.sample(torch.zeros(4, 8, 3), n_samples=4, sample_steps=steps,
                          condition_cfg=torch.as_tensor(g[f"cm{steps}/cond"]), w_cfg=1.0)
    assert runtime.STATS["engine_calls"] == before + 1
    np.testing.assert_allclose(x0.numpy(), g[f"cm{steps}/x0"], rtol=1e-4, atol=3e-4)


# ---------------------------------------------------------------------------------------------------------------
# bf16 tensor-core programs: same lowering, bf16 activations/weights in the interpreter.  Tolerances are the
# SURVEY 8(c) bf16 figures (single forward ~8e-3 relative); this pins the bf16 *lowering* (dtypes, [tap][Cout][Cin]
# weight packing, which ops go to which kernel family), the kernels themselves are checked on the GPU.
BF16_NETS = ["janner_cfg2", "janner_kitchen_cond", "chi_small", "chi_cm_fourier", "dit_small", "dit_pos_uncond"]


@pytest.mark.parametrize("name", BF16_NETS)
def test_lowered_denoiser_bf16(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "bf16")
    case = cases.NETS[name]
    net, _ = product_net(case)
    x, t, cond = cases.net_inputs(case)
    want = golden["nets"][name + "/y"]
    for i in range(cases.NET_BATCH):
        y = runtime.engine_forward(net, x, t[i:i + 1], cond)
        err = np.abs(y[i].numpy() - want[i])
        assert err.max() < 0.08 and err.mean() < 0.015, (name, i, err.max(), err.mean())


@pytest.mark.parametrize("name", list(cases.NETS))
def test_lowered_denoiser_tf32(golden, name, monkeypatch):
    """TF32 programs (the default math mode): fp32 activations, fp32 [tap][Cout][Cin] weights rounded to TF32, operands
    truncated to a 10-bit mantissa by the interpreter as wgmma .tf32 does."""
    monkeypatch.setenv("CDS_MATH", "tf32")
    case = cases.NETS[name]
    net, _ = product_net(case)
    x, t, cond = cases.net_inputs(case)
    want = golden["nets"][name + "/y"]
    for i in range(cases.NET_BATCH):
        y = runtime.engine_forward(net, x, t[i:i + 1], cond)
        err = np.abs(y[i].numpy() - want[i])
        assert err.max() < 2e-2 and err.mean() < 2e-3, (name, i, err.max(), err.mean())


def test_tf32_program_uses_tensor_core_ops(monkeypatch):
    monkeypatch.delenv("CDS_MATH", raising=False)            # tf32 is the default
    from cleandiffuser_b200.engine import cabi
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    assert runtime._math_mode() == cabi.MATH_TF32_TC
    net, _ = product_net(cases.NETS["janner_cfg2"])
    p = Program(torch.device("cpu"), 8, 1, cabi.MATH_TF32_TC)
    xin = p.buf(8, 32, 14)
    lower_denoiser(p, net, View(xin, 32, 14), (32, 14), False, 0)
    convs = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV]
    # x_t is handed over as a 16-channel fp32 copy (64-byte rows), every conv of the UNet is a TF32 tensor-core operator; what
    # feeds a TF32 MMA is written TF32-rounded (cds_dtype CDS_TF32), the prediction itself stays exact fp32
    assert p.ops[0].kind == cabi.OP_CAST and p.ops[0].u.cast.C_out == 16 and p.ops[0].u.cast.out_dtype == cabi.TF32
    assert len(convs) == 40 and all(c.math == cabi.MATH_TF32_TC and c.in_dtype == cabi.TF32 for c in convs)
    assert all(c.out_dtype == cabi.TF32 for c in convs[:-1]) and convs[-1].out_dtype == cabi.F32


@pytest.mark.parametrize("name", ["disc_dup_ddpm_x0", "cont_ddim_eps", "cont_cfg2branch_2M"])
def test_lowered_sampler_tf32(golden, name, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "tf32")
    from cleandiffuser_b200.engine import cabi
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    tape = NoiseTape(tape_of(golden["samplers"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    plan = next(iter(agent._engine_plans.values()))
    ops = plan.program.ops
    casts = [op for op in ops if op.kind == cabi.OP_CAST]
    assert len(casts) == 1 and casts[0].flags & cabi.OPF_ONCE
    upd = ops[-1].u.update
    assert ops[-1].kind == cabi.OP_UPDATE and upd.x_cast == casts[0].u.cast.out and upd.cast_C_out == 16
    assert upd.x_cast_dtype == cabi.TF32
    err = np.abs(x0.numpy() - golden["samplers"][name + "/x0"])
    # two-branch CFG (w_cfg = 2.5) multiplies the rounding of the two predictions by |w| + |1 - w| = 4, and this toy case clips
    # most of its outputs to x_max: an element that crosses the clip boundary at a different iteration is an isolated outlier
    mx, mean = (0.15, 8e-3) if "cfg2branch" in name else (2e-2, 2e-3)
    assert err.max() < mx and err.mean() < mean, (float(err.max()), float(err.mean()))


def test_bf16_program_uses_tensor_core_ops(monkeypatch):
    monkeypatch.setenv("CDS_MATH", "bf16")
    from cleandiffuser_b200.engine import cabi
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    net, _ = product_net(cases.NETS["janner_cfg2"])
    p = Program(torch.device("cpu"), 8, 1, cabi.MATH_BF16_TC)
    xin = p.buf(8, 32, 14)
    lower_denoiser(p, net, View(xin, 32, 14), (32, 14), False, 0)
    kinds = [op.u.conv.math for op in p.ops if op.kind == cabi.OP_CONV]
    # x_t is handed over as a 32-channel bf16 copy (CDS_OP_CAST), so EVERY conv of the UNet -- stride-2 down-sampling,
    # two-phase transposed up-sampling and the 14-channel 1x1 head included -- runs on wgmma
    assert p.ops[0].kind == cabi.OP_CAST
    assert kinds.count(cabi.MATH_BF16_TC) == len(kinds) == 40, kinds


@pytest.mark.parametrize("name", ["disc_dup_ddpm_x0", "cont_ddim_eps", "cont_cfg2branch_2M"])
def test_lowered_sampler_bf16(golden, name, monkeypatch):
    """bf16 programs inside the reverse loop: the x_t hand-over cast runs ONCE per call (CDS_OPF_ONCE) and every solver
    update refreshes the channel-padded bf16 copy itself (cds_update_op.x_cast)."""
    monkeypatch.setenv("CDS_MATH", "bf16")
    from cleandiffuser_b200.engine import cabi
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    tape = NoiseTape(tape_of(golden["samplers"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    plan = next(iter(agent._engine_plans.values()))
    ops = plan.program.ops
    casts = [op for op in ops if op.kind == cabi.OP_CAST]
    assert len(casts) == 1 and casts[0].flags & cabi.OPF_ONCE
    upd = ops[-1].u.update
    assert ops[-1].kind == cabi.OP_UPDATE and upd.x_cast == casts[0].u.cast.out and upd.cast_C_out == 32
    err = np.abs(x0.numpy() - golden["samplers"][name + "/x0"])
    # two-branch CFG multiplies the bf16 noise of the two predictions by |w| + |1 - w| (w_cfg = 2.5 in this case): a few
    # outliers, same mean
    max_tol = 1.5 if "cfg2branch" in name else 0.2
    assert err.max() < max_tol and err.mean() < 0.02, (float(err.max()), float(err.mean()))


def test_table_caches_follow_the_request(golden):
    """Coefficient / time-conditioning tables are cached per (solver, schedule) and per (weights, timesteps): repeated and
    interleaved requests on ONE agent must still give each request's own result."""
    name = "disc_dup_ddpm_x0"
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    want = golden["samplers"][name + "/x0"]

    def run(**over):
        tape = NoiseTape(tape_of(golden["samplers"], name))
        with tape.active(), torch.no_grad():
            return agent.sample(inp["prior"], **{**kw, **over})[0].numpy()

    a0 = run()
    np.testing.assert_allclose(a0, want, rtol=1e-4, atol=3e-4)
    b = run(solver="ddim")                               # other solver, same plan shapes -> other table
    assert np.abs(b - a0).max() > 1e-3
    np.testing.assert_array_equal(run(), a0)             # cached table + cached time rows
    with torch.no_grad():                                # weights change -> time rows must be rebuilt
        for p in agent.model_ema["diffusion"].parameters():
            p.mul_(1.01)
    assert np.abs(run() - a0).max() > 1e-4


def test_schedule_identity_fast_path_is_keyed_on_what_the_schedule_depends_on(golden):
    """The samplers hand the engine a ``sched_id``: the discrete SDE sampler its named step schedule, grid length and the identity +
    version of the alpha / sigma buffers; the consistency and EDM samplers their step count and sigma grid parameters.  A repeated
    request must not read the schedule back from the device (on a GPU each read is a stream synchronisation), a changed schedule
    must miss.  All of them share the agent's one table cache."""
    from test_edm import build_edm

    def ids(agent):                                        # the cache entries keyed on a schedule identity
        return [k for k in agent._engine_tables if k[0] == "id"]

    def hit(agent, run, steps):
        reads = []
        real_cpu = torch.Tensor.cpu
        try:
            torch.Tensor.cpu = lambda self, *a, **k: (reads.append(tuple(self.shape)), real_cpu(self, *a, **k))[1]
            out = run()
        finally:
            torch.Tensor.cpu = real_cpu
        assert not [r for r in reads if r == (steps,) or r == (steps + 1,)], reads     # no schedule read-back
        assert len(ids(agent)) == 1
        return out

    name = "disc_dup_ddpm_x0"
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)

    def run(**over):
        tape = NoiseTape(tape_of(golden["samplers"], name))
        with tape.active(), torch.no_grad():
            return agent.sample(inp["prior"], **{**kw, **over})[0].numpy()

    a0 = run()
    assert len(ids(agent)) == 1
    np.testing.assert_array_equal(hit(agent, run, kw["sample_steps"]), a0)
    with torch.no_grad():
        agent.alpha.mul_(0.999)                            # the schedule changes in place -> version bump -> new identity
    a2 = run()
    assert len(ids(agent)) == 2 and np.abs(a2 - a0).max() > 1e-6
    run(sample_step_schedule=lambda T, S: torch.arange(S + 1) * (T - 1) // S)       # callables carry no identity: no entry
    assert len(ids(agent)) == 2

    g = golden["consistency"]
    net, _ = product_net(cases.NETS["chi_cm_fourier"])
    cm = ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), x_max=torch.ones(1, 8, 3),
                                    x_min=-torch.ones(1, 8, 3), device="cpu")

    def run_cm():
        with NoiseTape(tape_of(g, "cm3")).active(), torch.no_grad():
            return cm.sample(torch.zeros(4, 8, 3), n_samples=4, sample_steps=3, condition_cfg=torch.as_tensor(g["cm3/cond"]),
                             w_cfg=1.0)[0].numpy()

    c0 = run_cm()
    assert len(ids(cm)) == 1
    np.testing.assert_array_equal(hit(cm, run_cm, 3), c0)
    cm.sigma_min *= 2                                      # another sigma grid -> another identity
    c2 = run_cm()
    assert len(ids(cm)) == 2 and np.abs(c2 - c0).max() > 1e-6

    name = "edm_heun_mask_clip_dx"
    edm, inp, kw, _ = build_edm(cases.edm_cases()[name])

    def run_edm():
        with NoiseTape(tape_of(golden["edm"], name)).active(), torch.no_grad():
            return edm.sample(inp["prior"], **kw)[0].numpy()

    e0 = run_edm()
    assert len(ids(edm)) == 1
    np.testing.assert_array_equal(hit(edm, run_edm, kw["sample_steps"]), e0)
    edm.sigma_max *= 0.5
    e2 = run_edm()
    assert len(ids(edm)) == 2 and np.abs(e2 - e0).max() > 1e-6


@pytest.mark.parametrize("name,math", [("disc_dup_ddpm_x0", "fp32"), ("cont_cfg2branch_2M", "fp32"), ("cont_ddim_eps", "bf16")])
def test_lowered_sampler_two_branches(golden, name, math, monkeypatch):
    """The batch split into two independent operator chains (cds_op.flags branch bits; parallel streams on the GPU): same
    results, every branch reads/writes its own slice of x_t / noise / prior / condition."""
    monkeypatch.setenv("CDS_MATH", math)
    monkeypatch.setenv("CDS_BRANCHES", "2")
    monkeypatch.setenv("CDS_BRANCH_MIN_BATCH", "1")
    from cleandiffuser_b200.engine import cabi
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    tape = NoiseTape(tape_of(golden["samplers"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    plan = next(iter(agent._engine_plans.values()))
    assert plan.n_branches == 2
    branches = sorted({(op.flags >> cabi.OPF_BRANCH_SHIFT) & 0xff for op in plan.program.ops})
    assert branches == [0, 1]
    upd = [op.u.update for op in plan.program.ops if op.kind == cabi.OP_UPDATE]
    assert len(upd) == 2 and upd[1].x == upd[0].x + 4 * upd[0].batch * upd[0].row
    want = golden["samplers"][name + "/x0"]
    if math == "fp32":
        np.testing.assert_allclose(x0.numpy(), want, rtol=1e-4, atol=3e-4)
    else:
        err = np.abs(x0.numpy() - want)
        assert err.max() < 0.2 and err.mean() < 0.02, (float(err.max()), float(err.mean()))


def test_wide_chiunet_layers_lower_to_tensor_core_ops(monkeypatch):
    """ChiUNet1d with C_out = 512 and 1024 layers (cumulative dim_mult, as at the pipelines' model_dim 256): the wide layers are
    tensor-core operators too (2-4 CTAs of 256 columns per row tile), and the lowered bf16 program agrees with the module."""
    monkeypatch.setenv("CDS_MATH", "bf16")
    from cleandiffuser_b200.engine import cabi
    from cleandiffuser_b200.nn_diffusion import ChiUNet1d
    from cleandiffuser_b200.testing import load_synth
    net = load_synth(ChiUNet1d(7, 20, 2, model_dim=128, emb_dim=64, kernel_size=5, dim_mult=[1, 2, 2]), seed=3).eval()
    g = torch.Generator().manual_seed(4)
    x, cond = torch.randn(2, 16, 7, generator=g), torch.randn(2, 40, generator=g)
    t = torch.tensor([17])
    with torch.no_grad():
        want = net(x, t.expand(2), cond).numpy()
    y = runtime.engine_forward(net, x, t, cond).numpy()
    err = np.abs(y - want)
    assert err.max() < 0.1 and err.mean() < 0.02, (float(err.max()), float(err.mean()))
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    p = Program(torch.device("cpu"), 2, 1, cabi.MATH_BF16_TC)
    lower_denoiser(p, net, View(p.buf(2, 16, 7), 16, 7), (16, 7), True, 0)
    wide = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV and op.u.conv.C_out == 512]
    assert len(wide) >= 6 and all(c.math == cabi.MATH_BF16_TC for c in wide)


def test_dit_tf32_program_keeps_attention_on_tensor_cores(monkeypatch):
    """TF32 programs: DiT1d's Linear layers are TF32 tensor-core operators over fp32 tokens; q/k/v are written TF32-rounded
    (cds_dtype CDS_TF32), which selects the mma.sync tf32 attention kernel (head_dim 32, L <= 128) instead of the fp32 one."""
    monkeypatch.setenv("CDS_MATH", "tf32")
    from cleandiffuser_b200.engine import cabi
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    from cleandiffuser_b200.nn_diffusion import DiT1d
    from cleandiffuser_b200.testing import load_synth
    net = load_synth(DiT1d(29, emb_dim=128, d_model=320, n_heads=10, depth=2, timestep_emb_type="fourier"), seed=0).eval()
    B, L = 3, 100
    p = Program(torch.device("cpu"), B, 1, cabi.MATH_TF32_TC)
    lower_denoiser(p, net, View(p.buf(B, L, 29), L, 29), (L, 29), True, 0)
    tc = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV and op.u.conv.math == cabi.MATH_TF32_TC]
    tokens = [c for c in tc if c.batch == B * L]                  # Linear layers over the flattened token stream
    assert sorted((c.C_in, c.C_out) for c in tokens) == sorted([(320, 960), (320, 320), (320, 1280), (1280, 320)] * 2 + [(32, 320), (320, 29)])
    # fp32 operands qualify for the TF32 kernels as they are: the per-trajectory conditioning GEMMs (map_emb 320 -> 320 and the
    # adaLN 320 -> 4480 Linear) run on wgmma too
    assert sorted((c.C_in, c.C_out) for c in tc if c.batch == B) == [(320, 320), (320, 4480)]
    attn = [op.u.attn for op in p.ops if op.kind == cabi.OP_ATTN]
    assert len(attn) == 2 and all(a.qkv_dtype == cabi.TF32 and a.out_dtype == cabi.TF32 for a in attn)
    # the form conv_tc's gated epilogue lane serves: a gated Linear with a dense fp32 residual, directly followed by the
    # LayerNorm+modulate that reads its output, one vector set per L tokens
    gated = 0
    for a, b in zip(p.ops[:-1], p.ops[1:]):
        if a.kind != cabi.OP_CONV or b.kind != cabi.OP_LNMOD:
            continue
        c, ln = a.u.conv, b.u.lnmod
        if (c.math == cabi.MATH_TF32_TC and c.scale.sample and not c.scale.step and c.res and not c.res_w and c.res_batch_mod == 0
                and c.taps == 1 and c.L_in == 1 and c.C_out == 320 and c.C_in % 32 == 0 and c.sample_row_div == L
                and c.out_dtype != cabi.BF16 and c.res_dtype != cabi.BF16 and c.bias.step and not c.bias.sample
                and ln.in_ == c.out and ln.C == c.C_out and ln.batch * ln.L == c.batch and ln.L == L and ln.out_dtype != cabi.BF16):
            gated += 1
    assert gated == 4                                    # attention out-projection and second MLP Linear of both blocks
    g = torch.Generator().manual_seed(2)
    x, cond, t = torch.randn(B, L, 29, generator=g), torch.randn(B, 128, generator=g), torch.tensor([0.37])
    with torch.no_grad():
        want = net(x, t.expand(B), cond).numpy()
    err = np.abs(runtime.engine_forward(net, x, t, cond).numpy() - want)
    assert err.max() < 2e-2 and err.mean() < 2e-3, (float(err.max()), float(err.mean()))


def test_dit_linear_layers_lower_to_flattened_tensor_core_ops(monkeypatch):
    """DiT1d on a tensor-core program: QKV / out-proj / MLP Linear layers become tensor-core operators over the token stream
    flattened to rows*L length-1 sequences (L = 100 is not a tile-friendly length), per-trajectory gates follow through
    sample_row_div, LayerNorm+modulate and attention hand bf16 to the Linear that follows."""
    monkeypatch.setenv("CDS_MATH", "bf16")
    from cleandiffuser_b200.engine import cabi
    from cleandiffuser_b200.engine.lower import Program, View, lower_denoiser
    from cleandiffuser_b200.nn_diffusion import DiT1d
    from cleandiffuser_b200.testing import load_synth
    net = load_synth(DiT1d(29, emb_dim=128, d_model=320, n_heads=10, depth=2, timestep_emb_type="fourier"), seed=0).eval()
    B, L = 3, 100
    p = Program(torch.device("cpu"), B, 1, cabi.MATH_BF16_TC)
    lower_denoiser(p, net, View(p.buf(B, L, 29), L, 29), (L, 29), True, 0)
    tc = [op.u.conv for op in p.ops if op.kind == cabi.OP_CONV and op.u.conv.math == cabi.MATH_BF16_TC]
    # per block QKV / out-proj / fc1 / fc2, plus the input projection (x_t padded 29 -> 32 channels) and the 29-wide output head
    assert sorted((c.C_in, c.C_out) for c in tc) == sorted([(320, 960), (320, 320), (320, 1280), (1280, 320)] * 2 + [(32, 320), (320, 29)])
    assert all(c.batch == B * L and c.L_in == 1 and c.sample_row_div == L for c in tc)
    assert [op.kind for op in p.ops].count(cabi.OP_CAST) == 1
    assert all(op.u.lnmod.out_dtype == cabi.BF16 for op in p.ops if op.kind == cabi.OP_LNMOD)
    assert all(op.u.attn.out_dtype == cabi.BF16 for op in p.ops if op.kind == cabi.OP_ATTN)
    g = torch.Generator().manual_seed(2)
    x, cond, t = torch.randn(B, L, 29, generator=g), torch.randn(B, 128, generator=g), torch.tensor([0.37])
    with torch.no_grad():
        want = net(x, t.expand(B), cond).numpy()
    err = np.abs(runtime.engine_forward(net, x, t, cond).numpy() - want)
    assert err.max() < 0.12 and err.mean() < 0.02, (float(err.max()), float(err.mean()))


# ---------------------------------------------------------------------------------------------------------------
# host runtime: noise-tape chunking, weight-version tracking through EMA updates, plan cache eviction
@pytest.mark.parametrize("name", ["disc_dup_ddpm_x0", "disc_dx_sde_dpmsolverpp_2M_eps", "cont_sde_dpmsolver_1_eps"])
def test_noise_tape_chunks_give_the_same_result(golden, name, monkeypatch):
    """A tape shorter than the loop's number of draws (CDS_NOISE_TAPE_MB) is refilled chunk by chunk: memory O(budget), same
    draws in the same order, same result as the all-up-front tape."""
    spec = cases.sampler_cases()[name]
    monkeypatch.setenv("CDS_NOISE_TAPE_MB", "0.0001")           # ~100 bytes: ONE slot of these toy shapes
    agent, inp, kw = build_agent(spec)
    tape = NoiseTape(tape_of(golden["samplers"], name))
    with tape.active(), torch.no_grad():
        x0, _ = agent.sample(inp["prior"], **kw)
    assert tape.pos == len(tape.draws)
    plan = next(iter(agent._engine_plans.values()))
    n_draws = len(tape.draws) - 1                                # the first draw is the initial x_T, not a loop draw
    assert plan.noise is not None and plan.noise.shape[0] < n_draws, (plan.noise.shape, n_draws)
    np.testing.assert_allclose(x0.numpy(), golden["samplers"][name + "/x0"], rtol=1e-4, atol=3e-4)


def test_ema_update_invalidates_packed_weights(golden):
    """sample(use_ema=True) -> update() -> sample(use_ema=True): the EMA twin changed through ema_update(), the plan must
    re-pack (ADVICE r1: writes through .data do not bump tensor versions; the agent's weight epoch does)."""
    name = "disc_dup_ddpm_x0"
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    agent.ema_rate = 0.5

    def run(backend, monkey_env):
        tape = NoiseTape(tape_of(golden["samplers"], name))
        with tape.active(), torch.no_grad():
            return agent.sample(inp["prior"], **kw)[0].numpy()

    a0 = run("cuda", None)
    x0 = torch.randn(8, *inp["prior"].shape[1:])
    agent.update(x0)                                             # optimiser step + ema_update()
    agent.model_ema.eval()
    a1 = run("cuda", None)
    assert np.abs(a1 - a0).max() > 1e-5
    import os
    os.environ["CDS_BACKEND"] = "torch"
    try:
        t1 = run("torch", None)
    finally:
        os.environ["CDS_BACKEND"] = "cuda"
    np.testing.assert_allclose(a1, t1, rtol=1e-4, atol=3e-4)


def test_plan_cache_is_bounded(golden, monkeypatch):
    monkeypatch.setenv("CDS_MAX_PLANS", "2")
    name = "disc_dup_ddpm_x0"
    spec = cases.sampler_cases()[name]
    agent, inp, kw = build_agent(spec)
    for n in (2, 3, 4, 5):
        with torch.no_grad():
            agent.sample(inp["prior"][:n], **{**kw, "n_samples": n})
        assert len(agent._engine_plans) <= 2
    keys = list(agent._engine_plans)
    with torch.no_grad():
        agent.sample(inp["prior"][:4], **{**kw, "n_samples": 4})      # cached plan: moves to the most-recently-used end
    assert list(agent._engine_plans)[-1] == keys[0] and len(agent._engine_plans) == 2
