"""TEST INFRASTRUCTURE: the MLP denoiser programs of the offline-RL and Diffusion-BC pipelines (IDQL, DQL / EDP, Veteran's
inverse dynamics, SfBC / QGPO, DBC), built by one ``sample()`` on synthetic weights, and the whole-network check of their
lowering against the PyTorch module in float64.

The per-operator audit (tests/program_audit.py) judges each kernel against its own descriptor; it cannot see a lowering
or weight-packing mistake (a wrong column offset into a table, a missing 1/1.414 in PearceMlp's packed weights, a wrong
concatenation offset).  ``denoiser_check`` runs the operators of one iteration up to the final Linear and compares that
Linear's output -- the denoiser's prediction -- with the fp64 module on the same x_t, time and condition.

Shapes follow the reference pipelines' configs (pipelines/*.py of CleanDiffuser); ``small=True`` gives CPU-sized versions
(hidden 64..128, batch <= 16) for the interpreter."""
import copy

import torch

import emulator
import program_audit as pa
from cleandiffuser_b200.diffusion import DDPM, ContinuousDiffusionSDE, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import cabi
from cleandiffuser_b200.nn_condition import IdentityCondition, MLPCondition
from cleandiffuser_b200.nn_diffusion import DQLMlp, DVInvMlp, IDQLMlp, PearceMlp, SfBCUNet
from cleandiffuser_b200.testing import load_synth

OBS, ACT = 17, 6                                   # halfcheetah / walker2d-sized observations and actions
# name -> (rows, sampling steps); rows = the pipeline's batch (IDQL: 50 environments x 256 candidates)
PROGRAMS = {"idql": (12800, 5), "dql": (2500, 5), "veteran50": (50, 10), "veteran4096": (4096, 10), "sfbc": (2500, 5),
            "sfbc-cfg": (2500, 5), "dbc10": (10, 50), "dbc4096": (4096, 50)}
SMALL_ROWS = 16
W_CFG = 1.7                                        # sfbc-cfg: two branches (conditional and unconditional)
DBC_EXTRA = 8                                      # DBC samples with sample_x: 8 noise-free steps at t = 0 after the loop
# normwise relative error of the whole denoiser vs the fp64 module: coarse on purpose -- a lowering mistake moves the output
# by O(1e-2 .. 1), far above the rounding of any math mode
LOWERING_TOL = {"fp32": 1e-5, "tf32": 2.0 ** -8, "bf16": 2.0 ** -5}


def _net(name, small):
    kind = name.rstrip("0123456789").replace("-cfg", "")
    h = 64 if small else None
    if kind == "idql":
        return load_synth(IDQLMlp(OBS, ACT, emb_dim=64, hidden_dim=h or 256, n_blocks=3, dropout=0.1), seed=11).eval()
    if kind == "dql":
        return load_synth(DQLMlp(OBS, ACT, emb_dim=64), seed=12)
    if kind == "veteran":
        return load_synth(DVInvMlp(OBS, ACT, emb_dim=64, hidden_dim=h or 256), seed=13)
    if kind == "sfbc":
        return load_synth(SfBCUNet(ACT, emb_dim=64, hidden_dims=(128, 64, 32) if small else (512, 256, 128)), seed=14)
    assert kind == "dbc", name
    return load_synth(PearceMlp(9, To=2, emb_dim=32 if small else 128, hidden_dim=128 if small else 512), seed=15)


def cond_shape(name, net):
    """shape of one trajectory's condition embedding, as the denoiser reads it"""
    kind = name.rstrip("0123456789").replace("-cfg", "")
    return {"idql": (OBS,), "dql": (OBS,), "veteran": (2 * OBS,), "sfbc": (64,)}.get(kind, (2, getattr(net, "emb_dim", 0)))


def sample(name, device, small=False):
    """the agent after one sample() of program ``name``; returns (agent, plan)"""
    rows, steps = PROGRAMS[name]
    rows = min(rows, SMALL_ROWS) if small else rows
    net = _net(name, small)
    g = torch.Generator().manual_seed(rows)
    ones = torch.ones(net.fcs[3].out_features if name.startswith("dbc") else ACT)
    act = ones.numel()
    if name.startswith("dbc"):
        agent = DDPM(net, IdentityCondition(dropout=0.0), diffusion_steps=steps, x_max=ones, x_min=-ones, device=device)
        cond = torch.randn(rows, *cond_shape(name, net), generator=g)
        agent.model_ema.eval()
        agent.sample_x(torch.zeros(rows, act, device=device), n_samples=rows, sample_steps=steps,
                       extra_sample_steps=DBC_EXTRA, condition_cfg=cond.to(device), w_cfg=1.0, use_ema=True)
    elif name.startswith("sfbc"):
        nc = load_synth(MLPCondition(OBS, 64, [64], torch.nn.SiLU()), seed=16)
        agent = ContinuousDiffusionSDE(net, nc, x_max=ones, x_min=-ones, device=device)
        agent.eval()
        obs = torch.randn(rows, OBS, generator=g)
        agent.sample(torch.zeros(rows, act, device=device), "ddpm", n_samples=rows, sample_steps=steps,
                     condition_cfg=obs.to(device), w_cfg=W_CFG if name == "sfbc-cfg" else 1.0, use_ema=True)
    else:
        clip = dict(x_max=ones, x_min=-ones) if name == "idql" else {}
        agent = DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), diffusion_steps=steps, device=device, **clip)
        agent.eval()
        cond = torch.randn(rows, *cond_shape(name, net), generator=g)
        agent.sample(torch.zeros(rows, act, device=device), "ddpm", n_samples=rows, sample_steps=steps,
                     condition_cfg=cond.to(device), w_cfg=1.0, use_ema=True)
    assert len(agent._engine_plans) == 1
    return agent, next(iter(agent._engine_plans.values()))


class _Widened(torch.nn.Module):
    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, t):
        return self.inner(t).to(torch.float64)


def check_forms(name, math_mode, plan):
    """the descriptor forms these programs are audited for are reached: conv_simt storing TF32 / bf16 (SfBCUNet's first
    block, PearceMlp's act_emb), LNMOD with one modulation row for the whole batch (IDQLMlp), and SfBCUNet's first block
    with both CFG row maps -- x_t read at b % in_batch_mod by its first operator, at b % res_batch_mod by its shortcut (two
    operators of one block, both on conv_simt: x_t has 6 channels)"""
    ops = plan.program.ops
    convs = [op.u.conv for op in ops if op.kind == cabi.OP_CONV]
    if name.startswith(("sfbc", "dbc")) and math_mode != "fp32":
        want = cabi.TF32 if math_mode == "tf32" else cabi.BF16
        assert any(c.out_dtype == want and cabi.conv_choice(c)["family"] == "simt" for c in convs), \
            f"no conv_simt op stores {math_mode}"
    if name == "idql":
        assert any(op.kind == cabi.OP_LNMOD and op.u.lnmod.mod_bstride == 0 for op in ops)
    if name == "sfbc-cfg":
        first = [c for c in convs if c.in_batch_mod or c.res_batch_mod]
        assert any(c.in_batch_mod == plan.batch for c in first) and any(c.res_batch_mod == plan.batch for c in first)
        assert all(cabi.conv_choice(c)["family"] == "simt" for c in first)


def prediction_op(ops):
    """index of the denoiser's final Linear: the last CDS_OP_CONV before the solver update"""
    upd = max(i for i, op in enumerate(ops) if op.kind == cabi.OP_UPDATE)
    return max(i for i in range(upd) if ops[i].kind == cabi.OP_CONV)


def denoiser_check(name, agent, plan, it=1, seed=5, stream=0, sync=lambda: None):
    """{label: normwise relative error} of the program's prediction at iteration ``it`` against the fp64 module, for a
    seeded x_t and condition (the call's own time column).  sfbc-cfg adds the combined prediction
    w pred(cond) + (1 - w) pred(uncond) of its two branches."""
    tab = next(iter(agent._engine_tables.values()))
    t = tab.t
    net = plan.net
    dev = plan.x.device
    B = plan.batch
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(B, *cond_shape(name, net), generator=g).to(dev)
    plan.fill_tables(t, cond)
    plan.x.copy_(torch.randn(plan.x.shape, generator=g).to(dev))
    ops = plan.program.ops
    j = prediction_op(ops)
    plan.handle.run(it, 0, stream, False)                  # the CDS_OPF_ONCE operators, if any
    plan.handle.run_range(it, 0, j + 1, stream)
    sync()
    mem = emulator.Owned(pa.plan_owners(plan))
    y = emulator.view(mem, *pa.declared_outputs(ops[j], it)[0]).to(torch.float64).reshape(-1, plan.x.shape[-1])
    net64 = copy.deepcopy(net).double()
    if t.is_floating_point():
        tt = t[it].to(torch.float64).expand(B)
    else:
        # integer steps (discrete-time and legacy samplers) enter the embedding as int64, whose phase the reference casts
        # to int64 too (utils/embeddings.py): evaluate it as the module does, then widen
        net64.map_noise = _Widened(net.map_noise)
        tt = t[it].expand(B)
    x64 = plan.x.to(torch.float64).reshape(B, -1)
    with torch.no_grad():
        ref = net64(x64, tt, cond.double())
        refs = {"pred": ref}
        if y.shape[0] == 2 * B:                            # two CFG branches: [conditional | unconditional (condition 0)]
            unc = net64(x64, tt, torch.zeros_like(cond, dtype=torch.float64))
            refs = {"pred (cond)": ref, "pred (uncond)": unc, "combined": W_CFG * ref + (1 - W_CFG) * unc}
            ys = {"pred (cond)": y[:B], "pred (uncond)": y[B:], "combined": W_CFG * y[:B] + (1 - W_CFG) * y[B:]}
        else:
            ys = {"pred": y}
    return {k: float((ys[k] - refs[k]).norm() / refs[k].norm()) for k in refs}
