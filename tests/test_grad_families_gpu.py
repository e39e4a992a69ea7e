"""``sample(requires_grad=True)`` with ContinuousConsistencyModel and RectifiedFlow over DQLMlp on the H100: CDS_OP_UPDATE_BWD's
kind CM and CDS_OP_PREP's backward mode against fp64 through ``cds_run_op``, an operator-by-operator audit of both programs,
whole-call gradients against fp64 autograd of the PyTorch loop, bitwise reproducibility (graph replay, direct launches, a
chunked noise tape), and 20 CPQL-shaped actor steps against CDS_BACKEND=torch.

Bounds follow tests/test_grad_sampling_gpu.py: an operator output within a rounding bound (few_step_grad_ref), a whole-call
gradient within C u ||ref|| (fp32: C = 4096, u = 2^-24; TF32 forward GEMMs: C = 16, u = 2^-11).  The TF32 calls run unclipped,
for the reason that file gives: a value within TF32 rounding of a bound can be clipped on one side of the comparison and not
on the other, a discrete difference no rounding bound covers.  The largest fraction seen is printed per check."""
import copy

import numpy as np
import pytest
import torch

import few_step_grad_ref
import program_audit as pa
from cleandiffuser_b200.diffusion import ContinuousConsistencyModel, ContinuousRectifiedFlow, DiscreteRectifiedFlow
from cleandiffuser_b200.diffusion import solvers as S
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import DQLMlp
from cleandiffuser_b200.testing import NoiseTape, load_synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U32 = 2.0 ** -24
UTF32 = 2.0 ** -11
D4RL = [(11, 3), (17, 6), (29, 8), (60, 9)]           # (obs_dim, act_dim): hopper, halfcheetah / walker2d, antmaze, kitchen
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    WORST.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print()
        for name, frac in sorted(WORST.items()):
            print(f"[grad families] {name}: largest error = {frac:.3g} of the bound")


def _record(name, frac):
    WORST[name] = max(WORST.get(name, 0.0), float(frac))
    assert frac <= 1.0, (name, frac)


def _run(op):
    cabi.run_op(0, op, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


# ================================================================================================ per-operator parity
def _coef(kind, k0=0.3, k1=0.5, k3=0.7):
    """two rows; the operator at iteration 0 reads row 1 through a signed stride"""
    t = torch.zeros(2, cabi.ROW_FLOATS)
    t[1, S.R_K0], t[1, S.R_K1], t[1, S.R_K3], t[1, S.R_KIND] = k0, k1, k3, float(kind)
    return t


@pytest.mark.parametrize("rows", [37, 1000])
@pytest.mark.parametrize("dims", D4RL)
@pytest.mark.parametrize("bounds", ["both", "min", "max", "none"])
def test_update_bwd_cm_operator(rows, dims, bounds):
    """kind CM: f recomputed in fp32, ties with a bound pass their gradient (rows with x = 0: f = 0.5 pred = the bound
    exactly), x_min > x_max in column 1 passes none, fix_mask on column 0"""
    a = dims[1]
    g = torch.Generator().manual_seed(rows + a)
    x = torch.randn(rows, a, generator=g) * 3
    pred = torch.randn(rows, a, generator=g)
    gx = torch.randn(rows, a, generator=g)
    mask = (torch.arange(a) == 0).float()
    x_min = None if bounds in ("max", "none") else torch.linspace(-0.6, -0.2, a)
    x_max = None if bounds in ("min", "none") else torch.linspace(0.3, 0.8, a)
    if x_min is not None and x_max is not None:
        x_min[1], x_max[1] = 0.4, -0.4
    x[:20] = 0.0
    if x_min is not None:
        pred[:10] = x_min / 0.5
    if x_max is not None:
        pred[10:20] = x_max / 0.5
    coef = _coef(S.UPD_CM)
    stash_x, stash_p = torch.stack([torch.zeros_like(x), x]), torch.stack([torch.zeros_like(pred), pred])
    dev = {k: (v.to(DEV) if v is not None else None) for k, v in dict(gx=gx.clone(), gp=torch.zeros_like(gx), x=stash_x,
                                                                        p=stash_p, m=mask, lo=x_min, hi=x_max, c=coef).items()}
    op = cabi.Op()
    op.kind = cabi.OP_UPDATE_BWD
    u = op.u.update_bwd
    u.batch, u.row, u.gx, u.gpred = rows, a, dev["gx"].data_ptr(), dev["gp"].data_ptr()
    u.x, u.x_iter_stride = dev["x"].data_ptr() + 4 * rows * a, -rows * a
    u.pred, u.pred_iter_stride = dev["p"].data_ptr() + 4 * rows * a, -rows * a
    u.mask = dev["m"].data_ptr()
    u.x_min = dev["lo"].data_ptr() if x_min is not None else None
    u.x_max = dev["hi"].data_ptr() if x_max is not None else None
    u.coef, u.coef_iter_stride = dev["c"].data_ptr() + 4 * cabi.ROW_FLOATS, -cabi.ROW_FLOATS
    _run(op)
    r = coef[1].double().numpy()
    gp, dx = few_step_grad_ref.cm_update_bwd(gx.numpy(), x.numpy(), pred.numpy(), k0=r[S.R_K0], k1=r[S.R_K1], mask=mask.numpy(),
                                             x_min=None if x_min is None else x_min.numpy(),
                                             x_max=None if x_max is None else x_max.numpy())
    bound = few_step_grad_ref.cm_update_bwd_bound(gx.numpy(), r[S.R_K0], r[S.R_K1]) + 1e-30
    _record("update_bwd cm d pred", (np.abs(dev["gp"].cpu().double().numpy() - gp) / bound).max())
    _record("update_bwd cm d x", (np.abs(dev["gx"].cpu().double().numpy() - dx) / bound).max())
    if bounds != "none":
        assert (gp[:20][:, 2:] != 0).any() and (gp[:20] == 0).any()     # ties pass; masked / empty-interval columns do not


def test_update_bwd_kind_without_backward_writes_nan():
    """kinds X2M, EDM, EDM_HEUN have no backward: both outputs are NaN, never another kind's formula"""
    for kind in (S.UPD_X2M, S.UPD_EDM, S.UPD_EDM_HEUN):
        B, a = 40, 3
        t = {k: torch.randn(2, B, a, device=DEV) for k in ("x", "p")}
        gx, gp, coef = torch.randn(B, a, device=DEV), torch.zeros(B, a, device=DEV), _coef(kind).to(DEV)
        op = cabi.Op()
        op.kind = cabi.OP_UPDATE_BWD
        u = op.u.update_bwd
        u.batch, u.row, u.gx, u.gpred = B, a, gx.data_ptr(), gp.data_ptr()
        u.x, u.pred, u.coef = t["x"].data_ptr(), t["p"].data_ptr(), coef.data_ptr() + 4 * cabi.ROW_FLOATS
        _run(op)
        assert torch.isnan(gx).all() and torch.isnan(gp).all(), kind


@pytest.mark.parametrize("rows", [37, 256, 1000])
@pytest.mark.parametrize("dims", D4RL)
def test_prep_bwd_operator(rows, dims):
    """gx += K3 * gxin: fp32 product then fp32 sum, bit for bit; the row of iteration 0 through a signed stride"""
    a = dims[1]
    g = torch.Generator().manual_seed(rows * 3 + a)
    gx, gxin = torch.randn(rows, a, generator=g), torch.randn(rows, a, generator=g)
    coef = _coef(S.UPD_CM, k3=0.0123456)
    d_gx, d_gxin, d_coef = gx.to(DEV), gxin.to(DEV), coef.to(DEV)
    op = cabi.Op()
    op.kind = cabi.OP_PREP
    q = op.u.prep
    q.batch, q.row, q.x, q.gxin = rows, a, d_gx.data_ptr(), d_gxin.data_ptr()
    q.coef, q.coef_iter_stride = d_coef.data_ptr() + 4 * cabi.ROW_FLOATS, -cabi.ROW_FLOATS
    _run(op)
    want = few_step_grad_ref.prep_bwd(gx.numpy(), gxin.numpy(), coef[1, S.R_K3].item())
    assert np.array_equal(d_gx.cpu().numpy().view(np.int32), want.view(np.int32))


# ================================================================================================ whole calls
class _Fp64(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, t):
        return self.m(t).double()


def _agent(family, net, dtype=torch.float32, clip=True, mask=False):
    a = net.final_layer.out_features
    kw = dict(device=DEV)
    if clip:
        kw.update(x_max=torch.full((1, a), 1.0, dtype=dtype), x_min=torch.full((1, a), -1.0, dtype=dtype))
    if mask:
        m = torch.zeros(a, dtype=dtype)
        m[0] = 1.
        kw["fix_mask"] = m
    if family == "cm":
        return ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), **kw)
    if family == "rf_discrete":
        return DiscreteRectifiedFlow(net, IdentityCondition(dropout=0.0), diffusion_steps=100, **kw)
    return ContinuousRectifiedFlow(net, IdentityCondition(dropout=0.0), **kw)


def _grads(agent, prior, cond, weight, tape, **kw):
    agent.model.zero_grad()
    cond = cond.clone().requires_grad_(True)
    with tape.active():
        x0, _ = agent.sample(prior, n_samples=prior.shape[0], use_ema=False, condition_cfg=cond, w_cfg=1.0,
                             requires_grad=True, **kw)
    (x0 * weight).sum().backward()
    out = {n: p.grad.detach().double().clone() for n, p in agent.model.named_parameters() if p.grad is not None}
    out["cond"] = cond.grad.detach().double().clone()
    return x0.detach(), out


def _inputs(batch, obs, act, seed=5):
    g = torch.Generator().manual_seed(seed)
    return (torch.zeros(batch, act).to(DEV), torch.randn(batch, obs, generator=g).to(DEV),
            torch.randn(batch, act, generator=g).to(DEV))


CALLS = {"cm-1": ("cm", dict(sample_steps=1)), "cm-2": ("cm", dict(sample_steps=2)),
         "rf-5": ("rf_continuous", dict(sample_steps=5)), "rf-discrete-5": ("rf_discrete", dict(sample_steps=5))}


@pytest.mark.parametrize("math_mode", ["fp32", "tf32"])
@pytest.mark.parametrize("batch", [256, 4096])
@pytest.mark.parametrize("call", list(CALLS))
def test_whole_call_gradients(call, batch, math_mode, monkeypatch):
    """every DQLMlp parameter and the condition: || engine - fp64 autograd of the loop || <= C u || fp64 ||; fp32 clips to
    [-1, 1] like CPQL's actor, TF32 runs unclipped"""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math_mode)
    family, kw = CALLS[call]
    obs, act = 17, 6
    net = load_synth(DQLMlp(obs, act, emb_dim=16), seed=1).to(DEV)
    clip = math_mode == "fp32"
    prior, cond, weight = _inputs(batch, obs, act)
    torch.manual_seed(11)
    tape = NoiseTape()
    before = runtime.STATS["engine_calls"]
    _, got = _grads(_agent(family, net, clip=clip), prior, cond, weight, tape, **kw)
    assert runtime.STATS["engine_calls"] == before + 1
    monkeypatch.setenv("CDS_BACKEND", "torch")
    net64 = copy.deepcopy(net).double()
    net64.map_noise = _Fp64(net64.map_noise)
    _, want = _grads(_agent(family, net64, dtype=torch.float64, clip=clip), prior.double(), cond.double(), weight.double(),
                     NoiseTape(tape.draws), **kw)
    C, u = (4096, U32) if math_mode == "fp32" else (16, UTF32)
    for name in want:
        err = (got[name] - want[name]).norm().item()
        _record(f"whole call {call} {math_mode} B={batch} {name}", err / (C * u * want[name].norm().item() + 1e-30))


@pytest.mark.parametrize("family", ["cm", "rf_continuous"])
def test_backward_is_bitwise_reproducible_graph_direct_and_chunked(family, monkeypatch):
    """two graph-replayed calls, direct launches (CDS_GRAPH=0) and a one-slot noise tape refilled between chunks
    (CDS_NOISE_TAPE_MB) give the same x0 and gradients bit for bit"""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "tf32")
    obs, act, B = 11, 3, 1000
    net = load_synth(DQLMlp(obs, act, emb_dim=16), seed=3).to(DEV)
    agent = _agent(family, net, mask=True)
    prior, cond, weight = _inputs(B, obs, act)
    torch.manual_seed(12)
    tape = NoiseTape()
    kw = dict(sample_steps=3, diffusion_x_sampling_steps=1)
    runs = []
    for graph, tape_mb in (("1", None), ("1", None), ("0", None), ("1", "0.01")):
        monkeypatch.setenv("CDS_GRAPH", graph)
        if tape_mb is not None:
            monkeypatch.setenv("CDS_NOISE_TAPE_MB", tape_mb)
        x0, g = _grads(agent, prior, cond, weight, tape if not runs else NoiseTape(tape.draws), **kw)
        runs.append((x0, g))
    if family == "cm":
        assert sorted(p.noise.shape[0] for p in agent._engine_plans.values()) == [1, 3]      # the chunked plan's tape: 1 slot
    for x0, g in runs[1:]:
        assert torch.equal(x0, runs[0][0])
        for name in g:
            assert torch.equal(g[name], runs[0][1][name]), name


@pytest.mark.parametrize("call", ["cm-2", "rf-discrete-5"])
@pytest.mark.parametrize("math_mode", ["fp32", "tf32"])
def test_programs_match_fp64_operator_by_operator(call, math_mode, monkeypatch):
    """every operator of every forward and backward iteration at a ragged batch against fp64 (tests/program_audit.py, taught
    kind CM and PREP's backward mode by few_step_grad_ref), with no write outside its declared outputs"""
    few_step_grad_ref.register(monkeypatch)
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math_mode)
    family, kw = CALLS[call]
    obs, act, B = 17, 6, 333
    agent = _agent(family, load_synth(DQLMlp(obs, act, emb_dim=16), seed=1).to(DEV), mask=True)
    prior, cond, _ = _inputs(B, obs, act)
    agent.sample(prior, n_samples=B, use_ema=False, condition_cfg=cond, w_cfg=1.0, requires_grad=True, **kw)
    (plan,) = agent._engine_plans.values()
    torch.cuda.synchronize()
    fa, ba = pa.audit_grad_plan(f"{call}-{math_mode}", plan, plan.handle, plan.back_handle,
                                torch.cuda.current_stream().cuda_stream, torch.cuda.synchronize)
    for aud in (fa, ba):
        for inst, (frac, where) in aud.worst.items():
            WORST[f"audit {aud.name} {inst}"] = max(WORST.get(f"audit {aud.name} {inst}", 0.0), frac)
    assert not fa.failures and not ba.failures, "\n".join((fa.failures + ba.failures)[:20])
    kinds = {op.kind for op in plan.back.ops}
    assert (cabi.OP_PREP in kinds) == (family == "cm")


def test_cpql_actor_training_matches_pytorch_loop(monkeypatch):
    """20 CPQL-shaped actor steps (a 2-step consistency policy clipped to [-1, 1]; loss = behaviour-cloning MSE of the sampled
    action + eta * Q loss against a fixed random critic, Adam) on the engine and on the PyTorch loop from the same initial
    weights, batches and noise.  Adam moves an element by at most ~lr per step, so |engine - torch| <= 2 lr steps for every
    element, and the mean stays far below."""
    monkeypatch.setenv("CDS_MATH", "fp32")
    obs, act, B, steps, lr, eta = 17, 6, 256, 20, 3e-4, 1.0
    torch.manual_seed(0)
    critic = torch.nn.Sequential(torch.nn.Linear(obs + act, 64), torch.nn.Mish(), torch.nn.Linear(64, 1)).to(DEV)
    critic.requires_grad_(False)
    base = load_synth(DQLMlp(obs, act, emb_dim=16), seed=4)
    g = torch.Generator().manual_seed(9)
    data = [(torch.randn(B, obs, generator=g).to(DEV), torch.randn(B, act, generator=g).clamp(-1, 1).to(DEV)) for _ in range(steps)]
    finals, tapes = {}, [NoiseTape() for _ in range(steps)]
    for backend in ("cuda", "torch"):
        monkeypatch.setenv("CDS_BACKEND", backend)
        actor = _agent("cm", copy.deepcopy(base).to(DEV))
        opt = torch.optim.Adam(actor.model.parameters(), lr=lr)
        calls = runtime.STATS["engine_calls"]
        for s, (o, a) in enumerate(data):
            tape = tapes[s] if backend == "cuda" else NoiseTape(tapes[s].draws)
            with tape.active():
                new_act, _ = actor.sample(torch.zeros(B, act, device=DEV), n_samples=B, sample_steps=2, use_ema=False,
                                          condition_cfg=o, requires_grad=True)
            q = critic(torch.cat([o, new_act], 1))
            loss = ((new_act - a) ** 2).mean() - eta * q.mean() / q.abs().mean().detach()
            opt.zero_grad()
            loss.backward()
            opt.step()
        if backend == "cuda":
            assert runtime.STATS["engine_calls"] == calls + steps
            assert len(actor._engine_plans) == 1                   # one plan, re-packed after every optimiser step
        finals[backend] = {n: p.detach().clone() for n, p in actor.model.named_parameters()}
    diffs = torch.cat([(finals["cuda"][n] - finals["torch"][n]).abs().flatten() for n in finals["torch"]])
    moved = torch.cat([(finals["torch"][n] - base.state_dict()[n.split(".", 1)[1]].to(DEV)).abs().flatten()
                       for n in finals["torch"] if n.startswith("diffusion.")])
    _record("cpql training max |engine - torch| / (2 lr steps)", diffs.max().item() / (2 * lr * steps))
    _record("cpql training mean |engine - torch| / (0.05 lr steps)", diffs.mean().item() / (0.05 * lr * steps))
    assert moved.mean().item() > 0.1 * lr * steps                  # the weights did move
