"""``sample(requires_grad=True)`` over DQLMlp on the H100: the backward operators (csrc/grad.cuh) against fp64 through
``cds_run_op``, whole-call gradients against fp64 autograd of the PyTorch reverse loop, bitwise reproducibility, graph replay
against direct launches, and a short Diffusion-QL-style actor training run against CDS_BACKEND=torch.

Bounds are fractions of a rounding bound with the unit roundoff u of the arithmetic (fp32: 2^-24; TF32 tensor-core forward:
2^-11): a GEMM-shaped output of reduction length n is bounded by (n + c) u sum|terms| (the standard dot-product bound), a
whole-call gradient by C u ||ref|| with the C stated next to it.  The largest fraction seen is printed per check."""
import copy
import math

import numpy as np
import pytest
import torch

import grad_ref
from cleandiffuser_b200.diffusion import ContinuousDiffusionSDE, DiscreteDiffusionSDE
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
            print(f"[grad] {name}: largest error = {frac:.3g} of the bound")


def _record(name, frac):
    WORST[name] = max(WORST.get(name, 0.0), float(frac))
    assert frac <= 1.0, (name, frac)


def _run(op):
    cabi.run_op(0, op, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


# ================================================================================================ per-operator parity
@pytest.mark.parametrize("rows", [37, 256, 1000])
@pytest.mark.parametrize("dims", D4RL)
@pytest.mark.parametrize("layer", ["hidden", "final", "input"])
def test_dgrad_wgrad_operators(rows, dims, layer):
    act_dim = dims[1]
    N, K, mish = {"hidden": (256, 256, True), "final": (act_dim, 256, True), "input": (256, act_dim, False)}[layer]
    g = torch.Generator().manual_seed(rows * 7 + act_dim)
    dz = torch.randn(rows, N, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(N)
    z = torch.randn(2, rows, K, generator=g) * 2            # two stash slots: the operator must read slot 1
    prev = torch.randn(rows, K, generator=g)
    act = cabi.ACT_MISH if mish else cabi.ACT_NONE
    # ---- dgrad, accumulate + out_sum
    d_dz, d_w, d_z, d_out, d_sum = (t.to(DEV) for t in (dz, w, z, prev.clone(), prev.clone()))
    op = cabi.Op()
    op.kind = cabi.OP_DGRAD
    d = op.u.dgrad
    d.rows, d.N, d.K, d.dz, d.ldz, d.w, d.ldw = rows, N, K, d_dz.data_ptr(), N, d_w.data_ptr(), K
    if mish:
        d.z, d.z_iter_stride = d_z.data_ptr() + 4 * rows * K, -rows * K      # iter 0 -> slot 1 (signed stride)
        d.act = act
    d.accumulate, d.out, d.ldo, d.out_sum = 1, d_out.data_ptr(), K, d_sum.data_ptr()
    _run(op)
    zz = z[1].double().numpy()
    y = grad_ref.dgrad(dz.numpy(), w.numpy(), zz, act)
    mg = np.abs(grad_ref.mish_grad(zz)) if mish else 1.0
    mag = (np.abs(dz.double().numpy()) @ np.abs(w.double().numpy())) * mg
    # fp32 Mish derivative: tanh(softplus(z)) and 1 - tanh^2 carry absolute errors of a few u, scaled by |z| through z sigmoid(z)
    mg_err = (8 + 8 * np.abs(zz)) * U32 if mish else 0.0
    bound = (N + 4) * U32 * mag + np.abs(dz.double().numpy() @ w.double().numpy()) * mg_err + \
        2 * U32 * (np.abs(prev.double().numpy()) + np.abs(y)) + 1e-30
    for got in (d_out, d_sum):
        err = np.abs(got.cpu().double().numpy() - (prev.double().numpy() + y))
        _record(f"dgrad {layer}", (err / bound).max())
    # ---- wgrad, accumulate, bias column (per-iteration row with a signed stride)
    dw0 = torch.randn(N, K, generator=g)
    db0 = torch.randn(2, N, generator=g)
    d_dw, d_db = dw0.to(DEV), db0.to(DEV)
    op = cabi.Op()
    op.kind = cabi.OP_WGRAD
    q = op.u.wgrad
    q.rows, q.N, q.K, q.dz, q.ldz = rows, N, K, d_dz.data_ptr(), N
    q.h, q.h_iter_stride, q.ldh, q.act = d_z.data_ptr() + 4 * rows * K, -rows * K, K, act
    q.dw, q.lddw, q.db, q.db_iter_stride, q.accumulate = d_dw.data_ptr(), K, d_db.data_ptr() + 4 * N, -N, 1
    _run(op)
    gw, gb = grad_ref.wgrad(dz.numpy(), zz, act)
    hmag = np.abs(grad_ref.act(act, zz))
    adz = np.abs(dz.double().numpy())
    bw = (rows + 8) * U32 * (adz.T @ hmag) + 2 * U32 * (np.abs(dw0.double().numpy()) + np.abs(gw)) + 1e-30
    bb = (rows + 2) * U32 * adz.sum(0) + 2 * U32 * (np.abs(db0[1].double().numpy()) + np.abs(gb)) + 1e-30
    _record(f"wgrad {layer}", (np.abs(d_dw.cpu().double().numpy() - (dw0.double().numpy() + gw)) / bw).max())
    _record(f"wgrad {layer} bias", (np.abs(d_db[1].cpu().double().numpy() - (db0[1].double().numpy() + gb)) / bb).max())
    assert torch.equal(d_db[0].cpu(), db0[0]), "wgrad wrote outside its iteration's bias row"


def _coef_row(kind, alpha=0.7, sigma=0.55, k0=1.2, k1=0.35):
    t = torch.zeros(2, cabi.ROW_FLOATS)
    t[1, 0], t[1, 1], t[1, 2], t[1, 3], t[1, 7] = alpha, sigma, k0, k1, float(kind)
    return t


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
@pytest.mark.parametrize("predict_noise", [True, False])
@pytest.mark.parametrize("bounds", ["both", "min", "max", "none"])
@pytest.mark.parametrize("act_dim", [3, 9])
def test_update_bwd_operator(kind, predict_noise, bounds, act_dim):
    """clipped elements and exact ties with a bound (the bound computed in fp32 like the kernel does), fix_mask, 1000 rows"""
    B = 1000
    g = torch.Generator().manual_seed(kind * 31 + act_dim)
    x = torch.randn(B, act_dim, generator=g)
    pred = torch.randn(B, act_dim, generator=g) * 2
    gx = torch.randn(B, act_dim, generator=g)
    mask = (torch.arange(act_dim) == 1).float()
    x_min = None if bounds in ("max", "none") else torch.full((act_dim,), -0.6)
    x_max = None if bounds in ("min", "none") else torch.full((act_dim,), 0.8)
    coef = _coef_row(kind)
    alpha, sigma = coef[1, 0], coef[1, 1]
    if predict_noise:       # fp32 op-by-op, as the kernel: (x - alpha*lim)/sigma
        lo = None if x_max is None else (x - alpha * x_max) / sigma
        hi = None if x_min is None else (x - alpha * x_min) / sigma
    else:
        lo, hi = x_min, x_max
    full = lambda b: torch.broadcast_to(b, (B, act_dim))        # noqa: E731
    if lo is not None:
        pred[:50] = full(lo)[:50]
    if hi is not None:
        pred[50:100] = full(hi)[50:100]
    stash_x = torch.stack([torch.zeros_like(x), x])            # slot 1 is the iteration's
    stash_p = torch.stack([torch.zeros_like(pred), pred])
    dev = {k: (v.to(DEV) if v is not None else None) for k, v in dict(gx=gx.clone(), gp=torch.zeros_like(gx), x=stash_x,
                                                                        p=stash_p, m=mask, lo=x_min, hi=x_max, c=coef).items()}
    op = cabi.Op()
    op.kind = cabi.OP_UPDATE_BWD
    u = op.u.update_bwd
    u.batch, u.row, u.gx, u.gpred = B, act_dim, dev["gx"].data_ptr(), dev["gp"].data_ptr()
    u.x, u.x_iter_stride = dev["x"].data_ptr() + 4 * B * act_dim, -B * act_dim
    u.pred, u.pred_iter_stride = dev["p"].data_ptr() + 4 * B * act_dim, -B * act_dim
    u.mask = dev["m"].data_ptr()
    u.x_min = dev["lo"].data_ptr() if x_min is not None else None
    u.x_max = dev["hi"].data_ptr() if x_max is not None else None
    u.coef, u.coef_iter_stride = dev["c"].data_ptr() + 4 * cabi.ROW_FLOATS, -cabi.ROW_FLOATS
    u.predict_noise = int(predict_noise)
    _run(op)
    r = coef[1].double().numpy()
    gp, dx = grad_ref.update_bwd(gx.numpy(), x.numpy(), pred.numpy(), alpha=r[0], sigma=r[1], k0=r[2], k1=r[3], kind=kind,
                                 predict_noise=predict_noise, mask=mask.numpy(),
                                 x_min=None if x_min is None else x_min.numpy(), x_max=None if x_max is None else x_max.numpy())
    # a handful of fp32 operations per element, each within u of its exact result; the terms are at most |g| (|k0| + |k1|)
    # (1 + 1/alpha + 1/sigma)^2 in size
    scale = np.abs(gx.double().numpy()) * (abs(r[2]) + abs(r[3])) * (1 + 1 / r[0] + 1 / r[1]) ** 2
    bound = 16 * U32 * scale + 1e-30
    _record("update_bwd d pred", (np.abs(dev["gp"].cpu().double().numpy() - gp) / bound).max())
    _record("update_bwd d x", (np.abs(dev["gx"].cpu().double().numpy() - dx) / bound).max())


# ================================================================================================ whole calls
class _Fp64(torch.nn.Module):
    def __init__(self, m):
        super().__init__()
        self.m = m

    def forward(self, t):
        return self.m(t).double()


def _agent(net, kind="discrete", dtype=torch.float32, predict_noise=True, clip=True):
    a = net.final_layer.out_features
    kw = dict(predict_noise=predict_noise, device=DEV)
    if clip:
        kw.update(x_max=torch.full((1, a), 1.0, dtype=dtype), x_min=torch.full((1, a), -1.0, dtype=dtype))
    if kind == "discrete":
        return DiscreteDiffusionSDE(net, IdentityCondition(dropout=0.0), diffusion_steps=5, **kw)
    return ContinuousDiffusionSDE(net, IdentityCondition(dropout=0.0), **kw)


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


@pytest.mark.parametrize("math_mode", ["fp32", "tf32"])
@pytest.mark.parametrize("batch", [256, 4096])
@pytest.mark.parametrize("solver", ["ddpm", "ddim"])
def test_whole_call_gradients(math_mode, batch, solver, monkeypatch):
    """every DQLMlp parameter and the condition: || engine - fp64 autograd of the loop || <= C u || fp64 ||, C = 4096
    (fp32) or 16 (TF32 forward GEMMs), over Diffusion-QL's call (5 steps, eps-prediction, w_cfg = 1).
    fp32 clips to [-1, 1] like Diffusion-QL.  TF32 runs unclipped: a prediction within TF32 rounding (~1e-3) of a bound can
    be clipped on one side and not on the other, which moves that element's whole gradient between the network and x_t -- a
    discrete difference, not a rounding error, that no rounding bound covers (the clip rule itself is pinned by
    test_update_bwd_operator and by the fp32 case)."""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math_mode)
    obs, act = 17, 6
    net = load_synth(DQLMlp(obs, act, emb_dim=16), seed=1).to(DEV)
    clip = math_mode == "fp32"
    agent = _agent(net, clip=clip)
    prior, cond, weight = _inputs(batch, obs, act)
    torch.manual_seed(11)                                          # the noise draws do not depend on the tests before
    tape = NoiseTape()
    before = runtime.STATS["engine_calls"]
    _, got = _grads(agent, prior, cond, weight, tape, solver=solver, sample_steps=5)
    assert runtime.STATS["engine_calls"] == before + 1
    monkeypatch.setenv("CDS_BACKEND", "torch")
    net64 = copy.deepcopy(net).double()
    net64.map_noise = _Fp64(net64.map_noise)
    _, want = _grads(_agent(net64, dtype=torch.float64, clip=clip), prior.double(), cond.double(), weight.double(), NoiseTape(tape.draws),
                     solver=solver, sample_steps=5)
    C, u = (4096, U32) if math_mode == "fp32" else (16, UTF32)
    for name in want:
        err = (got[name] - want[name]).norm().item()
        _record(f"whole call {math_mode} B={batch} {solver} {name}", err / (C * u * want[name].norm().item() + 1e-30))


def test_backward_is_bitwise_reproducible_and_graph_equals_direct(monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "tf32")
    obs, act = 11, 3
    net = load_synth(DQLMlp(obs, act, emb_dim=16), seed=3).to(DEV)
    agent = _agent(net, kind="continuous", predict_noise=False)
    prior, cond, weight = _inputs(1000, obs, act)
    torch.manual_seed(12)
    tape = NoiseTape()
    runs = []
    for graph in ("1", "1", "0"):
        monkeypatch.setenv("CDS_GRAPH", graph)
        x0, g = _grads(agent, prior, cond, weight, tape if not runs else NoiseTape(tape.draws), solver="sde_dpmsolver++_1",
                       sample_steps=5, diffusion_x_sampling_steps=2)
        runs.append((x0, g))
    for x0, g in runs[1:]:
        assert torch.equal(x0, runs[0][0])
        for name in g:
            assert torch.equal(g[name], runs[0][1][name]), name


def test_dql_actor_training_matches_pytorch_loop(monkeypatch):
    """20 Diffusion-QL actor steps (bc loss + eta * q loss against a fixed random critic, Adam) on the engine and on the
    PyTorch loop from the same initial weights, batches and noise.  The weights change in place at every step, so the engine
    re-packs them on every call (a stale copy would make the two runs drift apart at once).  Bound: Adam moves an element by at
    most ~lr per step whatever the gradient, so |engine - torch| <= 2 lr steps for every element; the mean stays far below."""
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
        actor = _agent(copy.deepcopy(base).to(DEV))
        opt = torch.optim.Adam(actor.model.parameters(), lr=lr)
        calls = runtime.STATS["engine_calls"]
        for s, (o, a) in enumerate(data):
            tape = tapes[s] if backend == "cuda" else NoiseTape(tapes[s].draws)
            torch.manual_seed(100 + s)
            with tape.active():
                bc = actor.loss(a, o)
                new_act, _ = actor.sample(torch.zeros(B, act, device=DEV), solver="ddpm", n_samples=B, sample_steps=5,
                                          use_ema=False, condition_cfg=o, w_cfg=1.0, requires_grad=True)
            q = critic(torch.cat([o, new_act], 1))
            loss = bc - eta * q.mean() / q.abs().mean().detach()
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
    _record("training max |engine - torch| / (2 lr steps)", diffs.max().item() / (2 * lr * steps))
    _record("training mean |engine - torch| / (0.05 lr steps)", diffs.mean().item() / (0.05 * lr * steps))
    assert moved.mean().item() > 0.1 * lr * steps                  # the weights did move
