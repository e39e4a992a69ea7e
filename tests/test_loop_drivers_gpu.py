"""Every sampler family through every loop driver on the H100.

One program of every family, built by a real ``sample()`` call at batch 256 (two or more row tiles in every tensor-core
convolution launch) and, where the family allows, 23 iterations (two 10-iteration graphs plus three single ones by default):
SDE DDPM, SDE-DPM-Solver++ 2M with two-branch classifier-free guidance, consistency, ContinuousEDM Heun, the legacy DDPM,
rectified flow, graph-path classifier guidance over HalfJannerUNet1d and over QGPO, callback guidance (a classifier the
lowering refuses) and ``sample(requires_grad=True)`` over DQLMlp, forward and backward.  Each runs in every math mode its
family serves, once per driver, with a fresh agent each (a plan latches CDS_GRAPH_ITERS at its first capture) and one noise
tape for all:
  - the default (graph replay, the whole tape up front);
  - CDS_NOISE_TAPE_MB sized for one and for three slots (the loop in chunks, ``cds_plan_run`` from ``first > 0`` after each
    refill, the CDS_OPF_ONCE cast re-run at every chunk);
  - CDS_GRAPH_ITERS = 1, 3, n_iters and n_iters + 1 (no unrolled graph, several, one, none);
  - CDS_GRAPH = 0 (direct launches).
Every driver gives the bits of the same program run one synchronised operator at a time (program_audit.run_op_by_op), x0
and, for the differentiable program, every gradient.  The golden case of every family run with a one-slot tape and
3-iteration graphs matches its golden within the tolerance its own GPU test states; the module prints the largest error as
a fraction of that tolerance per family."""
import time

import pytest
import torch

import cases
import cg_ref
import grad_ref
import loop_cases as lc
import make_golden_classifier as mgc
import program_audit as pa
import qgpo_ref
import test_guided
import test_legacy_ddpm
import test_rectifiedflow
from common import product_net
from test_edm import build_edm
from test_host_golden import build_agent
from cleandiffuser_b200.diffusion import ContinuousConsistencyModel, DiscreteDiffusionSDE
from cleandiffuser_b200.engine import runtime
from cleandiffuser_b200.nn_condition import IdentityCondition
from cleandiffuser_b200.nn_diffusion import JannerUNet1d
from cleandiffuser_b200.testing import NoiseTape

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, N = 256, 23
GOLDEN_FRAC, WALL = {}, {}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    GOLDEN_FRAC.clear()
    WALL.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print(f"\n[loops] {torch.cuda.get_device_name(0)}: golden error of the chunked run as a fraction of its tolerance")
        for k, v in sorted(GOLDEN_FRAC.items()):
            print(f"[loops] {k:<14} {v:.3f}")
        for k, v in sorted(WALL.items()):
            print(f"[loops] {k}: {v:.1f} s")


@pytest.fixture(autouse=True)
def _engine(monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    for k in ("CDS_BRANCHES", "CDS_GRAPH", "CDS_GRAPH_ITERS", "CDS_NOISE_TAPE_MB"):
        monkeypatch.delenv(k, raising=False)
    torch.backends.cuda.matmul.allow_tf32 = False


def _rows(t):
    """B rows cycling through the rows of ``t`` (a golden case's inputs at the batch of this module)"""
    return None if t is None else t[torch.arange(B, device=t.device) % t.shape[0]]


def _to(kw):
    return {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in kw.items()}


# family -> builder() -> (agent, prior, run(prior) -> x0 or (x0, gradients))
def _sde(name, **over):
    def make():
        spec = dict(cases.sampler_cases()[name], **over)
        agent, inp, kw = build_agent(spec, device=DEV)
        kw = _to(dict(kw, n_samples=B, condition_cfg=_rows(kw["condition_cfg"])))
        return agent, _rows(inp["prior"]).to(DEV), lambda p: agent.sample(p, **kw)[0]
    return make


def _consistency():
    net, _ = product_net(cases.NETS["chi_cm_fourier"])
    agent = ContinuousConsistencyModel(net, IdentityCondition(dropout=0.0), x_max=torch.ones(1, 8, 3), x_min=-torch.ones(1, 8, 3),
                                       device=DEV)
    cond = torch.randn(B, 2, 5, generator=torch.Generator().manual_seed(3)).to(DEV)
    return agent, torch.zeros(B, 8, 3, device=DEV), \
        lambda p: agent.sample(p, n_samples=B, sample_steps=N, condition_cfg=cond, w_cfg=1.0)[0]


def _edm_heun():
    # 2 (steps - 1) + 1 evaluations + 2 Diffusion-X repeats = 23
    agent, inp, kw, _ = build_edm(dict(cases.edm_cases()["edm_heun_mask_clip_dx"], steps=11, diffusion_x=2), device=DEV)
    kw = _to(dict(kw, n_samples=B, condition_cfg=_rows(kw["condition_cfg"])))
    return agent, _rows(inp["prior"]).to(DEV), lambda p: agent.sample(p, **kw)[0]


def _legacy():
    spec = dict(cases.legacy_cases()["ddpm_eps_mask_clip"], T=N)
    agent, inp, kw, _ = test_legacy_ddpm.build(spec, device=DEV)
    kw = _to(dict(kw, n_samples=B, condition_cfg=_rows(kw["condition_cfg"])))
    return agent, _rows(inp["prior"]).to(DEV), lambda p: test_legacy_ddpm.run(agent, spec, p, kw)[0]


def _rf():
    agent, inp, kw = test_rectifiedflow.build(dict(cases.rf_cases()["rf_cont_cfg2branch"], steps=N), device=DEV)
    kw = _to(dict(kw, n_samples=B, condition_cfg=_rows(kw["condition_cfg"])))
    return agent, _rows(inp["prior"]).to(DEV), lambda p: agent.sample(p, **kw)[0]


def _cg_graph():
    """tests/golden/make_golden_classifier.py's DDPM call over T = 23 steps"""
    prior, mask = mgc.sample_inputs()
    clf = cg_ref.make_classifier(dict(horizon=mgc.H, in_dim=mgc.D, dim_mult=(1, 2)), 32, DEV)
    agent = DiscreteDiffusionSDE(mgc.make_denoiser(JannerUNet1d), diffusion_steps=N, fix_mask=mask, predict_noise=True, device=DEV,
                                 classifier=clf)
    return agent, _rows(prior).to(DEV), lambda p: agent.sample(p, solver="ddpm", n_samples=B, sample_steps=N, use_ema=True,
                                                            temperature=0.8, w_cg=mgc.W_CG)[0].detach()


def _qgpo():
    agent, _, kw = qgpo_ref.make_sample_agent("ddpm_eps", device=DEV)
    obs = _rows(kw["condition_cfg"])
    kw = dict(kw, n_samples=B, sample_steps=N, condition_cfg=obs, condition_cg=obs)
    return agent, torch.zeros(B, agent.model["diffusion"].out_layer.out_features, device=DEV), \
        lambda p: agent.sample(p, **kw)[0].detach()


def _cg_callback():
    spec = dict(cases.guided_cases()["cg_disc_ddpm_x0"], T=N, steps=N)
    agent, inp, kw = test_guided.build(spec, device=DEV)
    kw = dict(kw, n_samples=B)
    return agent, _rows(inp["prior"]).to(DEV), lambda p: agent.sample(p, **kw)[0].detach()


def _dql_grad():
    agent, kw = grad_ref.grad_agent("dql-x0", DEV)
    act, obs = grad_ref.GRAD_CASES["dql-x0"]["net"]["act_dim"], grad_ref.GRAD_CASES["dql-x0"]["net"]["obs_dim"]
    g = torch.Generator().manual_seed(5)
    cond0, weight = torch.randn(B, obs, generator=g).to(DEV), torch.randn(B, act, generator=g).to(DEV)

    def run(p):
        agent.model.zero_grad()
        cond = cond0.clone().requires_grad_(True)
        x0, _ = agent.sample(p, n_samples=B, condition_cfg=cond, **dict(kw, sample_steps=N))
        (x0 * weight).sum().backward()
        grads = {n: q.grad.detach().clone() for n, q in agent.model.named_parameters() if q.grad is not None}
        grads["cond"] = cond.grad.detach().clone()
        return x0.detach(), grads
    return agent, torch.zeros(B, act, device=DEV), run


ALL3, NO_BF16 = ("fp32", "tf32", "bf16"), ("fp32", "tf32")
FAMILIES = {
    "sde_ddpm": (_sde("disc_dup_ddpm_x0", T=N, steps=N), ALL3),
    "sde_2m_cfg2": (_sde("cont_cfg2branch_2M", solver="sde_dpmsolver++_2M", steps=N), ALL3),
    "consistency": (_consistency, ALL3),
    "edm_heun": (_edm_heun, ALL3),
    "legacy_ddpm": (_legacy, ALL3),
    "rf": (_rf, ALL3),
    "cg_graph": (_cg_graph, NO_BF16),           # bf16 programs keep the guidance callback
    "qgpo": (_qgpo, NO_BF16),
    "cg_callback": (_cg_callback, ALL3),
    "dql_grad": (_dql_grad, NO_BF16),           # differentiable programs: fp32 and tf32 only
}
GUIDANCE = {"cg_graph": "graph", "qgpo": "graph", "cg_callback": "callback"}


class _OpByOp:
    """a cabi.Plan driven one synchronised operator at a time: ``run`` through program_audit.run_op_by_op, ``run_range``
    split into single operators"""

    def __init__(self, handle, ops):
        self.handle, self.ops = handle, list(ops)

    def run(self, first, count, stream, use_graph=True):
        pa.run_op_by_op(self.handle, self.ops, first, count, stream, torch.cuda.synchronize)

    def run_range(self, it, op_first, op_count, stream):
        for i in range(op_first, op_first + op_count):
            self.handle.run_range(it, i, 1, stream)
            torch.cuda.synchronize()

    def __getattr__(self, name):
        return getattr(self.handle, name)


def _bits_equal(a, b):
    if isinstance(a, tuple):
        return _bits_equal(a[0], b[0]) and a[1].keys() == b[1].keys() and all(_bits_equal(a[1][k], b[1][k]) for k in a[1])
    return pa.same_bits(a, b)


def _describe(a, b):
    if isinstance(a, tuple):
        bad = [k for k in a[1] if not pa.same_bits(a[1][k], b[1][k])]
        return f"x0 {'same' if pa.same_bits(a[0], b[0]) else 'differs'}, gradients that differ: {bad}"
    return f"max |diff| {float((a - b).abs().max()):.3g} over {int((a != b).sum())} elements"


def _run(make, tape, monkeypatch, env=(), op_by_op=False):
    """(result, plan) of one sample() call with a fresh agent under the environment ``env``"""
    with monkeypatch.context() as mp:
        for k, v in env:
            mp.setenv(k, v)
        if op_by_op:
            make_handle = runtime._make_handle
            mp.setattr(runtime, "_make_handle", lambda device, ops, n: _OpByOp(make_handle(device, ops, n), ops))
        agent, prior, run = make()
        calls = runtime.STATS["engine_calls"]
        with tape.active():
            out = run(prior)
        torch.cuda.synchronize()
        assert runtime.STATS["engine_calls"] == calls + 1
        assert not tape.replay or tape.pos == len(tape.draws)
        (plan,) = agent._engine_plans.values()
        return out, plan, prior


@pytest.mark.parametrize("family,math", [(f, m) for f, (_, maths) in FAMILIES.items() for m in maths])
def test_every_driver_gives_the_operator_by_operator_bits(family, math, monkeypatch):
    make, _ = FAMILIES[family]
    monkeypatch.setenv("CDS_MATH", math)
    t0 = time.perf_counter()
    torch.manual_seed(1234)
    tape = NoiseTape()                                         # recorded by the reference run, replayed by every driver
    want, plan, prior = _run(make, tape, monkeypatch, op_by_op=True)
    if family in GUIDANCE:
        assert runtime.STATS["guidance_path"] == GUIDANCE[family], runtime.STATS["guidance_reason"]
    n = plan.n_iters
    n_slots = 0 if plan.noise is None else plan.noise.shape[0]
    assert n == N, n
    x0 = want[0] if isinstance(want, tuple) else want
    assert x0.shape[0] == B and torch.isfinite(x0).all()
    drivers = {"default": (), "tape 1 slot": (("CDS_NOISE_TAPE_MB", lc.tape_mb(1, prior)),),
               "tape 3 slots": (("CDS_NOISE_TAPE_MB", lc.tape_mb(3, prior)),),
               "CDS_GRAPH=0": (("CDS_GRAPH", "0"),)}
    for k in (1, 3, n, n + 1):
        drivers[f"CDS_GRAPH_ITERS={k}"] = (("CDS_GRAPH_ITERS", str(k)),)
    for name, env in drivers.items():
        got, p, _ = _run(make, NoiseTape(tape.draws), monkeypatch, env)
        if "tape" in name and n_slots:
            assert p.noise.shape[0] == min(int(name.split()[1]), n_slots), (name, p.noise.shape)
        assert _bits_equal(got, want), f"{family} {math} {name}: {_describe(got, want)}"
    WALL[f"{family}-{math}"] = time.perf_counter() - t0


@pytest.mark.parametrize("family", list(lc.GOLDEN))
def test_chunked_run_matches_the_golden(family, monkeypatch):
    """the family's golden case with a one-slot tape and 3-iteration graphs: the bits of the default run, the golden within
    the fp32 tolerance of the family's own GPU test"""
    monkeypatch.setenv("CDS_MATH", "fp32")
    out = []
    for chunked in (False, True):
        with monkeypatch.context() as mp:
            agent, prior, run, draws, want = lc.golden_case(family, DEV)
            if chunked:
                mp.setenv("CDS_NOISE_TAPE_MB", lc.tape_mb(1, prior))
                mp.setenv("CDS_GRAPH_ITERS", "3")
            tape = NoiseTape(draws)
            with tape.active():
                out.append(run(prior).cpu())
            assert tape.pos == len(tape.draws)
            (plan,) = agent._engine_plans.values()
            if chunked and plan.noise is not None:
                assert plan.noise.shape[0] == 1
    assert torch.equal(out[0], out[1]), float((out[0] - out[1]).abs().max())
    frac = lc.GPU_TOL[lc.GOLDEN[family][0]](out[1].numpy(), want)
    GOLDEN_FRAC[family] = frac
    assert frac <= 1.0, (family, frac)
