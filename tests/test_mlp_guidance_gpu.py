"""Classifier guidance with MLPNNClassifier inside the replayed loop on the H100: CDS_OP_STASH / CDS_OP_DGRAD with ReLU against
fp64 (tests/relu_ref.py: ReLU and its derivative are exact, so the STASH must be bitwise and the DGRAD within the dot-product
bound), the lowered input gradient against fp64 autograd, the reference tutorial's guided call against the host-callback
path, the goldens, graph replay / reproducibility, and an operator-by-operator audit of the guided iteration
(tests/program_audit.py)."""
import numpy as np
import pytest
import torch

import cg_ref
import emulator
import grad_ref
import make_golden_mlp_classifier as mg
import mlp_cg_ref
import program_audit as pa
import relu_ref
from common import load_golden, tape_of
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape, load_synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}
ROWS = [50, 333, 4096]             # the tutorial's 50 envs, a count that is no multiple of 32, a large batch
WIDTHS = [9, 60, 256]              # the tutorial's action (x_dim), observation (out_dim) and hidden widths


@pytest.fixture(autouse=True)
def relu_semantics(monkeypatch):
    relu_ref.register(monkeypatch)     # CDS_ACT_RELU in the shared operator references for this test (tests/relu_ref.py)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _run(op, it=0):
    cabi.run_op(0, op, it, _stream())
    torch.cuda.synchronize()


def _frac(got, want, bound):
    err = np.abs(got.cpu().numpy().astype(np.float64) - want)
    return float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), np.where(err > 0, np.inf, 0.0))))


def _with_zeros(t, g):
    """about one element in eight set to exactly 0 (the ReLU derivative's tie), plus +-0 at the front"""
    t = t.clone()
    t[torch.rand(t.shape, generator=g) < 0.125] = 0.0
    t.view(-1)[:2] = torch.tensor([0.0, -0.0])
    return t


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("width", WIDTHS)
def test_stash_relu_is_exact(rows, width):
    """act_out = relu(src) bit for bit (a select), with and without the slot copy; nothing written past n"""
    n = rows * width
    g = torch.Generator().manual_seed(n)
    src = _with_zeros(4 * torch.randn(n, generator=g), g).to(DEV)
    slots = torch.full((2, n + 3), 7.0, device=DEV)
    out = torch.full((n + 3,), 7.0, device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_STASH
    s = op.u.stash
    s.n, s.act, s.src, s.act_out = n, cabi.ACT_RELU, src.data_ptr(), out.data_ptr()
    s.dst, s.dst_iter_stride = slots.data_ptr(), n + 3
    _run(op, 1)
    want = torch.relu(src)
    assert torch.equal(out[:n], want) and bool((out[:n] >= 0).all())
    assert bool((out[:n][src == 0] == 0).all())
    assert bool((out[n:] == 7.0).all()) and torch.equal(slots[1, :n], src) and bool((slots[0] == 7.0).all())
    frac = _frac(out[:n], grad_ref.act(cabi.ACT_RELU, src.cpu().numpy()), grad_ref.ACT_BOUND[cabi.ACT_RELU](src.cpu().numpy()))
    assert frac == 0.0, frac


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("N", WIDTHS)
@pytest.mark.parametrize("K", WIDTHS)
def test_dgrad_relu_matches_fp64(rows, N, K):
    """out = (dz W) relu'(z) under grad_ref.dgrad_bound (exactly 0 where z <= 0, including z == 0), bitwise equal over two
    runs"""
    g = torch.Generator().manual_seed(rows + 7 * N + K)
    dz, w = torch.randn(rows, N, generator=g), torch.randn(N, K, generator=g) / N ** 0.5
    z = _with_zeros(3 * torch.randn(2, rows, K, generator=g), g)
    dz, w, z = dz.to(DEV), w.to(DEV), z.to(DEV)
    out = torch.full((rows, K), 7.0, device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_DGRAD
    d = op.u.dgrad
    d.rows, d.N, d.K, d.dz, d.ldz, d.w, d.ldw = rows, N, K, dz.data_ptr(), N, w.data_ptr(), K
    d.z, d.z_iter_stride, d.act = z.data_ptr(), rows * K, cabi.ACT_RELU
    d.out, d.ldo = out.data_ptr(), K
    _run(op, 1)                                             # iteration 1: the second slot of z
    first = out.clone()
    args = (dz.cpu().numpy(), w.cpu().numpy(), z[1].cpu().numpy(), cabi.ACT_RELU)
    frac = _frac(out, grad_ref.dgrad(*args), grad_ref.dgrad_bound(*args))
    assert frac <= 1.0, frac
    assert bool((out[z[1] <= 0] == 0).all()) and bool((z[1] == 0).any())
    _run(op, 1)
    assert torch.equal(out, first)
    print(f"[mlp-cg] dgrad relu rows={rows} N={N} K={K}: {frac:.3g} of the bound")


def _handle(ops, n, owners):
    return runtime._make_handle(torch.device(DEV), ops, n)


# (golden net case giving the shape, hidden activation): both heads, every activation
GRAD_CASES = {"mse-relu": ("mse_relu", "ReLU"), "mse-silu": ("tutorial_mse_silu", "SiLU"), "mse-mish": ("mse_relu", "Mish"),
              "cumrew-relu": ("cumrew_relu", "ReLU"), "cumrew-silu": ("cumrew_relu", "SiLU")}


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("batch", [50, 800, 4096])
@pytest.mark.parametrize("case", list(GRAD_CASES))
def test_input_gradient_matches_fp64_autograd(case, batch, math):
    name, act = GRAD_CASES[case]
    kw = mg.NETS[name]
    clf = mlp_cg_ref.make_classifier(name, 31, DEV, act=act)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(batch, kw["x_dim"], generator=g).clamp(-1, 1).to(DEV)
    c = torch.randn(batch, kw["out_dim"], generator=g).to(DEV) if kw["head"] == "mse" else None
    t = torch.tensor([4, 1], device=DEV)
    got, _ = cg_ref.lowered_gradient(clf, x, t, 1, MATHS[math], DEV, cond=c, handle=_handle)
    torch.cuda.synchronize()
    want = mlp_cg_ref.input_gradient_fp64(clf, x, t[1].expand(batch), c)
    rel = float((got.double() - want).norm() / want.norm())
    # fp32: summation order only.  TF32: the 256-wide Linears read 10-bit mantissas (QGPO's classifier, the same stack:
    # 3e-4 to 5e-4); under ReLU a pre-activation within the TF32 error of 0 can change sign and switch its unit's term of the
    # gradient on or off (up to 1.4e-2 on the interpreter).  A wrong column block of W_1, a missing activation derivative or a
    # wrong MSE factor gives rel ~ 1
    print(f"[mlp-cg] input gradient {case} B={batch} {math}: rel {rel:.3g}")
    assert rel < (1e-5 if math == "fp32" else (5e-2 if act == "ReLU" else 1e-2)), rel


class _Wrapped:
    """the same classifier behind a class the lowering does not recognise: the host-callback path"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


def tutorial_agent(device=DEV):
    """the reference tutorial's actor and classifier (kitchen: act 9, obs 60), synthetic weights"""
    from cleandiffuser_b200.classifier import MSEClassifier
    from cleandiffuser_b200.diffusion import DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_classifier import MLPNNClassifier
    from cleandiffuser_b200.nn_diffusion import PearceMlp
    nn_diffusion = load_synth(PearceMlp(9, To=0, emb_dim=64, hidden_dim=256, timestep_emb_type="positional"), seed=41)
    nn_classifier = load_synth(MLPNNClassifier(9, 60, 32, [256], activation=torch.nn.SiLU()), seed=31)
    classifier = MSEClassifier(nn_classifier, temperature=1.0, device=device)
    actor = DiscreteDiffusionSDE(nn_diffusion, classifier=classifier, predict_noise=False, x_max=torch.ones((1, 9)),
                                 x_min=-torch.ones((1, 9)), diffusion_steps=5, ema_rate=0.9999, device=device)
    actor.eval()
    classifier.eval()
    return actor


def tutorial_call(actor, obs, tape, w_cg=0.1):
    with tape.active():
        x0, log = actor.sample(torch.zeros(obs.shape[0], 9, device=obs.device), solver="ddpm", n_samples=obs.shape[0],
                               sample_steps=5, temperature=0.5, w_cg=w_cg, condition_cg=obs)
    torch.cuda.synchronize()
    return x0, log


def _obs(batch, seed=1):
    return torch.randn(batch, 60, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("math", list(MATHS))
def test_tutorial_call_graph_against_callback(math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    actor = tutorial_agent()
    clf = actor.classifier
    obs = _obs(50)
    tape = NoiseTape()
    x_graph, log = tutorial_call(actor, obs, tape)
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    print(f"[mlp-cg] tutorial math={math}: {runtime.STATS['launches']} launches per call")
    actor.classifier = _Wrapped(clf)
    x_cb, log_cb = tutorial_call(actor, obs, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "callback"
    err = float((x_graph - x_cb).abs().max())
    print(f"[mlp-cg] tutorial math={math}: x0 graph vs callback max {err:.3g}")
    # log_p is the classifier's PyTorch logp of x0 after the loop on both paths
    if math == "fp32":
        assert err < 1e-5, err
        torch.testing.assert_close(log["log_p"], log_cb["log_p"], rtol=1e-5, atol=1e-5)
        return
    # TF32: both paths run the same TF32 denoiser program; only the classifier's input gradient differs (TF32 Linears in
    # the graph, fp32 PyTorch in the callback: cuBLAS TF32 is off by default).  x0 depends on the gradients through the
    # guidance term w_cg * sigma^2 / alpha * g of each step, so to first order a gradient with relative error eps moves x0
    # by eps times the guidance's whole effect on x0, D = max |x0(w_cg) - x0(w_cg = 0)|.  eps = 1e-2 is the relative bound
    # test_input_gradient_matches_fp64_autograd holds the TF32 gradient to; twice eps D covers the second-order terms (the
    # denoiser sees the moved x_t of later steps), and 1e-5 the fp32 floor above
    actor.classifier = clf
    x_free, _ = tutorial_call(actor, obs, NoiseTape(tape.draws), w_cg=0.0)
    effect = float((x_cb - x_free).abs().max())
    bound = 2 * 1e-2 * effect + 1e-5
    print(f"[mlp-cg] tutorial tf32: guidance effect on x0 {effect:.3g}, bound {bound:.3g}")
    assert effect > 1e-3, "the guidance does not move x0: the comparison shows nothing"
    assert err < bound, (err, bound)
    torch.testing.assert_close(log["log_p"], log_cb["log_p"], rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_goldens_on_the_gpu(name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "fp32")
    G = load_golden("mlp_classifier")
    agent, prior, kw = mlp_cg_ref.make_sample_agent(name, device=DEV)

    def refuse(*a, **k):
        raise AssertionError("classifier.gradients called: guidance left the program")
    monkeypatch.setattr(agent.classifier, "gradients", refuse)
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = agent.sample(prior, **kw)
    assert runtime.STATS["guidance_path"] == "graph"
    assert np.abs(x0.cpu().numpy() - G[f"sample/{name}/x0"]).max() < 1e-3
    np.testing.assert_allclose(log["log_p"].cpu().numpy(), G[f"sample/{name}/log_p"], rtol=2e-3, atol=2e-3)


def relu_agent():
    """golden sample case "dql_eps": a ContinuousDiffusionSDE over DQLMlp guided by an MSEClassifier over a ReLU
    MLPNNClassifier [256, 256]"""
    agent, _, _ = mlp_cg_ref.make_sample_agent("dql_eps", device=DEV)
    return agent


def relu_call(agent, c, steps, tape):
    with tape.active():
        x0, log = agent.sample(torch.zeros(c.shape[0], 9, device=DEV), "ddpm", n_samples=c.shape[0], sample_steps=steps,
                               sample_step_schedule="uniform_continuous", condition_cfg=c[:, :11], w_cfg=1.0,
                               condition_cg=c, w_cg=0.5)
    torch.cuda.synchronize()
    return x0, log


@pytest.mark.parametrize("math", list(MATHS))
def test_graph_replay_equals_direct_launches_and_repeats_bitwise(math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent = relu_agent()
    c = _obs(800)
    tape = NoiseTape()
    a, la = relu_call(agent, c, 10, tape)
    b, lb = relu_call(agent, c, 10, NoiseTape(tape.draws))
    monkeypatch.setenv("CDS_GRAPH", "0")
    d, _ = relu_call(agent, c, 10, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "graph"
    assert torch.equal(a, b) and torch.equal(a, d) and torch.equal(la["log_p"], lb["log_p"])


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("call", ["tutorial", "relu"])
def test_every_operator_of_the_guided_iteration_matches_fp64(call, math, monkeypatch):
    """tests/program_audit.py over every iteration of the guided call: each operator within its bound, nothing written outside
    its declared outputs; then whole iterations by graph replay give the operator-by-operator bits"""
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    if call == "tutorial":
        agent = tutorial_agent()
        tutorial_call(agent, _obs(50), NoiseTape())
    else:
        agent = relu_agent()
        relu_call(agent, _obs(800), 5, NoiseTape())
    assert len(agent._engine_plans) == 1
    plan = next(iter(agent._engine_plans.values()))
    ops, n, st = plan.program.ops, plan.n_iters, _stream()
    assert cabi.OP_GUIDE in {op.kind for op in ops}
    torch.cuda.synchronize()
    start = torch.rand(plan.x.shape, generator=torch.Generator().manual_seed(7)).to(DEV) * 2 - 1
    plan.x.copy_(start)
    aud = pa.Auditor(f"mlp-{call}-{math}", ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    aud.audit_once(0)
    for it in range(n):
        aud.audit_iteration(it)
    for line in pa.report_lines({(aud.name, k): v for k, v in aud.worst.items()}):
        print("[mlp-cg audit]", line)
    assert not aud.failures, "\n".join(aud.failures[:20])
    act = "silu" if call == "tutorial" else "relu"
    assert {f"dgrad {act}", f"stash {act} (no slot)"} <= set(aud.worst)
    assert plan.handle.launches_per_iter() == pa.launches_per_iter(ops)

    mem = emulator.Owned(pa.plan_owners(plan))
    written = [mem.owners[i] for i in pa.written_owners(mem, ops, range(n))]
    outs = {}
    for mode in ("op by op", "graph"):
        plan.x.copy_(start)
        torch.cuda.synchronize()
        if mode == "op by op":
            pa.run_op_by_op(plan.handle, ops, 0, n, st, torch.cuda.synchronize)
        else:
            plan.handle.run(0, n, st, True)
        torch.cuda.synchronize()
        outs[mode] = [t.clone() for t in written]
    assert all(pa.same_bits(a, b) for a, b in zip(outs["op by op"], outs["graph"]))
