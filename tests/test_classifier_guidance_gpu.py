"""Classifier guidance inside the replayed loop on the H100: CDS_OP_GN / CDS_OP_GN_BWD / CDS_OP_GUIDE against fp64
(tests/cg_ref.py), HalfJannerUNet1d's lowered input gradient against fp64 autograd at the reference pipelines' classifier
shapes, whole guided sample() calls against the host-callback path and the goldens, and graph replay / reproducibility."""

import numpy as np
import pytest
import torch

import cg_ref
import make_golden_classifier as mg
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape, load_synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MATHS = {"fp32": cabi.MATH_FP32, "tf32": cabi.MATH_TF32_TC}


def _run(op):
    cabi.run_op(0, op, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def _bound(want, dtype, rel=2e-6):
    """fp32 arithmetic error (rel of the largest magnitude) plus, for a TF32 store, half a TF32 ulp of each element"""
    b = rel * want.abs().max() + 1e-7
    return b + (want.abs() * 2.0 ** -11 if dtype == cabi.TF32 else 0)


# (C, L) combinations of the pipelines' classifiers: 4-channel groups at C = 32, L = 1 at the halfcheetah mid blocks
SHAPES = [(32, 64), (32, 4), (64, 32), (64, 8), (128, 2), (128, 16), (256, 1), (256, 4)]
BATCH = 333                      # not a multiple of the 8 (trajectory, group) warps of a CTA


@pytest.mark.parametrize("dtype", [cabi.F32, cabi.TF32])
@pytest.mark.parametrize("C,L", SHAPES)
def test_gn_and_gn_bwd_match_fp64(C, L, dtype):
    g = torch.Generator(device="cpu").manual_seed(C * 100 + L)
    groups = min(8, C // 4)
    h, res, dout = (torch.randn(BATCH, L, C, generator=g).to(DEV) * s for s in (2.0, 1.0, 1.0))
    h = h + 0.5
    gamma, beta = (1 + 0.1 * torch.randn(C, generator=g)).to(DEV), (0.1 * torch.randn(C, generator=g)).to(DEV)
    step = torch.randn(3, C, generator=g).to(DEV)
    out, dh = torch.zeros(BATCH, L, C, device=DEV), torch.zeros(BATCH, L, C, device=DEV)
    op = cabi.Op()
    op.kind = cabi.OP_GN
    q = op.u.gn
    q.batch, q.L, q.C, q.groups, q.eps, q.act = BATCH, L, C, groups, 1e-5, cabi.ACT_MISH
    q.h, q.h_bstride, q.h_lstride, q.gamma, q.beta = h.data_ptr(), L * C, C, gamma.data_ptr(), beta.data_ptr()
    q.vec.step, q.vec.step_stride = step.data_ptr(), C            # iteration 0's row
    q.res, q.res_bstride, q.res_lstride = res.data_ptr(), L * C, C
    q.out, q.out_bstride, q.out_lstride, q.out_dtype = out.data_ptr(), L * C, C, dtype
    _run(op)
    want = cg_ref.gn(h, gamma, beta, groups, 1e-5, cabi.ACT_MISH, step[0], res)
    assert ((out.double() - want).abs() <= _bound(want, dtype)).all(), float((out.double() - want).abs().max())
    assert dtype != cabi.TF32 or torch.equal(out, cg_ref.opref.tf32_round(out))

    op = cabi.Op()
    op.kind = cabi.OP_GN_BWD
    q = op.u.gn_bwd
    q.batch, q.L, q.C, q.groups, q.eps, q.act = BATCH, L, C, groups, 1e-5, cabi.ACT_MISH
    q.h, q.h_bstride, q.h_lstride, q.gamma, q.beta = h.data_ptr(), L * C, C, gamma.data_ptr(), beta.data_ptr()
    q.dout, q.dout_bstride, q.dout_lstride = dout.data_ptr(), L * C, C
    q.dh, q.dh_bstride, q.dh_lstride, q.dh_dtype = dh.data_ptr(), L * C, C, dtype
    _run(op)
    want = cg_ref.gn_bwd(h, gamma, beta, dout, groups, 1e-5)
    # dh is a difference of group means: its error is relative to rstd * |dxhat|, not to dh itself
    assert ((dh.double() - want).abs() <= _bound(want, dtype, rel=2e-5)).all(), float((dh.double() - want).abs().max())


@pytest.mark.parametrize("C,pad", [(14, 16), (23, 23), (37, 48)])
def test_guide_is_the_reference_expression_bit_for_bit(C, pad):
    g_ = torch.Generator(device="cpu").manual_seed(C)
    L = 32
    pred = torch.randn(BATCH, L, C, generator=g_).to(DEV)
    grad = torch.randn(BATCH, L, pad, generator=g_).to(DEV)
    sig = torch.rand(4, generator=g_).to(DEV)
    scale = -(0.3 * sig)
    want = pred - 0.3 * sig[2] * grad[..., :C]                        # sde.py::classifier_guidance, eps-prediction
    op = cabi.Op()
    op.kind = cabi.OP_GUIDE
    q = op.u.guide
    q.batch, q.L, q.C, q.pred, q.g, q.g_bstride, q.g_lstride, q.s = BATCH, L, C, pred.data_ptr(), grad.data_ptr(), L * pad, pad, \
        scale.data_ptr()
    cabi.run_op(0, op, 2, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(pred, want)


# the classifiers of the reference's guided pipelines (diffuser / adaptdiffuser / veteran on D4RL)
PIPELINES = {"hopper": dict(horizon=32, in_dim=14), "walker": dict(horizon=32, in_dim=23),
             "halfcheetah": dict(horizon=4, in_dim=23, dim_mult=(1, 4, 2)), "antmaze": dict(horizon=64, in_dim=37),
             "kitchen": dict(horizon=32, in_dim=69)}


def _handle(ops, n, owners):
    return runtime._make_handle(torch.device(DEV), ops, n)


@pytest.mark.parametrize("math", list(MATHS))
@pytest.mark.parametrize("name", list(PIPELINES))
def test_input_gradient_matches_fp64_autograd(name, math):
    kw = PIPELINES[name]
    clf = cg_ref.make_classifier(kw, 31, DEV)
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(3200, kw["horizon"], kw["in_dim"], generator=g).to(DEV)
    t = torch.tensor([17, 3], device=DEV)
    got, _ = cg_ref.lowered_gradient(clf, x, t, 1, MATHS[math], DEV, handle=_handle)
    torch.cuda.synchronize()
    want = cg_ref.input_gradient_fp64(clf, x, t[1].expand(3200))
    rel = float((got.double() - want).norm() / want.norm())
    # fp32: summation order only.  TF32: the convolutions read 10-bit mantissas; measured 1.7e-3 on the CPU interpreter.  A
    # wrong tap order or phase packing gives rel ~ 1.
    assert rel < (1e-5 if math == "fp32" else 1e-2), rel


def _hopper_agent(clf):
    from cleandiffuser_b200.diffusion import DiscreteDiffusionSDE
    from cleandiffuser_b200.nn_diffusion import JannerUNet1d
    net = load_synth(JannerUNet1d(14, model_dim=32, emb_dim=32, kernel_size=5, dim_mult=[1, 2, 2, 2]), seed=0)
    mask = torch.zeros(32, 14)
    mask[0, :11] = 1.
    return DiscreteDiffusionSDE(net, None, fix_mask=mask, predict_noise=True, diffusion_steps=20, device=DEV, classifier=clf)


class _Wrapped:
    """the same classifier behind a class the lowering does not recognise: the host-callback path"""

    def __init__(self, clf):
        self.clf = clf

    def logp(self, x, noise, c=None):
        return self.clf.logp(x, noise, c)

    def gradients(self, x, noise, c=None):
        return self.clf.gradients(x, noise, c)


def _hopper_call(agent, prior, tape):
    with tape.active():
        x0, log = agent.sample(prior, solver="ddpm", n_samples=prior.shape[0], sample_steps=20, use_ema=True, temperature=0.5,
                               w_cg=0.3)
    torch.cuda.synchronize()
    return x0, log


@pytest.mark.parametrize("math", list(MATHS))
def test_diffuser_hopper_call_graph_against_callback(math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    # the callback's classifier is PyTorch: cuDNN convolutions would read TF32 by default, the fp32 comparison wants fp32
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", math == "tf32")
    clf = cg_ref.make_classifier(PIPELINES["hopper"], 31, DEV)
    agent = _hopper_agent(clf)
    g = torch.Generator(device="cpu").manual_seed(1)
    prior = torch.zeros(3200, 32, 14)
    prior[:, 0, :11] = torch.randn(3200, 11, generator=g)
    prior = prior.to(DEV)
    tape = NoiseTape()
    x_graph, log = _hopper_call(agent, prior, tape)
    assert runtime.STATS["guidance_path"] == "graph"
    print(f"[cg] hopper B=3200 math={math}: {runtime.STATS['launches']} launches per call")
    agent.classifier = _Wrapped(clf)
    x_cb, log_cb = _hopper_call(agent, prior, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "callback"
    err = (x_graph - x_cb).abs()
    if math == "fp32":
        assert err.max() < 1e-3, float(err.max())
        # log_p is the classifier's PyTorch logp of x0 after the loop on both paths
        torch.testing.assert_close(log["log_p"], log_cb["log_p"], rtol=2e-3, atol=2e-3)
    else:
        # two TF32 classifiers (the engine's, cuDNN's) whose gradient roundings differ, through 20 steps of a synthetic-weight
        # denoiser: measured 0.082 max / 0.0076 mean on an H100; a wrong gradient moves x0 by O(1)
        assert err.max() < 0.15 and err.mean() < 1e-2, (float(err.max()), float(err.mean()))


@pytest.mark.parametrize("name", list(mg.SAMPLES))
def test_goldens_on_the_gpu(name, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", "fp32")
    G = cg_ref.golden()
    agent, prior, kw = cg_ref.make_sample_agent(name, device=DEV)
    tape = NoiseTape(cg_ref.tape_of(G, name))
    with tape.active():
        x0, log = agent.sample(prior, **kw)
    assert runtime.STATS["guidance_path"] == "graph"
    assert np.abs(x0.cpu().numpy() - G[f"sample/{name}/x0"]).max() < 1e-3
    np.testing.assert_allclose(log["log_p"].cpu().numpy(), G[f"sample/{name}/log_p"], rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("math", list(MATHS))
def test_graph_replay_equals_direct_launches_and_repeats_bitwise(math, monkeypatch):
    monkeypatch.setenv("CDS_BACKEND", "cuda")
    monkeypatch.setenv("CDS_MATH", math)
    agent = _hopper_agent(cg_ref.make_classifier(PIPELINES["hopper"], 31, DEV))
    prior = torch.zeros(512, 32, 14, device=DEV)
    tape = NoiseTape()
    a, _ = _hopper_call(agent, prior, tape)
    b, _ = _hopper_call(agent, prior, NoiseTape(tape.draws))
    monkeypatch.setenv("CDS_GRAPH", "0")
    c, _ = _hopper_call(agent, prior, NoiseTape(tape.draws))
    assert runtime.STATS["guidance_path"] == "graph"
    assert torch.equal(a, b) and torch.equal(a, c)
