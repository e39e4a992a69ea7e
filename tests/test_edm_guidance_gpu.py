"""Classifier guidance in ContinuousEDM and the legacy DDPM class on the H100: the four lowered classifier families (CumRew over
HalfJannerUNet1d and over HalfDiT1d, MSE over MLPNNClassifier, QGPO) x {EDM Euler, EDM Heun, legacy eps, legacy x0} in fp32
and TF32 inside the replayed program against this package's PyTorch loop on the CPU with the same noise tape, the host
callback with ToyClassifier, and an operator audit of a guided EDM iteration (the update with its guidance operand bit for bit
against the interpreter, every other operator against fp64)."""
import numpy as np
import pytest
import torch

import edm_guide_ref
import make_golden_edm_guided as mg
import program_audit as pa
from common import load_golden, tape_of
from test_edm_guidance_cpu import CLS
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape, ToyClassifier, synth_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
G = load_golden("edm_guided")
PAIR = {"half_janner": "janner", "half_dit": "janner", "mlp": "mlp", "qgpo": "mlp"}
SAMPLERS = {"edm_euler": {"janner": "edm_euler_janner", "mlp": "edm_euler_mlp"},
            "edm_heun": {"janner": "edm_heun_janner", "mlp": "edm_heun_mlp"},
            "ddpm_eps": {"janner": "ddpm_sample_eps_janner", "mlp": "ddpm_sample_x_eps_mlp"},
            "ddpm_x0": {"janner": "ddpm_sample_x_x0_janner", "mlp": "ddpm_sample_x0_mlp"}}
# |engine - PyTorch loop| <= TOL (|loop| + 1).  fp32: summation order through every step.  TF32: the denoiser's and the
# classifier's GEMMs read 10-bit mantissas, and the classifier's gradient enters every step scaled by w sigma^2 (up to 80^2 w at
# the first EDM step), so the bound only catches a non-finite or grossly wrong result, as tests/guidance_space.py's TF32 bound does
TOL = {"fp32": 2e-3, "tf32": 0.25}


@pytest.fixture(autouse=True)
def engine(monkeypatch):
    edm_guide_ref.register(monkeypatch)
    monkeypatch.setenv("CDS_BACKEND", "cuda")


def classifier(family, device):
    if family in ("half_janner", "mlp"):
        return mg.make_classifier(PAIR[family], CLS, device)
    if family == "half_dit":
        from cleandiffuser_b200.classifier import CumRewClassifier
        from cleandiffuser_b200.nn_classifier import HalfDiT1d
        net = HalfDiT1d(mg.D, 1, 16, d_model=64, n_heads=2, depth=2)
        net.load_state_dict(synth_state_dict(net.state_dict(), 33))
        return CumRewClassifier(net, device=device)
    from cleandiffuser_b200.classifier import QGPOClassifier
    from cleandiffuser_b200.nn_classifier import QGPONNClassifier
    net = QGPONNClassifier(mg.OBS, mg.A, 64, [256, 256], "untrainable_fourier")
    net.load_state_dict(synth_state_dict(net.state_dict(), 33))
    return QGPOClassifier(net, device=device)


def run(name, clf, device, **over):
    agent = mg.make_agent(name, CLS, classifier=clf, device=device)
    prior, c = (torch.from_numpy(G[f"sample/{name}/{k}"]).to(device) for k in ("prior", "c"))
    fn, kw = mg.sample_call(name, agent, prior, c)
    kw.update(over)
    tape = NoiseTape(tape_of(G, f"sample/{name}"))
    with tape.active():
        x0, log = fn(prior.clone(), **kw)
    return agent, x0, log


def _close(got, want, tol):
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    assert torch.isfinite(got).all()
    err = ((got - want).abs() / (want.abs() + 1)).max()
    assert err <= tol, float(err)


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("sampler", list(SAMPLERS))
@pytest.mark.parametrize("family", list(PAIR))
def test_graph_path_matches_pytorch_loop(family, sampler, math, monkeypatch):
    monkeypatch.setenv("CDS_MATH", math)
    name = SAMPLERS[sampler][PAIR[family]]
    _, got, log = run(name, classifier(family, DEV), DEV)
    assert runtime.STATS["guidance_path"] == "graph", runtime.STATS["guidance_reason"]
    _, want, want_log = run(name, classifier(family, "cpu"), "cpu")
    _close(got, want, TOL[math])
    _close(log["log_p"], want_log["log_p"], TOL[math])


@pytest.mark.parametrize("sampler", list(SAMPLERS))
def test_callback_path_with_toy_classifier(sampler, monkeypatch):
    monkeypatch.setenv("CDS_MATH", "fp32")
    name = SAMPLERS[sampler]["janner"]
    _, got, log = run(name, ToyClassifier((mg.H, mg.D), device=DEV), DEV)
    assert runtime.STATS["guidance_path"] == "callback" and "ToyClassifier" in runtime.STATS["guidance_reason"]
    _, want, want_log = run(name, ToyClassifier((mg.H, mg.D)), "cpu")
    _close(got, want, TOL["fp32"])
    _close(log["log_p"], want_log["log_p"], TOL["fp32"])


@pytest.mark.parametrize("math", ["fp32", "tf32"])
@pytest.mark.parametrize("name", ["edm_heun_janner", "edm_euler_mlp"])
def test_guided_edm_iteration_audit(name, math, monkeypatch):
    """every operator of one guided EDM iteration: PREP, the denoiser, the classifier's input gradient and the update with its
    guidance operand (bit for bit against the interpreter), writes outside the outputs included"""
    monkeypatch.setenv("CDS_MATH", math)
    agent, _, _ = run(name, None, DEV)
    assert runtime.STATS["guidance_path"] == "graph"
    (plan,) = agent._engine_plans.values()
    ops = plan.program.ops
    assert ops[-1].kind == cabi.OP_UPDATE and ops[-1].u.update.guide
    torch.cuda.synchronize()
    st = torch.cuda.current_stream().cuda_stream
    aud = pa.Auditor(f"{name}-{math} guided", ops, plan.handle, pa.plan_owners(plan), st, torch.cuda.synchronize)
    plan.x.copy_(torch.randn(plan.x.shape, generator=torch.Generator().manual_seed(7)).to(DEV).clamp(-1, 1))
    for it in range(plan.n_iters):                       # every evaluation: Euler / Heun predictor and corrector rows
        aud.audit_iteration(it)
    assert not aud.failures, "\n".join(aud.failures[:20])
    assert "update + guide" in aud.worst


def test_guided_edm_update_kernel_bitwise():
    """the update's guidance operand alone: kinds EDM and EDM_HEUN, with and without the clip, against the interpreter's
    fp32 restatement bit for bit (the scalar path: the float4 path is never taken with the operand)"""
    import emulator
    from cleandiffuser_b200.diffusion import solvers as S
    g = torch.Generator().manual_seed(3)
    B, R = 37, 24
    for kind in (S.UPD_EDM, S.UPD_EDM_HEUN):
        for clip in (0, 1):
            t = {k: torch.randn(B, R, generator=g) for k in ("x", "pred", "guide", "hist", "aux", "prior")}
            coef = torch.zeros(2, cabi.ROW_FLOATS)
            coef[1, S.R_K0], coef[1, S.R_K1], coef[1, S.R_K2], coef[1, S.R_SIGMA] = 0.3, 0.7, 0.05, 1.7
            coef[1, S.R_KIND], coef[1, S.R_K4] = float(kind), 1.0 if kind == S.UPD_EDM else 0.0
            scale = torch.tensor([0.0, 2.5])
            mask, xmin, xmax = (torch.rand(R, generator=g) > 0.7).float(), -torch.rand(R, generator=g), torch.rand(R, generator=g)
            outs = []
            for dev in ("cpu", DEV):
                d = {k: v.clone().to(dev) for k, v in {**t, "coef": coef, "scale": scale, "mask": mask, "xmin": xmin,
                                                       "xmax": xmax}.items()}
                op = cabi.Op()
                op.kind = cabi.OP_UPDATE
                u = op.u.update
                u.batch, u.row, u.x, u.pred, u.coef = B, R, d["x"].data_ptr(), d["pred"].data_ptr(), d["coef"].data_ptr()
                u.prior, u.mask = d["prior"].data_ptr(), d["mask"].data_ptr()
                u.xhat_prev, u.aux = d["hist"].data_ptr(), d["aux"].data_ptr()
                u.final_clip = clip
                if clip:
                    u.x_min, u.x_max = d["xmin"].data_ptr(), d["xmax"].data_ptr()
                u.guide, u.guide_s = d["guide"].data_ptr(), d["scale"].data_ptr()
                if dev == "cpu":
                    emulator.OPS[cabi.OP_UPDATE][1](u, 1)
                else:
                    cabi.run_op(0, op, 1, torch.cuda.current_stream().cuda_stream)
                    torch.cuda.synchronize()
                outs.append({k: d[k].cpu() for k in ("x", "hist", "aux")})
            for k in outs[0]:
                assert pa.same_bits(outs[0][k], outs[1][k]), (kind, clip, k)
            np.testing.assert_array_equal(outs[0]["x"].numpy(), outs[1]["x"].numpy())
