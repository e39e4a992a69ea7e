"""Operator-level parity of the elementwise operators (csrc/elementwise.cuh).

UPDATE, PREP and CAST promise fp32 results identical to the operation-by-operation fp32 mirror in tests/emulator.py, so
they are compared bit for bit: every descriptor is built from one dict of buffers twice, over CPU tensors for the emulator
and over their GPU copies for ``cds_run_op``, and every buffer (NaN guards included) must come out with the same bits.
LNMOD is compared with tests/opref.py's fp64 LayerNorm under the bound of tests/test_linear_ln_gpu.py."""
import pytest
import torch

import emulator
import opref
from cleandiffuser_b200.engine import cabi

DEV = "cuda:0"
GUARD = 64                      # NaN floats after every written buffer
ITER = 3
DDPM, DDIM, EPS, X, X2M, CM, EDM, HEUN = range(8)
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    WORST.clear()
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print()
        for path, (frac, name) in sorted(WORST.items()):
            print(f"[lnmod] {path}: largest error = {frac:.3f} of the bound ({name})")


def _ptr(d, name):
    """device address of operand ``name``: its buffer plus the case's element offset ("name@" entry)"""
    if name not in d:
        return 0
    t = d[name]
    return t.data_ptr() + t.element_size() * d.get(name + "@", 0)


def _same_bits(a, b):
    """bitwise equality, with every NaN equal to every NaN"""
    ib = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    na, nb = torch.isnan(a.float()), torch.isnan(b.float())
    return bool(torch.equal(na, nb) and torch.equal(a.view(ib)[~na], b.view(ib)[~nb]))


def _to(d, device):
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _compare(cpu, gpu, names):
    for n in names:
        if n in cpu:
            assert _same_bits(cpu[n], gpu[n].cpu()), f"{n} differs from the emulator"


# ============================================================================================================ UPDATE
def _coef(rows, kind, slot, xw=0.0, k4=None):
    """[rows][CDS_ROW_FLOATS] table with distinct rows; row ITER has the case's kind and noise slot"""
    t = torch.zeros(rows, cabi.ROW_FLOATS)
    for i in range(rows):
        t[i, 0] = 0.9 - 0.05 * i                  # alpha
        t[i, 1] = 0.4 + 0.07 * i                  # sigma
        t[i, 2:7] = torch.tensor([1.01, 0.37, 0.11, 0.83, 0.29]) + 0.013 * i
        t[i, 7] = (kind + i) % 8
        t[i, 9] = 10 - i
    t[ITER, 7] = kind
    t[ITER, 8] = slot + 1 if slot is not None else 0
    if k4 is not None:
        t[ITER, 6] = k4
    if xw:
        t[ITER, 10], t[ITER, 11] = xw, 0.71
    return t


def U(name, kind, path, *, pn=0, clip=None, mask=False, cfg=False, noise=None, hist=False, aux=False, cast=None, xw=0.0,
      k4=None, final_clip=0):
    return dict(name=name, kind=kind, path=path, pn=pn, clip=clip, mask=mask, cfg=cfg, noise=noise, hist=hist, aux=aux,
                cast=cast, xw=xw, k4=k4, final_clip=final_clip)


CAST_GEO = {"bf16": (14, 32, cabi.BF16), "tf32": (14, 16, cabi.TF32), "f32": (3, 4, cabi.F32)}
UPDATE_CASES = [
    # kinds on both paths ("vec": float4 path; "row": row % 4 != 0, "xoff": x one float off 16-byte alignment -- scalar).
    # x2m_vec / heun_vec run those kinds without their history buffers, which the kernel then reads as 0: the float4 path
    # cannot take a history buffer, and the lowering never emits these two, so they pin the kernel's behaviour only.
    *[U(f"{k}_{p}", kind, p) for kind, k in enumerate(("ddpm", "ddim", "eps", "x", "x2m", "cm", "edm", "heun"))
      for p in ("vec", "row")],
    U("ddpm_noise_vec", DDPM, "vec", noise="slot"), U("ddpm_noise_row", DDPM, "row", noise="slot"),
    U("ddpm_noise_xoff", DDPM, "xoff", noise="slot"),
    U("ddpm_branch_noise_vec", DDPM, "vec", noise="branch"), U("ddpm_branch_noise_row", DDPM, "row", noise="branch"),
    U("eps_noise_vec", EPS, "vec", noise="slot", pn=1), U("x_noise_row", X, "row", noise="branch"),
    U("ddim_pn_vec", DDIM, "vec", pn=1), U("ddim_pn_row", DDIM, "row", pn=1),
    U("eps_pn_xoff", EPS, "xoff", pn=1),
    # clipping: eps-prediction (to (x - alpha x_max) / sigma ...) and x0-prediction, to x_min, to x_max, to both
    *[U(f"{k}_clip{c}_pn{pn}_{p}", kind, p, pn=pn, clip=c) for (k, kind) in (("ddpm", DDPM), ("x", X))
      for c in ("min", "max", "both") for pn in (0, 1) for p in (("vec", "row") if c == "both" else ("vec",))],
    U("cm_clip_vec", CM, "vec", clip="both", final_clip=1), U("cm_clipmin_row", CM, "row", clip="min", final_clip=1),
    U("cm_clip_off_vec", CM, "vec", clip="both"),
    U("edm_clip_vec", EDM, "vec", clip="both", final_clip=1), U("edm_clipmax_row", EDM, "row", clip="max", final_clip=1),
    # mask (values 0, 1 and 0.3 across the row) and prior
    U("ddpm_mask_vec", DDPM, "vec", mask=True, noise="slot"), U("ddpm_mask_row", DDPM, "row", mask=True),
    U("x_mask_xoff", X, "xoff", mask=True, clip="both"), U("cm_mask_vec", CM, "vec", mask=True),
    U("edm_mask_row", EDM, "row", mask=True), U("heun_mask", HEUN, "vec", mask=True, hist=True, aux=True),
    # CFG (always the scalar path)
    U("ddpm_cfg", DDPM, "vec", cfg=True, noise="slot", mask=True), U("eps_cfg_pn", EPS, "row", cfg=True, pn=1, clip="both"),
    U("cm_cfg", CM, "vec", cfg=True, clip="both", final_clip=1),
    # history: the X2M solver, the EDM predictor (K4 != 0 writes xhat_prev and aux) and the Heun corrector
    U("x2m_hist", X2M, "vec", hist=True), U("x2m_hist_pn_clip", X2M, "row", hist=True, pn=1, clip="both"),
    U("eps_hist", EPS, "vec", hist=True), U("x_hist_cfg", X, "vec", hist=True, cfg=True),
    U("ddpm_hist_unused", DDPM, "vec", hist=True, noise="slot"),
    U("edm_predictor", EDM, "vec", hist=True, aux=True, k4=1.0), U("edm_predictor_xw", EDM, "row", hist=True, aux=True,
                                                                   k4=1.0, xw=1.3),
    # K4 == 0 with both history buffers present: a plain Euler step, which must leave xhat_prev and aux untouched
    U("edm_no_predictor", EDM, "vec", hist=True, aux=True, k4=0.0), U("heun", HEUN, "vec", hist=True, aux=True),
    U("heun_clip", HEUN, "row", hist=True, aux=True, clip="both", final_clip=1),
    U("edm_xw_vec", EDM, "vec", xw=1.3), U("heun_xw", HEUN, "vec", hist=True, aux=True, xw=1.3),
    # the channel-padded copy of x for the tensor-core UNets: bf16 14 -> 32, TF32 14 -> 16, fp32 3 -> 4
    *[U(f"{k}_cast_{ct}_{p}", kind, p, cast=ct) for ct in ("bf16", "tf32", "f32")
      for (k, kind, p) in (("ddpm", DDPM, "vec"), ("x", X, "row"))],
    U("ddpm_cast_bf16_noise_mask", DDPM, "vec", cast="bf16", noise="slot", mask=True),
    U("edm_cast_tf32_cfg", EDM, "vec", cast="tf32", cfg=True), U("x2m_cast_f32_hist", X2M, "xoff", cast="f32", hist=True),
]
UPDATE_CASES = {c["name"]: c for c in UPDATE_CASES}


def _update_setup(c, B=37):
    """buffers (CPU) and the descriptor builder of update case c"""
    g = torch.Generator().manual_seed(sum(map(ord, c["name"])))
    row = {"vec": 56, "row": 42, "xoff": 56}[c["path"]]
    if c["cast"] == "f32":
        row = 60 if c["path"] != "row" else 63
    n = B * row
    rnd = lambda *s: torch.randn(*s, generator=g)
    d = {"x": torch.cat([torch.full((1,), float("nan")), rnd(n), torch.full((GUARD,), float("nan"))]),
         "pred": rnd(n), "coef": _coef(5, c["kind"], 1 if c["noise"] else None, c["xw"], c["k4"])}
    d["x@"] = 1 if c["path"] == "xoff" else 0
    if c["path"] != "xoff":
        d["x"] = torch.cat([d["x"][1:], torch.full((1,), float("nan"))])
    stride = 0
    if c["noise"] == "slot":
        d["noise"] = rnd(3 * n)
    elif c["noise"] == "branch":                  # a sub-batch of a 2.5x larger tape: slots of stride > batch * row
        stride = n * 5 // 2
        d["noise"], d["noise@"] = rnd(3 * stride), row * (B // 2)
    if c["cfg"]:
        d["pred_uncond"] = rnd(n)
    if c["mask"]:
        d["prior"] = rnd(n)
        d["mask"] = torch.tensor([0.0, 1.0, 0.3]).repeat(row // 3 + 1)[:row].contiguous()
    if c["clip"] in ("min", "both"):
        d["x_min"] = -0.6 - 0.2 * torch.rand(row, generator=g)
    if c["clip"] in ("max", "both"):
        d["x_max"] = 0.6 + 0.2 * torch.rand(row, generator=g)
    if c["hist"]:
        d["xhat_prev"] = torch.cat([rnd(n), torch.full((GUARD,), float("nan"))])
    if c["aux"]:
        d["aux"] = torch.cat([rnd(n), torch.full((GUARD,), float("nan"))])
    if c["cast"]:
        ci, co, dt = CAST_GEO[c["cast"]]
        d["x_cast"] = torch.full((n // ci * co + GUARD,), float("nan"), dtype=torch.bfloat16 if dt == cabi.BF16 else torch.float32)

    def op_of(dd):
        op = cabi.Op()
        op.kind = cabi.OP_UPDATE
        u = op.u.update
        u.batch, u.row = B, row
        u.x, u.pred, u.pred_uncond = _ptr(dd, "x"), _ptr(dd, "pred"), _ptr(dd, "pred_uncond")
        u.w_cfg, u.w_uncond = 1.7, -0.7
        u.noise, u.noise_slot_stride = _ptr(dd, "noise"), stride
        u.prior, u.mask, u.x_min, u.x_max = _ptr(dd, "prior"), _ptr(dd, "mask"), _ptr(dd, "x_min"), _ptr(dd, "x_max")
        u.xhat_prev, u.aux, u.coef = _ptr(dd, "xhat_prev"), _ptr(dd, "aux"), _ptr(dd, "coef")
        u.predict_noise, u.final_clip = c["pn"], c["final_clip"]
        if c["cast"]:
            u.x_cast, (u.cast_C_in, u.cast_C_out, u.x_cast_dtype) = _ptr(dd, "x_cast"), CAST_GEO[c["cast"]]
        return op
    return d, op_of


def _update_path(u):
    """the branch solver_update_kernel takes at ITER (noise slot 1): "vec" (float4) or "scalar" (mirrors its vec4
    condition)"""
    noise = u.noise + 4 * (u.noise_slot_stride or u.batch * u.row) if u.noise else 0
    aligned = all(p % 16 == 0 for p in (u.x, u.pred, u.prior or 0, noise))
    return "vec" if (u.row % 4 == 0 and not u.pred_uncond and not u.xhat_prev and aligned) else "scalar"


def test_update_cases_cover_every_kind_on_both_paths_and_every_operand():
    seen = set()
    for c in UPDATE_CASES.values():
        d, op_of = _update_setup(c)
        u = op_of(d).u.update
        path = _update_path(u)
        seen.add((c["kind"], path))
        for f in ("noise", "pred_uncond", "prior", "x_min", "x_max", "xhat_prev", "aux", "x_cast"):
            if getattr(u, f):
                seen.add((f, path))
        if u.noise_slot_stride:
            seen.add(("noise_slot_stride", path))
    assert {(k, p) for k in range(8) for p in ("vec", "scalar")} <= seen
    assert {(f, p) for f in ("noise", "noise_slot_stride", "prior", "x_min", "x_max", "x_cast") for p in ("vec", "scalar")} <= seen
    assert {("pred_uncond", "scalar"), ("xhat_prev", "scalar"), ("aux", "scalar")} <= seen


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(UPDATE_CASES))
def test_update_is_bit_exact(name):
    c = UPDATE_CASES[name]
    cpu, op_of = _update_setup(c)
    gpu = _to(cpu, DEV)
    emulator.run_update(op_of(cpu).u.update, ITER)
    cabi.run_op(0, op_of(gpu), ITER, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _compare(cpu, gpu, ("x", "xhat_prev", "aux", "x_cast"))
    if c["cast"]:
        ci, co, _ = CAST_GEO[c["cast"]]
        pads = gpu["x_cast"][:-GUARD].view(-1, co)[:, ci:]
        assert torch.isnan(pads.float()).all(), "a pad channel of x_cast was written"


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [True, False])
def test_update_plan_five_iterations(use_graph):
    """one-operator plan: the update advances the iteration counter from its last block; every block of the 8 x SM grid
    runs several grid-stride steps"""
    B, row = 2200, 1024
    sms = cabi.load().cds_device_sm_count(0)
    assert B * row // 4 >= 2 * 8 * sms * 256
    g = torch.Generator().manual_seed(5)
    n = B * row
    coef = _coef(5, DDPM, 0)
    coef[:, 7] = torch.tensor([DDPM, EPS, X, DDIM, DDPM], dtype=torch.float32)
    coef[:, 8] = torch.tensor([1, 2, 0, 0, 3], dtype=torch.float32)
    cpu = {"x": torch.randn(n, generator=g), "pred": torch.randn(n, generator=g), "noise": torch.randn(3 * n, generator=g),
           "x_min": -torch.ones(row), "x_max": torch.ones(row), "coef": coef}
    gpu = _to(cpu, DEV)

    def op_of(dd):
        op = cabi.Op()
        op.kind = cabi.OP_UPDATE
        u = op.u.update
        u.batch, u.row, u.x, u.pred, u.noise, u.coef = B, row, _ptr(dd, "x"), _ptr(dd, "pred"), _ptr(dd, "noise"), _ptr(dd, "coef")
        u.x_min, u.x_max = _ptr(dd, "x_min"), _ptr(dd, "x_max")
        return op
    emulator.run_program([op_of(cpu)], 5, 0)
    plan = cabi.Plan(0)
    plan.append([op_of(gpu)])
    plan.finalize(5)
    assert plan.launches_per_iter() == 1                 # the counter advance is fused into the update
    plan.run(0, 5, torch.cuda.current_stream().cuda_stream, use_graph=use_graph)
    torch.cuda.synchronize()
    plan.close()
    _compare(cpu, gpu, ("x",))


@pytest.mark.gpu
def test_update_with_64bit_indices():
    """batch * row >= 2^31 takes the scalar path with 64-bit index arithmetic; compared on row-aligned slices at the start,
    across element 2^31 and at the end"""
    row = 257
    B = (1 << 31) // row + 3
    n = B * row
    need = 2 * 4 * n
    free = torch.cuda.mem_get_info(0)[0]
    if free < 20 * 2 ** 30:
        pytest.skip(f"needs 20 GB of free device memory for {need / 2 ** 30:.1f} GB of buffers, {free / 2 ** 30:.1f} GB free")
    g = torch.Generator(device=DEV).manual_seed(64)
    x = torch.randn(n, generator=g, device=DEV)
    pred = torch.randn(n, generator=g, device=DEV)
    gc = torch.Generator().manual_seed(64)
    small = {"x_min": -0.5 - torch.rand(row, generator=gc), "x_max": 0.5 + torch.rand(row, generator=gc),
             "coef": _coef(5, EPS, None)}
    small_gpu = _to(small, DEV)
    edge = (1 << 31) // row
    slices = [(0, 4), (edge - 2, edge + 3), (B - 4, B)]
    cpu = [{"x": x[r0 * row:r1 * row].cpu(), "pred": pred[r0 * row:r1 * row].cpu(), **small} for r0, r1 in slices]

    def op_of(xp, pp, rows, dd):
        op = cabi.Op()
        op.kind = cabi.OP_UPDATE
        u = op.u.update
        u.batch, u.row, u.x, u.pred, u.coef = rows, row, xp, pp, _ptr(dd, "coef")
        u.x_min, u.x_max, u.predict_noise = _ptr(dd, "x_min"), _ptr(dd, "x_max"), 1
        return op
    cabi.run_op(0, op_of(x.data_ptr(), pred.data_ptr(), B, small_gpu), ITER, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for (r0, r1), d in zip(slices, cpu):
        emulator.run_update(op_of(d["x"].data_ptr(), d["pred"].data_ptr(), r1 - r0, d).u.update, ITER)
        assert _same_bits(d["x"], x[r0 * row:r1 * row].cpu()), f"rows [{r0}, {r1}) differ"
    print(f"[update] 64-bit index path ran: batch*row = {n} (2^31 + {n - (1 << 31)})")
    del x, pred


# ======================================================================================================= PREP, CAST
@pytest.mark.gpu
@pytest.mark.parametrize("noise", [False, True])
def test_prep_is_bit_exact(noise):
    B, row = 29, 54
    n = B * row
    g = torch.Generator().manual_seed(11)
    cpu = {"x": torch.cat([torch.randn(n, generator=g), torch.full((GUARD,), float("nan"))]),
           "xin": torch.full((n + GUARD,), float("nan")), "noise": torch.randn(3 * n, generator=g),
           "coef": _coef(5, CM, 2 if noise else None)}
    gpu = _to(cpu, DEV)

    def op_of(dd):
        op = cabi.Op()
        op.kind = cabi.OP_PREP
        p = op.u.prep
        p.batch, p.row, p.x, p.xin, p.noise, p.coef = B, row, _ptr(dd, "x"), _ptr(dd, "xin"), _ptr(dd, "noise"), _ptr(dd, "coef")
        return op
    emulator.run_prep(op_of(cpu).u.prep, ITER)
    cabi.run_op(0, op_of(gpu), ITER, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _compare(cpu, gpu, ("x", "xin"))
    assert not torch.isnan(gpu["xin"][:n]).any()


@pytest.mark.gpu
@pytest.mark.parametrize("C_in,C_out", [(3, 6), (14, 16), (14, 32), (7, 12), (30, 32)])
@pytest.mark.parametrize("out_dtype", [cabi.F32, cabi.TF32, cabi.BF16])
def test_cast_is_bit_exact(C_in, C_out, out_dtype):
    B, L = 13, 17
    g = torch.Generator().manual_seed(C_in * 100 + C_out)
    cpu = {"in": torch.randn(B * L * C_in, generator=g),
           "out": torch.full((B * L * C_out + GUARD,), float("nan"), dtype=torch.bfloat16 if out_dtype == cabi.BF16 else torch.float32)}
    gpu = _to(cpu, DEV)

    def op_of(dd):
        op = cabi.Op()
        op.kind = cabi.OP_CAST
        k = op.u.cast
        k.batch, k.L, k.C_in, k.C_out, k.in_, k.out, k.out_dtype = B, L, C_in, C_out, _ptr(dd, "in"), _ptr(dd, "out"), out_dtype
        return op
    emulator.run_cast(op_of(cpu).u.cast)
    cabi.run_op(0, op_of(gpu), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _compare(cpu, gpu, ("out",))
    pads = gpu["out"][:-GUARD].view(-1, C_out)[:, C_in:]
    assert (pads.float() == 0).all() and not torch.signbit(pads.float()).any(), "pad channels are not +0"


# ============================================================================================================== LNMOD
ATOL = 1e-4
R_OUT = {cabi.F32: 0.0, cabi.TF32: 2.0 ** -10, cabi.BF16: 2.0 ** -8}
SPARE = 1024


def ln_path(C, out_off, bstride):
    """the branch ln_modulate_kernel takes (mirrors its conditions)"""
    if C % 4 == 0 and C <= 512 and out_off % 4 == 0 and bstride % 4 == 0:
        n4 = C // 4
        return "<16,3>" if n4 <= 48 else "<16,6>" if (n4 <= 96 and n4 % 16 == 0) else "<32,4>"
    return "scalar" if C <= 512 else "streaming"


LN_CASES = [(C, 0, p) for p, Cs in (("<16,3>", (32, 64, 192)), ("<16,6>", (256, 320, 384)), ("<32,4>", (200, 448, 512)),
                                     ("scalar", (30, 322)), ("streaming", (768, 1024))) for C in Cs] + [(320, 1, "scalar")]


@pytest.mark.gpu
@pytest.mark.parametrize("C,out_off,path", LN_CASES)
def test_lnmod_matches_fp64(C, out_off, path):
    B, L = 37, 7                                            # 259 rows: the 16-lane paths leave a half-warp idle
    st = torch.cuda.current_stream().cuda_stream
    for bstride in (C, 2 * C + 4):
        assert ln_path(C, out_off, bstride) == path
        g = torch.Generator().manual_seed(C + bstride)
        x = (2 * torch.randn(B, L, C, generator=g) + 0.5).to(DEV)
        shift = (0.3 * torch.randn(B, bstride, generator=g)).to(DEV)[:, :C]
        scale = (0.3 * torch.randn(B, bstride, generator=g)).to(DEV)[:, :C]
        ref = opref.lnmod(x, shift, scale, 1e-6)
        y32 = None
        for od in (cabi.F32, cabi.TF32, cabi.BF16):
            runs = []
            for _ in range(2):
                buf = torch.full((out_off + B * L * C + SPARE,), float("nan"), device=DEV,
                                 dtype=torch.bfloat16 if od == cabi.BF16 else torch.float32)
                out = buf[out_off:out_off + B * L * C].view(B, L, C)
                op = cabi.Op()
                op.kind = cabi.OP_LNMOD
                m = op.u.lnmod
                m.batch, m.L, m.C, m.eps = B, L, C, 1e-6
                m.in_, m.out, m.out_dtype = x.data_ptr(), out.data_ptr(), od
                m.shift, m.scale, m.mod_bstride = shift.data_ptr(), scale.data_ptr(), bstride
                cabi.run_op(0, op, 0, st)
                torch.cuda.synchronize()
                assert torch.isnan(buf[:out_off].float()).all() and torch.isnan(buf[out_off + B * L * C:].float()).all(), \
                    "a write outside the output"
                runs.append(out.float().clone())
            assert _same_bits(runs[0], runs[1]), "two runs differ"
            y = runs[0]
            s = max(1.0, ref.abs().mean().item())
            frac = ((y.double() - ref).abs() / (ATOL * s + R_OUT[od] * ref.abs())).max().item()
            assert torch.isfinite(y).all()
            name = f"C={C} off={out_off} bstride={bstride} out={od}"
            if frac > WORST.get(path, (0.0, ""))[0]:
                WORST[path] = (frac, name)
            assert frac <= 1, f"{name}: {frac:.3f} of the bound"
            if od == cabi.F32:
                y32 = y
            else:
                assert _same_bits(opref.store(y32, od), y), f"{name}: not the rounding of the fp32 output"
