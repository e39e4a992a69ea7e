"""Host runtime of the CUDA sampling engine: plan cache, per-call table fill, graph replay.

``try_sample`` is called by ``{Discrete,Continuous}DiffusionSDE.sample`` after the prologue (initial
noise, mask, nn_condition) and replaces the whole Python reverse loop (diffusionsde.py:525-594) by

    tables  <- per-iteration solver coefficients + time-conditioning rows      (host, tiny)
    noise   <- the loop's torch.randn_like draws, taken up front IN THE SAME ORDER (so a seeded run consumes
               the generator exactly like the reference loop would)
    x_t     <- one device buffer, updated in place by the last operator of every iteration
    replay  <- cds_plan_run: one CUDA graph per iteration, indexed by a device-side counter

It returns ``None`` when the request is outside what the kernels cover (custom backbone, attention UNet,
odd shapes ...) and the caller continues on the PyTorch path; a missing/unsound extension raises.

Environment switches (no flag system, pipelines stay unchanged):
  CDS_BACKEND = auto | torch | cuda    (torch: never use the engine; cuda: raise instead of falling back)
  CDS_MATH    = tf32 | bf16 | fp32     (conv/linear GEMMs: wgmma with fp32 activations read as TF32 -- the default, the
                                        arithmetic of the reference's own GPU path --, wgmma with bf16 operands and
                                        activations, or fp32 FMA on CUDA cores)
  CDS_GRAPH   = 1 | 0                  (0: launch kernels directly, for profilers)
  CDS_NOISE_TAPE_MB                    (cap of the pre-drawn noise tape, default 4096: longer loops are run in chunks)
  CDS_MAX_PLANS                        (plans kept per agent, default 8, least recently used evicted)
"""
import os
import types
from typing import Optional

import torch
import torch.nn.functional as F

from . import cabi
from .lower import (DQLGrad, Program, Unsupported, View, _rev, guide as emit_guide, half_janner_guidable, lower_denoiser,
                    lower_half_janner_grad)
from ..diffusion import solvers as S

# guidance_path: how the latest engine call with classifier guidance was served -- "graph" (the classifier's input gradient is
# part of the replayed program) or "callback" (step by step, PyTorch autograd between the denoiser and the update); None when
# the latest call had no guidance.  guidance_reason: why a guided call took the callback path.
STATS = {"engine_calls": 0, "fallbacks": 0, "last_fallback_reason": None, "launches": 0, "guidance_path": None,
         "guidance_reason": None}


def _backend():
    return os.environ.get("CDS_BACKEND", "auto")


_MATH_MODES = {"fp32": cabi.MATH_FP32, "bf16": cabi.MATH_BF16_TC, "tf32": cabi.MATH_TF32_TC}


def _math_mode():
    name = os.environ.get("CDS_MATH", "tf32")
    if name not in _MATH_MODES:
        raise ValueError(f"CDS_MATH={name!r}: expected one of {sorted(_MATH_MODES)}")
    return _MATH_MODES[name]


def _weights_version(module: torch.nn.Module, epoch: int = 0):
    """Fingerprint of the parameters a plan has packed copies of: tensor identities + autograd version counters (bumped by
    every in-place op on the parameter) + the owner's ``_weights_epoch`` (bumped by optimiser steps, EMA updates and
    checkpoint loads of DiffusionModel -- writes through ``.data`` do not touch the version counters)."""
    acc = int(epoch) & 0xFFFFFFFFFFFF
    for p in module.parameters():
        acc = (acc * 1000003 + p._version * 31 + p.data_ptr()) & 0xFFFFFFFFFFFF
    return acc


def _device_ok(device: torch.device) -> bool:
    """Can the engine serve tensors on ``device``?  CDS_BACKEND=auto: only a CUDA device of compute capability 9.0 (H100) with
    the sm_90a library built; anything else (CPU, other architectures, extension not built) quietly takes the PyTorch loop like
    the reference would.  CDS_BACKEND=cuda: any CUDA device qualifies here and a missing library / wrong architecture fails
    loudly further down (tests and bench run that way)."""
    if device.type != "cuda":
        return False
    if _backend() == "cuda":
        return True
    try:
        cap = torch.cuda.get_device_capability(device)
    except Exception:
        return False
    return cap == (9, 0) and os.path.exists(cabi.lib_path())


def _tape_budget_bytes():
    return int(float(os.environ.get("CDS_NOISE_TAPE_MB", "4096")) * (1 << 20))


def _randn_is_patched():
    """True when a harness replaced torch.randn_like (tests replay recorded draws through it)."""
    return not isinstance(torch.randn_like, types.BuiltinFunctionType)


def _draw_noise(dst, like):
    """One of the loop's ``torch.randn_like(x_t)`` draws, written into tape slot ``dst`` (batch, row).  Filling the slot in
    place with ``normal_`` consumes the device generator exactly like ``randn_like`` (= ``empty_like().normal_()``) without
    the temporary and the copy; a patched ``torch.randn_like`` (replay harness) is honoured."""
    if _randn_is_patched():
        dst.copy_(torch.randn_like(like).reshape(dst.shape))
    else:
        dst.view(like.shape).normal_()


def _make_handle(device: torch.device, ops, n_iters: int):
    """Hand the operator program to libcds (tests substitute a numpy interpreter to check the lowering on CPU)."""
    cabi.load()                                   # raises loudly if the extension is not built
    handle = cabi.Plan(device.index if device.index is not None else torch.cuda.current_device())
    handle.append(ops)
    handle.finalize(n_iters)
    return handle


class _Ctx:
    """What the per-call table fillers see."""

    def __init__(self, t_all, cond_rows):
        self.t_all, self.cond_rows = t_all, cond_rows


def _n_branches(batch, row, consistency):
    """Independent sub-batches ("branches") whose kernel chains run on parallel streams: while one chain sits at a kernel
    boundary (drain, dependency latency, ramp-up: ~3 us of every ~12 us layer) the other chain's kernel keeps the SMs busy.
    CDS_BRANCHES sets the count, CDS_BRANCH_MIN_BATCH the smallest sub-batch worth a branch (default 1024).  Default 1."""
    want = int(os.environ.get("CDS_BRANCHES", "1"))
    min_sub = int(os.environ.get("CDS_BRANCH_MIN_BATCH", "1024"))
    if consistency:
        return 1
    while want > 1 and (batch % want != 0 or batch // want < min_sub or (batch // want * row) % 4 != 0):
        want -= 1
    return max(want, 1)


class SamplerPlan:
    """Everything resident on the device for one (model, batch, x_shape, option set)."""

    def __init__(self, device, net, batch, x_shape, n_iters, n_slots, *, cfg_mode, predict_noise, has_mask,
                 has_min, has_max, keep_history, math, consistency=False, aux_history=False, classifier=None):
        """classifier: a CumRewClassifier over HalfJannerUNet1d (``half_janner_guidable``) whose input gradient at x_t enters the
        prediction between the denoiser and the update of every iteration (``pred += cg_scale[iter] * grad``).
        consistency: the EDM-preconditioned family (ContinuousConsistencyModel, ContinuousEDM): a CDS_OP_PREP in front of the
        denoiser (re-noise + c_in scaling) and the c_skip / c_out combine in the update; aux_history: second history buffer (the
        EDM Heun corrector needs the predictor's x_t and slope)."""
        self.device, self.net, self.batch, self.x_shape = device, net, batch, tuple(x_shape)
        self.classifier = classifier
        row = 1
        for s in x_shape:
            row *= s
        self.row, self.n_iters = row, n_iters
        self.cfg_mode = cfg_mode
        K = _n_branches(batch, row, consistency)
        self.n_branches = K
        root = Program(device, batch * (2 if cfg_mode == 2 else 1), n_iters, math)     # owns the shared buffers
        self.program = root
        self.x = root.buf(batch, *x_shape)
        self.prior = root.buf(batch, *x_shape) if has_mask else None
        self.mask = root.buf(row) if has_mask else None
        self.x_min = root.buf(row) if has_min else None
        self.x_max = root.buf(row) if has_max else None
        self.coef = root.buf(n_iters, cabi.ROW_FLOATS)
        self.noise = root.buf(max(n_slots, 1), batch, row) if n_slots > 0 else None
        self.xhat_prev = root.buf(batch, row) if keep_history else None
        self.aux = root.buf(batch, row) if (keep_history and aux_history) else None
        if consistency:
            self.xin = root.buf(batch, *x_shape)

        L = x_shape[0] if len(x_shape) == 2 else 1
        Cn = x_shape[-1]
        self._update_ops = []
        self._fillers = []                 # (per-call table filler, sub-batch slice)
        sub = batch // K
        for k in range(K):
            off = k * sub                  # first trajectory of this branch
            sl = slice(off, off + sub)
            p = root if K == 1 else Program(device, sub * (2 if cfg_mode == 2 else 1), n_iters, math)
            n_before = len(p.ops)
            fo = 4 * off * row             # byte offset of the branch inside the (batch, row) fp32 buffers
            xin_ptr_t, xin_off = self.x, off * row
            if consistency:
                op = cabi.Op()
                op.kind = cabi.OP_PREP
                q = op.u.prep
                q.batch, q.row, q.x, q.xin, q.coef = sub, row, self.x.data_ptr() + fo, self.xin.data_ptr() + fo, self.coef.data_ptr()
                q.noise = self.noise.data_ptr() if self.noise is not None else None
                p.ops.append(op)
                xin_ptr_t = self.xin
            xview = View(xin_ptr_t, L, Cn, offset=xin_off)
            pred = lower_denoiser(p, net, xview, x_shape, cfg_mode != 0, sub if cfg_mode == 2 else 0)
            if K == 1:                 # the prediction buffer, for host callbacks between denoiser and update (guidance)
                self.pred = pred.t if (pred.offset == 0 and pred.lstride == pred.C and pred.bstride == pred.L * pred.C) else None
            if classifier is not None:
                assert K == 1 and cfg_mode != 2
                grad = lower_half_janner_grad(p, classifier, _input_view(p, n_before, xview))
                self.cg_scale = root.buf(n_iters)           # per-iteration guidance scale, filled by every guided call
                emit_guide(p, pred, grad, self.cg_scale)

            op = cabi.Op()
            op.kind = cabi.OP_UPDATE
            u = op.u.update
            u.batch, u.row, u.x = sub, row, self.x.data_ptr() + fo
            u.pred = pred.ptr
            if cfg_mode == 2:
                u.pred_uncond = pred.ptr + 4 * sub * row
            if self.noise is not None:
                u.noise, u.noise_slot_stride = self.noise.data_ptr() + fo, batch * row
            u.prior = self.prior.data_ptr() + fo if has_mask else None
            u.mask = self.mask.data_ptr() if has_mask else None
            u.x_min = self.x_min.data_ptr() if has_min else None
            u.x_max = self.x_max.data_ptr() if has_max else None
            u.xhat_prev = self.xhat_prev.data_ptr() + fo if keep_history else None
            u.aux = self.aux.data_ptr() + fo if self.aux is not None else None
            u.coef = self.coef.data_ptr()
            u.predict_noise = 1 if predict_noise else 0
            u.final_clip = 1 if consistency else 0
            # tensor-core UNets read x_t through a channel-padded bf16 copy (CDS_OP_CAST).  When that cast converts the very
            # buffer the update writes, the update emits the copy itself and the cast runs only once per sample() call.
            for cop in p.ops[n_before:]:
                if cop.kind == cabi.OP_CAST and cop.u.cast.in_ == self.x.data_ptr() + fo and cop.u.cast.batch == sub:
                    cop.flags |= cabi.OPF_ONCE
                    u.x_cast, u.cast_C_in, u.cast_C_out = cop.u.cast.out, cop.u.cast.C_in, cop.u.cast.C_out
                    u.x_cast_dtype = cop.u.cast.out_dtype
            self._update_ops.append(op)
            p.ops.append(op)
            self._fillers += [(fn, sl) for fn in p.per_call]
            if p is not root:
                for o in p.ops:
                    o.flags |= k << cabi.OPF_BRANCH_SHIFT
                root.ops += p.ops
                root.keep += p.keep + [p]
                root.packers += p.packers

        self.handle: Optional[cabi.Plan] = None
        self.version = None              # set by the first refresh_weights()

    def build(self, w_cfg: float):
        for op in self._update_ops:
            op.u.update.w_cfg, op.u.update.w_uncond = float(w_cfg), float(1 - w_cfg)
        self.w_cfg = w_cfg
        self.handle = _make_handle(self.device, self.program.ops, self.n_iters)

    def refresh_weights(self, epoch: int = 0):
        v = _weights_version(self.net, epoch)
        if self.classifier is not None:
            v = _weights_version(self.classifier.model_ema, v)
        if self.version is None:         # packed at construction
            self.version = v
        elif v != self.version:
            for fn in self.program.packers:
                fn()
            self.version = v

    def close(self):
        if self.handle is not None:
            self.handle.close()
            self.handle = None

    def fill_tables(self, t_all, cond_emb, t_key=None):
        """Per-call tables (time-conditioning rows, per-trajectory condition terms), once per ``sample()``."""
        # table fillers that depend on (weights, timesteps) only are skipped when neither changed since the last call
        fresh = t_key is None or (t_key, self.version) != getattr(self, "_time_tables_key", None)
        with torch.no_grad():
            for fn, sl in self._fillers:             # every branch fills its own tables from its slice of the condition
                if fresh or not getattr(fn, "time_only", False):
                    fn(_Ctx(t_all, _cond_rows(self.cfg_mode, None if cond_emb is None else cond_emb[sl])))
        self._time_tables_key = (t_key, self.version) if t_key is not None else None

    def run(self, t_all, cond_emb, use_graph=True, t_key=None, first=0, count=None, fill=True):
        if fill:
            self.fill_tables(t_all, cond_emb, t_key)
        stream = torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else 0
        self.handle.run(first, self.n_iters - first if count is None else count, stream, use_graph)
        STATS["launches"] = self.handle.launches_per_iter() * self.n_iters + 1

    def run_guided(self, t_all, cond_emb, xt, noise_slots, guide, t_key=None):
        """The loop with a host callback between the denoiser and the update of every iteration (classifier guidance,
        diffusionsde.py:153-173): per iteration the denoiser operators are enqueued through the single-step entry
        (cds_plan_run_range), ``guide(n, x_t, pred)`` edits the prediction in place with ordinary PyTorch ops on the same stream,
        then the update operator runs.  ``noise_slots[n]`` = 1 + tape slot of iteration n's draw, 0 = none."""
        assert self.n_branches == 1 and self.pred is not None
        ops = self.program.ops
        upd = max(i for i, op in enumerate(ops) if op.kind == cabi.OP_UPDATE)
        assert upd == len(ops) - 1, "the update must be the program's last operator"
        self.fill_tables(t_all, cond_emb, t_key)
        stream = torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else 0
        x_view = self.x.view(self.batch, *self.x_shape)
        pred_view = self.pred.view(-1, *self.x_shape)[:self.batch]
        self.handle.run(0, 0, stream, False)                       # the CDS_OPF_ONCE operators (x_t hand-over cast)
        for n in range(self.n_iters):
            slot = int(noise_slots[n]) - 1
            if slot >= 0:
                with torch.no_grad():
                    _draw_noise(self.noise[slot], xt)
            self.handle.run_range(n, 0, upd, stream)
            guide(n, x_view, pred_view)
            self.handle.run_range(n, upd, 1, stream)
        STATS["launches"] = (self.handle.launches_per_iter() + 2) * self.n_iters + 1

    def run_chunked(self, t_all, cond_emb, xt, noise_rows, use_graph=True, t_key=None):
        """The whole loop, with the noise tape refilled between chunks when it is shorter than the number of draws
        (``noise_rows[n]`` = does iteration n draw?).  The draws are taken in loop order, so a seeded run consumes the
        generator like the reference loop; everything is enqueued on one stream, so a refill cannot overtake its readers."""
        cap = self.noise.shape[0] if self.noise is not None else 0
        self.fill_tables(t_all, cond_emb, t_key)
        timed = STATS.get("time_loop") and self.device.type == "cuda"
        if timed:           # bench.py: device time of the reverse loop alone (noise draws + replayed iterations; events on the
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)    # launching stream)
            e0.record()
        first, used = 0, 0
        with torch.no_grad():
            for n in range(self.n_iters + 1):
                draws = n < self.n_iters and bool(noise_rows[n])
                if n == self.n_iters or (draws and used == cap):
                    if n > first:
                        self.run(t_all, cond_emb, use_graph, t_key, first=first, count=n - first, fill=False)
                    first, used = n, 0
                if draws:
                    _draw_noise(self.noise[used], xt)
                    used += 1
        if timed:
            e1.record()
            STATS.setdefault("loop_events", []).append((e0, e1))


def _input_view(p: Program, n_before: int, x: View) -> View:
    """x_t as the denoiser's operators read it: the channel-padded copy of a CDS_OP_CAST appended since ``n_before`` when there
    is one (tensor-core programs), else ``x``"""
    for op in p.ops[n_before:]:
        k = op.u.cast
        if op.kind == cabi.OP_CAST and k.in_ == x.ptr:
            t = next(t for t in p.keep if t.data_ptr() == k.out)
            return View(t, k.L, k.C_out, tf32=k.out_dtype == cabi.TF32)
    return x


def _row(t, x_shape, device):
    return torch.broadcast_to(t.to(device=device, dtype=torch.float32), (1, *x_shape)).reshape(-1)


def _device_of(agent):
    return torch.device(agent.device)


def _fallback(reason):
    STATS["fallbacks"] += 1
    STATS["last_fallback_reason"] = reason
    if _backend() == "cuda":
        raise RuntimeError(f"CDS_BACKEND=cuda but the engine cannot serve this call: {reason}")
    return None


def _cfg_mode(w_cfg, cond_emb):
    if w_cfg == 0.0 or cond_emb is None:
        return 0 if (w_cfg == 0.0 or w_cfg == 1.0) else None     # two-branch CFG without a condition is an error upstream
    return 1 if w_cfg == 1.0 else 2


def _get_plan(agent, key, factory):
    """Plan cache of one agent: least-recently-used order, at most CDS_MAX_PLANS entries (each pins device buffers)."""
    plans = agent._engine_plans
    plan = plans.pop(key, None)
    if plan is None:
        plan = factory()
        limit = max(1, int(os.environ.get("CDS_MAX_PLANS", "8")))
        while len(plans) >= limit:
            old = plans.pop(next(iter(plans)))
            if hasattr(old, "close"):
                old.close()
    plans[key] = plan                      # (re-)insert at the most-recently-used end
    plan.refresh_weights(getattr(agent, "_weights_epoch", 0))
    return plan


def _cond_rows(cfg_mode, cond_emb):
    if cfg_mode == 0 or cond_emb is None:
        return None
    c = cond_emb.to(torch.float32)
    return torch.cat([c, torch.zeros_like(c)], 0) if cfg_mode == 2 else c


def try_sample(agent, *, model, xt, prior, solver, sample_steps, order, step_values, alphas, sigmas, hs, stds,
               cond_emb, w_cfg, n_samples, guide=None, table=None, clip_in_loop=True, predict_noise=None, sched_id=None,
               classifier=None, w_cg=0.0):
    """``table``: optional ready-made ``(coefficient rows [n_iters, ROW], number of noise slots, int64/float32 time per iteration)``
    for samplers that are "the same update kernel with another coefficient table" (the legacy DDPM class, RectifiedFlow's Euler
    step): ``solver`` / ``alphas`` / ``sigmas`` / ``hs`` / ``stds`` / ``step_values`` are then unused.
    ``clip_in_loop=False``: the sampler clips only its final sample (RectifiedFlow); ``predict_noise``: overrides
    ``agent.predict_noise`` (classes without that attribute).
    ``guide``: optional host callback ``guide(n, i, x_t, pred)`` (n = iteration, i = its loop index) run between the denoiser
    and the update of every iteration (classifier guidance); the loop then runs step by step instead of as a replayed graph --
    unless ``classifier`` (the one ``guide`` evaluates, with weight ``w_cg``) is a CumRewClassifier over HalfJannerUNet1d under
    CDS_MATH = fp32 | tf32 with one sub-batch chain: its input gradient and the guidance term are then operators of the replayed
    program, and ``guide`` is not called."""
    if _backend() == "torch":
        return None
    device = _device_of(agent)
    if not _device_ok(device) or xt.dtype != torch.float32:
        return None
    net = model["diffusion"]
    cfg_mode = _cfg_mode(w_cfg, cond_emb)
    if cfg_mode is None:
        return _fallback("two-branch CFG without condition")
    batch, x_shape = xt.shape[0], tuple(xt.shape[1:])
    if n_samples != batch:
        return _fallback("n_samples != prior.shape[0]")
    if guide is not None and cfg_mode == 2:
        # the update operator combines the two CFG branches itself; a guidance term would have to enter after that combine
        return _fallback("classifier guidance together with two-branch classifier-free guidance")

    table, n_slots, t_cpu, sched_key, order, table_given = _step_table(
        agent, solver=solver, sample_steps=sample_steps, order=order, step_values=step_values, alphas=alphas, sigmas=sigmas,
        hs=hs, stds=stds, table=table, sched_id=sched_id)
    keep_history = (not table_given) and S.solver_keeps_history(solver)
    has_mask = isinstance(agent.fix_mask, torch.Tensor)
    has_min, has_max = (agent.x_min is not None and clip_in_loop), (agent.x_max is not None and clip_in_loop)
    pn = bool(agent.predict_noise) if predict_noise is None else bool(predict_noise)
    math = _math_mode()
    row_elems = 1
    for s_ in x_shape:
        row_elems *= s_
    cg_reason = None                       # why a guided call keeps the host callback (None: the graph serves it)
    if guide is not None:
        cg_reason = "no classifier" if classifier is None else half_janner_guidable(classifier, x_shape)
        if cg_reason is None and math == cabi.MATH_BF16_TC:
            cg_reason = "CDS_MATH=bf16"
        if cg_reason is None and _n_branches(batch, row_elems, False) != 1:
            cg_reason = "more than one sub-batch chain (CDS_BRANCHES)"
    lowered_cg = guide is not None and cg_reason is None
    # noise tape: all draws of the loop up front when they fit the budget, else as many slots as fit (the loop then runs in
    # chunks with the tape refilled in between -- O(budget) memory instead of O(sample_steps x batch x row))
    tape_slots = min(n_slots, max(1, _tape_budget_bytes() // (4 * batch * row_elems))) if n_slots > 0 else 0
    key = ("sde", id(net), batch, x_shape, len(order), tape_slots, cfg_mode, pn, has_mask,
           has_min, has_max, keep_history, math, float(w_cfg) if cfg_mode == 2 else 0.0,
           id(classifier.model_ema) if lowered_cg else None)

    def factory():
        plan = SamplerPlan(device, net, batch, x_shape, len(order), tape_slots, cfg_mode=cfg_mode,
                           predict_noise=pn, has_mask=has_mask, has_min=has_min, has_max=has_max,
                           keep_history=keep_history, math=math, classifier=classifier if lowered_cg else None)
        plan.build(w_cfg)
        return plan

    try:
        plan = _get_plan(agent, key, factory)
    except Unsupported as e:
        return _fallback(str(e))
    except cabi.CdsError as e:
        if e.code == -3:
            return _fallback(str(e))
        raise

    t_all = _load_resident(agent, plan, xt, prior, table, sched_key, tape_slots, n_slots, x_shape, order, t_cpu, device)
    # the loop's draws: same calls, same order, same shapes as the reference loop's (diffusionsde.py:548,571,...)
    t_key = (t_cpu.numpy().tobytes(), tuple(order))
    STATS["guidance_path"], STATS["guidance_reason"] = None, cg_reason
    if lowered_cg:
        # the guidance scale of every iteration, the reference's own expression (classifier_guidance), evaluated on the device
        with torch.no_grad():
            idx = torch.as_tensor(order, dtype=torch.long).to(device)
            sig = sigmas.to(device)[idx]
            plan.cg_scale.copy_(-(w_cg * sig) if pn else w_cg * ((sig ** 2) / alphas.to(device)[idx]))
        STATS["guidance_path"] = "graph"
        guide = None
    if guide is not None:
        STATS["guidance_path"] = "callback"
        if plan.n_branches != 1 or getattr(plan, "pred", None) is None:
            return _fallback("guided sampling needs a single-branch program with a dense prediction buffer")
        slots = plan.coef[:, S.R_NOISE].cpu().tolist()              # tape slot per iteration as the update kernel sees it
        plan.run_guided(t_all, cond_emb, xt, slots, lambda n, x, p: guide(n, order[n], x, p), t_key=t_key)
    else:
        plan.run_chunked(t_all, cond_emb, xt, (table[:, S.R_NOISE] > 0).tolist(),
                         use_graph=os.environ.get("CDS_GRAPH", "1") != "0", t_key=t_key)
    STATS["engine_calls"] += 1
    return plan.x.clone()


def _step_table(agent, *, solver, sample_steps, order, step_values, alphas, sigmas, hs, stds, table, sched_id):
    """The coefficient table of one ``sample()`` call -> ``(table [n_iters, ROW], number of noise slots, time per step (CPU),
    schedule key, iteration order, table_given)``."""
    # ---- per-iteration scalars (host, reference op order); identical requests reuse the table (building it costs ~10 ms
    # of Python scalar arithmetic for 100 steps -- more than a tenth of a whole cfg2 sample() on the engine) ---------------
    table_given = table is not None
    if table_given:
        rows_given, slots_given, t_given = table
        t_cpu = t_given.detach().cpu()
        order = list(range(rows_given.shape[0]))
        sched_key = (solver, rows_given.numpy().tobytes(), t_cpu.numpy().tobytes())
        cached = (rows_given, int(slots_given))
    else:
        # ``sched_id``: a hashable the caller vouches for -- everything alphas / sigmas / hs / stds / step_values are functions of.
        # A hit skips the five device->host reads below: each of them is a stream synchronisation, which would keep the host from
        # preparing call n + 1 while call n still runs (1-step samplers: a quarter of the wall time).
        fast_key = None if sched_id is None else (sched_id, solver, sample_steps, tuple(order))
        fast = agent.__dict__.setdefault("_engine_sched_ids", {}).get(fast_key) if fast_key is not None else None
        if fast is not None:
            sched_key, t_cpu = fast
            cached = agent._engine_tables.get(sched_key) if hasattr(agent, "_engine_tables") else None
        else:
            cached = None
        if cached is None:
            alphas_c, sigmas_c, hs_c, stds_c = (z.detach().float().cpu() for z in (alphas, sigmas, hs, stds))
            t_cpu = step_values.detach().cpu()
            sched_key = (solver, sample_steps, tuple(order), alphas_c.numpy().tobytes(), sigmas_c.numpy().tobytes(),
                         hs_c.numpy().tobytes(), stds_c.numpy().tobytes(), t_cpu.numpy().tobytes())
            cached = agent._engine_tables.get(sched_key) if hasattr(agent, "_engine_tables") else None
            if fast_key is not None:
                if len(agent._engine_sched_ids) > 16:
                    agent._engine_sched_ids.clear()
                agent._engine_sched_ids[fast_key] = (sched_key, t_cpu)
    if cached is None:
        table = S.coeff_table(solver, order, sample_steps, alphas_c, sigmas_c, hs_c, stds_c, t_cpu.double())
        n_slots = 0
        for n in range(len(order)):
            if table[n, S.R_NOISE] > 0:
                n_slots += 1
                table[n, S.R_NOISE] = float(n_slots)       # 1 + slot index
        if not hasattr(agent, "_engine_tables"):
            agent._engine_tables = {}
        if len(agent._engine_tables) > 16:
            agent._engine_tables.clear()
        agent._engine_tables[sched_key] = (table, n_slots)
    else:
        table, n_slots = cached
    return table, n_slots, t_cpu, sched_key, order, table_given


def _load_resident(agent, plan, xt, prior, table, sched_key, tape_slots, n_slots, x_shape, order, t_cpu, device):
    """Fill the plan's resident buffers (x_t, coefficient rows, mask, clip bounds) -> the time value of every iteration."""
    with torch.no_grad():
        plan.x.copy_(xt)
        if getattr(plan, "_coef_key", None) != sched_key:
            if tape_slots and tape_slots < n_slots:          # slots are reused chunk by chunk: k-th draw -> slot k mod tape_slots
                local = table.clone()
                draws = local[:, S.R_NOISE] > 0
                local[draws, S.R_NOISE] = (local[draws, S.R_NOISE] - 1) % tape_slots + 1
                plan.coef.copy_(local)
            else:
                plan.coef.copy_(table)
            plan._coef_key = sched_key
        if plan.mask is not None:
            plan.prior.copy_(prior)
            plan.mask.copy_(_row(agent.fix_mask, x_shape, device))
        if plan.x_min is not None:
            plan.x_min.copy_(_row(agent.x_min, x_shape, device))
        if plan.x_max is not None:
            plan.x_max.copy_(_row(agent.x_max, x_shape, device))
        idx = torch.as_tensor(order, dtype=torch.long)
        return t_cpu[idx].to(device)      # int64 (discrete) or float32 (continuous), one entry per iteration


def try_sample_consistency(agent, *, model, xt, prior, sigmas, order, cond_emb, n_samples, sched_id=None):
    """ContinuousConsistencyModel.sample on the engine: iteration 0 evaluates f at sigma_max, the following
    iterations re-noise to sigma_i and evaluate f again (consistency_model.py:401-426)."""
    if _backend() == "torch":
        return None
    device = _device_of(agent)
    if not _device_ok(device) or xt.dtype != torch.float32:
        return None
    net = model["diffusion"]
    batch, x_shape = xt.shape[0], tuple(xt.shape[1:])
    if n_samples != batch:
        return _fallback("n_samples != prior.shape[0]")
    cfg_mode = 0 if cond_emb is None else 1
    # ``sched_id`` (see try_sample): a hit reuses the coefficient table and its device copy of the time column -- no device->host
    # read, so the host can prepare the next call while this one runs (the 1-step sampler is 8 ms of GPU work per call)
    cm_key = None if sched_id is None else (sched_id, tuple(order), str(device))
    hit = agent.__dict__.setdefault("_engine_cm_tables", {}).get(cm_key) if cm_key is not None else None
    sig = None if hit is not None else sigmas.detach().float().cpu()
    levels = [] if hit is not None else [sig[-1]] + [sig[i] for i in order]
    n_iters = hit[0].shape[0] if hit is not None else len(levels)
    sd, smin = agent.sigma_data, agent.sigma_min
    table = hit[0] if hit is not None else torch.zeros((n_iters, S.ROW), dtype=torch.float32)
    for n, s in enumerate(levels):                     # 0-d fp32 tensors, reference op order (:241-251, :423)
        table[n, S.R_K0] = float(sd ** 2 / (sd ** 2 + (s - smin) ** 2))                      # c_skip
        table[n, S.R_K1] = float((s - smin) * sd / (sd ** 2 + s ** 2).sqrt())               # c_out
        table[n, S.R_K3] = float(1 / (sd ** 2 + s ** 2).sqrt())                              # c_in
        table[n, S.R_KIND] = float(S.UPD_CM)
        if n > 0:
            table[n, S.R_K2] = float((s ** 2 - smin ** 2).sqrt())                            # re-noise scale
            table[n, S.R_NOISE] = float(n)
        table[n, S.R_T] = float(0.25 * s.log())                                               # c_noise
    n_slots = n_iters - 1
    has_mask = isinstance(agent.fix_mask, torch.Tensor)
    has_min, has_max = agent.x_min is not None, agent.x_max is not None
    math = _math_mode()
    key = ("cm", id(net), batch, x_shape, n_iters, cfg_mode, has_mask, has_min, has_max, math)

    def factory():
        plan = SamplerPlan(device, net, batch, x_shape, n_iters, n_slots, cfg_mode=cfg_mode, predict_noise=False,
                           has_mask=has_mask, has_min=has_min, has_max=has_max, keep_history=False, math=math,
                           consistency=True)
        plan.build(1.0)
        return plan

    try:
        plan = _get_plan(agent, key, factory)
    except Unsupported as e:
        return _fallback(str(e))
    except cabi.CdsError as e:
        if e.code == -3:
            return _fallback(str(e))
        raise
    with torch.no_grad():
        plan.x.copy_(xt)
        plan.coef.copy_(table, non_blocking=True)
        if has_mask:
            plan.prior.copy_(prior)
            plan.mask.copy_(_row(agent.fix_mask, x_shape, device))
        if has_min:
            plan.x_min.copy_(_row(agent.x_min, x_shape, device))
        if has_max:
            plan.x_max.copy_(_row(agent.x_max, x_shape, device))
        for k in range(n_slots):
            _draw_noise(plan.noise[k], xt)
        if hit is not None:
            t_all = hit[1]
        else:
            t_all = table[:, S.R_T].to(device)         # the network sees c_noise = ln(sigma)/4 as its "time"
            if cm_key is not None:
                if len(agent._engine_cm_tables) > 16:
                    agent._engine_cm_tables.clear()
                agent._engine_cm_tables[cm_key] = (table, t_all)
    plan.run(t_all, cond_emb, use_graph=os.environ.get("CDS_GRAPH", "1") != "0")
    STATS["engine_calls"] += 1
    return plan.x.clone()


def try_sample_edm(agent, *, model, xt, prior, solver, sigmas, order, cond_emb, w_cfg, n_samples, evals=None, clip=True,
                   sched_id=None):
    """ContinuousEDM.sample on the engine (newedm.py:395-431).  Every network evaluation is one engine iteration:
    ``euler``: one per reverse step; ``heun``: predictor + corrector (two evaluations) for every step but the last.
    ``sigmas``: the Karras grid (sample_steps + 1 entries, fp32), ``order``: the reverse steps i in loop order."""
    if _backend() == "torch":
        return None
    device = _device_of(agent)
    if not _device_ok(device) or xt.dtype != torch.float32:
        return None
    net = model["diffusion"]
    cfg_mode = _cfg_mode(w_cfg, cond_emb)
    if cfg_mode is None:
        return _fallback("two-branch CFG without condition")
    batch, x_shape = xt.shape[0], tuple(xt.shape[1:])
    if n_samples != batch:
        return _fallback("n_samples != prior.shape[0]")
    sd = agent.sigma_data
    given = evals is not None                    # legacy EDM: the caller lists the evaluations (sigma, kind, dt, flag, xw, dw)
    # ``sched_id`` (see try_sample): a hit reuses the table without reading the Karras grid back from the device
    edm_key = None if (sched_id is None or given) else (sched_id, solver, tuple(order), str(device))
    hit = agent.__dict__.setdefault("_engine_edm_tables", {}).get(edm_key) if edm_key is not None else None
    sig = sigmas.detach().float().cpu() if (not given and hit is None) else None
    evals = list(evals) if given else []         # (sigma of the evaluation, kind, dt, predictor flag[, x_weight, D_weight])
    for i in ([] if (given or hit is not None) else order):
        dt = sig[i] - sig[i - 1]
        heun = solver == "heun" and i > 1
        evals.append((sig[i], S.UPD_EDM, dt, 1.0 if heun else 0.0))
        if heun:
            # the corrector evaluates at t = t_i / sigma_i * sigma_{i-1} (newedm.py:421) = sigma_{i-1} exactly (x / x == 1)
            evals.append((sig[i - 1], S.UPD_EDM_HEUN, dt, 0.0))
    n_iters = hit[0].shape[0] if hit is not None else len(evals)
    table = hit[0] if hit is not None else torch.zeros((n_iters, S.ROW), dtype=torch.float32)
    for n, ev in enumerate(evals):                         # 0-d fp32 tensors, reference op order (newedm.py:128-148)
        s, kind, dt, pred_flag = ev[:4]
        if len(ev) > 4:
            table[n, S.R_XW], table[n, S.R_DW] = float(ev[4]), float(ev[5])
        table[n, S.R_K0] = float(sd ** 2 / (sd ** 2 + s ** 2))                  # c_skip
        table[n, S.R_K1] = float(s * sd / (sd ** 2 + s ** 2).sqrt())            # c_out
        table[n, S.R_K3] = float(1 / (sd ** 2 + s ** 2).sqrt())                 # c_in
        table[n, S.R_K2] = float(dt)
        table[n, S.R_K4] = pred_flag
        table[n, S.R_SIGMA] = float(s)                                          # the slope divides by it
        table[n, S.R_KIND] = float(kind)
        table[n, S.R_T] = float(0.25 * s.log())                                 # c_noise
    has_mask = isinstance(agent.fix_mask, torch.Tensor)
    has_min = clip and getattr(agent, "x_min", None) is not None
    has_max = clip and getattr(agent, "x_max", None) is not None
    math = _math_mode()
    heun = solver == "heun"
    key = ("edm", id(net), batch, x_shape, n_iters, cfg_mode, has_mask, has_min, has_max, heun, math,
           float(w_cfg) if cfg_mode == 2 else 0.0)

    def factory():
        plan = SamplerPlan(device, net, batch, x_shape, n_iters, 0, cfg_mode=cfg_mode, predict_noise=False,
                           has_mask=has_mask, has_min=has_min, has_max=has_max, keep_history=heun, math=math,
                           consistency=True, aux_history=heun)
        plan.build(w_cfg)
        return plan

    try:
        plan = _get_plan(agent, key, factory)
    except Unsupported as e:
        return _fallback(str(e))
    except cabi.CdsError as e:
        if e.code == -3:
            return _fallback(str(e))
        raise
    with torch.no_grad():
        plan.x.copy_(xt)
        plan.coef.copy_(table, non_blocking=True)
        if has_mask:
            plan.prior.copy_(prior)
            plan.mask.copy_(_row(agent.fix_mask, x_shape, device))
        if has_min:
            plan.x_min.copy_(_row(agent.x_min, x_shape, device))
        if has_max:
            plan.x_max.copy_(_row(agent.x_max, x_shape, device))
        if hit is not None:
            t_all = hit[1]
        else:
            t_all = table[:, S.R_T].to(device)         # the network sees c_noise = ln(sigma)/4 as its "time"
            if edm_key is not None:
                if len(agent._engine_edm_tables) > 16:
                    agent._engine_edm_tables.clear()
                agent._engine_edm_tables[edm_key] = (table, t_all)
    plan.run(t_all, cond_emb, use_graph=os.environ.get("CDS_GRAPH", "1") != "0")
    STATS["engine_calls"] += 1
    return plan.x.clone()


# ============================================================================ differentiable sampling (requires_grad=True)
class GradSamplerPlan(SamplerPlan):
    """The resident state of ``sample(requires_grad=True)`` over DQLMlp: a forward program (``lower.DQLGrad``'s network
    operators, which stash x_n, the hidden pre-activations and the raw prediction of every iteration, then the solver update)
    and a backward program that walks the iterations in reverse.  Each is one cds_plan replayed from a CUDA graph.  One branch,
    no CFG combine, no solver history."""

    def __init__(self, device, net, batch, x_shape, n_iters, n_slots, *, predict_noise, has_mask, has_min, has_max, math):
        self.device, self.net, self.batch, self.x_shape = device, net, batch, tuple(x_shape)
        row = x_shape[0]
        self.row, self.n_iters, self.cfg_mode, self.n_branches = row, n_iters, 1, 1
        root = Program(device, batch, n_iters, math)
        back = Program(device, batch, n_iters, math)
        self.program, self.back = root, back
        self.x = root.buf(batch, row)
        self.prior = root.buf(batch, row) if has_mask else None
        self.mask = root.buf(row) if has_mask else None
        self.x_min = root.buf(row) if has_min else None
        self.x_max = root.buf(row) if has_max else None
        self.coef = root.buf(n_iters, cabi.ROW_FLOATS)
        self.noise = root.buf(max(n_slots, 1), batch, row) if n_slots > 0 else None
        self.grad = g = DQLGrad(root, back, net, View(self.x, 1, row))
        self.pred = g.pred.t

        op = cabi.Op()
        op.kind = cabi.OP_UPDATE
        u = op.u.update
        u.batch, u.row, u.x, u.pred = batch, row, self.x.data_ptr(), g.pred.ptr
        if self.noise is not None:
            u.noise, u.noise_slot_stride = self.noise.data_ptr(), batch * row
        u.prior = self.prior.data_ptr() if has_mask else None
        u.mask = self.mask.data_ptr() if has_mask else None
        u.x_min = self.x_min.data_ptr() if has_min else None
        u.x_max = self.x_max.data_ptr() if has_max else None
        u.coef = self.coef.data_ptr()
        u.predict_noise = 1 if predict_noise else 0
        root.ops.append(op)
        self._update_ops = [op]

        bop = cabi.Op()                                      # the update's backward opens every backward iteration
        bop.kind = cabi.OP_UPDATE_BWD
        b = bop.u.update_bwd
        b.batch, b.row, b.gx, b.gpred = batch, row, g.gx.data_ptr(), g.gpred.data_ptr()
        b.x, b.x_iter_stride = _rev(g.xs)
        b.pred, b.pred_iter_stride = _rev(g.ps)
        b.mask = u.mask
        b.x_min, b.x_max = u.x_min, u.x_max
        b.coef, b.coef_iter_stride = _rev(self.coef)
        b.predict_noise = u.predict_noise
        back.ops.insert(0, bop)

        self._fillers = []                 # the tables are autograd inputs, copied in by _GradSampleFn
        self.handle: Optional[cabi.Plan] = None
        self.back_handle: Optional[cabi.Plan] = None
        self.version = None
        self.generation = 0                # forward runs so far: a backward must belong to the latest one

    def build(self, w_cfg: float):
        super().build(w_cfg)
        self.back_handle = _make_handle(self.device, self.back.ops, self.n_iters)

    def refresh_weights(self, epoch: int = 0):
        v = _weights_version(self.net, epoch)
        if self.version is None:
            self.version = v
        elif v != self.version:
            for fn in self.program.packers + self.back.packers:
                fn()
            self.version = v

    def close(self):
        super().close()
        if self.back_handle is not None:
            self.back_handle.close()
            self.back_handle = None

    def backward(self, grad_x0, generation):
        """d x0 -> the gradients of the Function's inputs (step_tab, samp_tab, W_x, W2, b2, W3, b3, W_f, b_f)."""
        if generation != self.generation:
            raise RuntimeError("the engine's saved iterations of this sample(requires_grad=True) call were overwritten by a later "
                               "call with the same shapes; call backward() before sampling again")
        g = self.grad
        with torch.no_grad():
            for t in g.accumulators:
                t.zero_()
            g.gx.copy_(grad_x0.reshape(g.gx.shape))
        stream = torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else 0
        self.back_handle.run(0, self.n_iters, stream, os.environ.get("CDS_GRAPH", "1") != "0")
        STATS["backward_launches"] = self.back_handle.launches_per_iter() * self.n_iters + 1
        return (g.g_step.clone(), g.g_samp.clone(), g.g_w[0].clone(), g.g_w[1].clone(), g.g_b[1].clone(),
                g.g_w[2].clone(), g.g_b[2].clone(), g.g_w[3].clone(), g.g_b[3].clone())


class _GradSampleFn(torch.autograd.Function):
    """x0 of the engine's reverse loop as a function of the per-call tables and the DQLMlp weights the loop reads."""

    @staticmethod
    def forward(ctx, plan, run, step_tab, samp_tab, w_x, w2, b2, w3, b3, w_f, b_f):
        plan.grad.step_tab.copy_(step_tab)
        plan.grad.samp_tab.copy_(samp_tab)
        run()
        plan.generation += 1
        ctx.plan, ctx.generation = plan, plan.generation
        return plan.x.clone()

    @staticmethod
    def backward(ctx, grad_x0):
        return (None, None) + ctx.plan.backward(grad_x0, ctx.generation)


def grad_fallback(agent):
    """``requires_grad=True`` on a sampler class that has no differentiable engine program: recorded (raised under
    CDS_BACKEND=cuda) like every other fallback; the caller then runs its PyTorch loop, which autograd differentiates."""
    if _backend() != "torch" and _device_ok(_device_of(agent)):
        return _fallback(f"requires_grad=True: {type(agent).__name__} has no differentiable engine program")
    return None


def try_sample_grad(agent, *, model, xt, prior, solver, sample_steps, order, step_values, alphas, sigmas, hs, stds,
                    cond_emb, w_cfg, n_samples, guided=False, sched_id=None):
    """``sample(requires_grad=True)`` on the engine: x0 connected to autograd through ``_GradSampleFn``.  Covers DQLMlp with
    the DDPM / DDIM / first-order DPM-Solver updates, one CFG branch and CDS_MATH = fp32 | tf32; everything else takes the
    PyTorch loop (which autograd differentiates) through ``_fallback``."""
    if _backend() == "torch":
        return None
    device = _device_of(agent)
    if not _device_ok(device) or xt.dtype != torch.float32:
        return None
    net = model["diffusion"]
    name = type(net).__name__
    if name != "DQLMlp" or xt.dim() != 2:
        return _fallback(f"requires_grad=True: backbone {name} has no differentiable engine program (DQLMlp only)")
    if S.solver_keeps_history(solver):
        return _fallback(f"requires_grad=True with the multistep solver {solver} (history)")
    cfg_mode = _cfg_mode(w_cfg, cond_emb)
    if cfg_mode is None or cfg_mode == 2:
        return _fallback("requires_grad=True with two-branch classifier-free guidance")
    if guided:
        return _fallback("requires_grad=True with classifier guidance")
    math = _math_mode()
    if math == cabi.MATH_BF16_TC:
        return _fallback("requires_grad=True with CDS_MATH=bf16 (fp32 and tf32 only)")
    batch, x_shape = xt.shape[0], tuple(xt.shape[1:])
    if n_samples != batch:
        return _fallback("n_samples != prior.shape[0]")

    table, n_slots, t_cpu, sched_key, order, _ = _step_table(
        agent, solver=solver, sample_steps=sample_steps, order=order, step_values=step_values, alphas=alphas, sigmas=sigmas,
        hs=hs, stds=stds, table=None, sched_id=sched_id)
    has_mask = isinstance(agent.fix_mask, torch.Tensor)
    has_min, has_max = agent.x_min is not None, agent.x_max is not None
    pn = bool(agent.predict_noise)
    tape_slots = min(n_slots, max(1, _tape_budget_bytes() // (4 * batch * x_shape[0]))) if n_slots > 0 else 0
    key = ("sde", id(net), batch, x_shape, len(order), tape_slots, cfg_mode, pn, has_mask, has_min, has_max, False, math, 0.0,
           "grad")

    def factory():
        plan = GradSamplerPlan(device, net, batch, x_shape, len(order), tape_slots, predict_noise=pn, has_mask=has_mask,
                               has_min=has_min, has_max=has_max, math=math)
        plan.build(1.0)
        return plan

    try:
        plan = _get_plan(agent, key, factory)
    except Unsupported as e:
        return _fallback(str(e))
    except cabi.CdsError as e:
        if e.code == -3:
            return _fallback(str(e))
        raise

    t_all = _load_resident(agent, plan, xt, prior, table, sched_key, tape_slots, n_slots, x_shape, order, t_cpu, device)
    lin1, fl = net.mid_layer[0], net.final_layer
    a, e = x_shape[0], net.time_mlp[2].out_features
    with torch.enable_grad():
        # the per-call tables with autograd: Linear over cat[x, time_mlp(map_noise(t)), obs] = W_x x + (W_t temb + b) + W_o obs
        step_tab = F.linear(net.time_mlp(net.map_noise(t_all)), lin1.weight[:, a:a + e], lin1.bias)
        if cfg_mode == 1:
            samp_tab = F.linear(_cond_rows(cfg_mode, cond_emb), lin1.weight[:, a + e:])
        else:
            samp_tab = torch.zeros((batch, lin1.out_features), device=device)
        noise_rows = (table[:, S.R_NOISE] > 0).tolist()
        run = lambda: plan.run_chunked(t_all, None, xt, noise_rows, use_graph=os.environ.get("CDS_GRAPH", "1") != "0")  # noqa: E731
        x0 = _GradSampleFn.apply(plan, run, step_tab, samp_tab, lin1.weight[:, :a], net.mid_layer[2].weight,
                                 net.mid_layer[2].bias, net.mid_layer[4].weight, net.mid_layer[4].bias, fl.weight, fl.bias)
    STATS["engine_calls"] += 1
    return x0


def engine_forward(net, x, t, cond_emb=None, math=None, use_graph=False):
    """Run ONLY the lowered denoiser once (no solver update): ``net(x, t.expand(b), cond_emb)`` on the engine.

    ``t`` is a 1-element tensor (int64 or float32): inside ``sample()`` the time is batch-constant.  Used by the
    parity tests and by profiling scripts; raises ``Unsupported`` if the backbone cannot be lowered."""
    device = x.device
    batch, x_shape = x.shape[0], tuple(x.shape[1:])
    p = Program(device, batch, 1, _math_mode() if math is None else math)
    xin = p.buf(batch, *x_shape)
    xin.copy_(x)
    L = x_shape[0] if len(x_shape) == 2 else 1
    pred = lower_denoiser(p, net, View(xin, L, x_shape[-1]), x_shape, cond_emb is not None, 0)
    handle = _make_handle(device, p.ops, 1)
    with torch.no_grad():
        ctx = _Ctx(t.reshape(1).to(device), None if cond_emb is None else cond_emb.to(torch.float32))
        for fn in p.per_call:
            fn(ctx)
    handle.run(0, 1, torch.cuda.current_stream(device).cuda_stream if device.type == "cuda" else 0, use_graph)
    out = pred.t.clone().reshape(batch, *x_shape)
    if device.type == "cuda":
        torch.cuda.synchronize(device)
    handle.close()
    return out
