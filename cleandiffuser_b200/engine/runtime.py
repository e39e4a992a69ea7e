"""Host runtime of the CUDA sampling engine: plan cache, schedule-table cache, per-call table fill, graph replay.

``try_sample`` is called by the ``sample()`` of every sampler family (``{Discrete,Continuous}DiffusionSDE``,
``ContinuousConsistencyModel``, ``ContinuousEDM``, RectifiedFlow, the legacy DDPM and EDM classes) after the prologue (initial
noise, mask, nn_condition) and replaces the whole Python reverse loop (diffusionsde.py:525-594) by

    tables  <- per-iteration solver coefficients (cached per schedule) + time-conditioning rows      (host, tiny)
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
import collections
import os
import types
from typing import Optional

import torch
import torch.nn.functional as F

from . import cabi
from .lower import (DQLGrad, Program, Unsupported, View, _rev, guidable, guide as emit_guide, lower_classifier_grad,
                    lower_denoiser)
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
    checkpoint loads of DiffusionModel -- writes through ``.data`` do not touch the version counters) or, for a classifier, its
    ``weights_epoch`` (bumped by ``ema_update`` and ``load``).  A classifier object without that counter (the reference's own
    classes) is fingerprinted by its version counters alone: after its ``update()`` / ``load()`` outside
    ``agent.update_classifier`` the packed copies are stale until the plan is rebuilt."""
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

    def __init__(self, t_all, cond_rows, cond_cg=None):
        # cond_cg: the classifier's per-trajectory condition (condition_cg), rows of this program's sub-batch
        self.t_all, self.cond_rows, self.cond_cg = t_all, cond_rows, cond_cg


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
                 has_min, has_max, keep_history, math, consistency=False, aux_history=False, classifier=None,
                 guide_operand=False):
        """classifier: a classifier ``lower.guidable`` accepts, whose input gradient at x_t enters the prediction between the
        denoiser and the update of every iteration (``pred += cg_scale[iter] * grad``); in a consistency program (ContinuousEDM)
        the gradient is instead the update's guidance operand, added to the denoised D inside the update.
        consistency: the EDM-preconditioned family (ContinuousConsistencyModel, ContinuousEDM): a CDS_OP_PREP in front of the
        denoiser (re-noise + c_in scaling) and the c_skip / c_out combine in the update; aux_history: second history buffer (the
        EDM Heun corrector needs the predictor's x_t and slope).  guide_operand: the update of a consistency program takes a
        guidance operand even without a lowered classifier -- ``cg_grad``, which a host callback fills every iteration."""
        self._resident(device, net, batch, x_shape, n_iters, n_slots, cfg_mode=cfg_mode, has_mask=has_mask, has_min=has_min,
                       has_max=has_max, keep_history=keep_history, aux_history=aux_history, math=math)
        self.classifier = classifier
        self._cg_fillers = set()          # ids of the lowered classifier's table fillers (they read the classifier's time column)
        row, root = self.row, self.program
        K = _n_branches(batch, row, consistency)
        self.n_branches = K
        if consistency:
            self.xin = root.buf(batch, *x_shape)

        L = x_shape[0] if len(x_shape) == 2 else 1
        Cn = x_shape[-1]
        sub = batch // K
        for k in range(K):
            off = k * sub                  # first trajectory of this branch
            sl = slice(off, off + sub)
            p = root if K == 1 else Program(device, sub * (2 if cfg_mode == 2 else 1), n_iters, math)
            n_before = len(p.ops)
            fo = 4 * off * row             # byte offset of the branch inside the (batch, row) fp32 buffers
            xin_ptr_t, xin_off = self.x, off * row
            if consistency:
                self._prep_op(p, sub, fo)
                xin_ptr_t = self.xin
            xview = View(xin_ptr_t, L, Cn, offset=xin_off)
            pred = lower_denoiser(p, net, xview, x_shape, cfg_mode != 0, sub if cfg_mode == 2 else 0)
            if K == 1:                 # the prediction buffer, for host callbacks between denoiser and update (guidance)
                self.pred = pred.t if (pred.offset == 0 and pred.lstride == pred.C and pred.bstride == pred.L * pred.C) else None
            grad = None
            if classifier is not None:
                assert K == 1 and cfg_mode != 2
                n_fill = len(p.per_call)
                # the classifier reads the raw x_t: in a consistency program the denoiser's input is CDS_OP_PREP's c_in x
                cx = View(self.x, L, Cn, offset=off * row) if consistency else _input_view(p, n_before, xview)
                grad = lower_classifier_grad(p, classifier, cx)
                self._cg_fillers = {id(fn) for fn in p.per_call[n_fill:]}
                self.cg_scale = root.buf(n_iters)           # per-iteration guidance scale, filled by every guided call
                if not consistency:
                    emit_guide(p, pred, grad, self.cg_scale)
            elif guide_operand:
                assert K == 1 and consistency
                self.cg_scale = root.buf(n_iters)
                self.cg_grad = root.buf(batch, *x_shape)    # written by the host callback of every iteration
                grad = View(self.cg_grad, L, Cn)

            u = self._update_op(p, pred.ptr, sub, fo, predict_noise, consistency)
            if consistency and grad is not None:            # ContinuousEDM: D += cg_scale[iter] * grad inside the update
                assert grad.offset == 0 and grad.lstride == grad.C and grad.bstride == grad.L * grad.C and grad.C * grad.L == row
                u.guide, u.guide_s = grad.ptr, self.cg_scale.data_ptr()
            # tensor-core UNets read x_t through a channel-padded bf16 copy (CDS_OP_CAST).  When that cast converts the very
            # buffer the update writes, the update emits the copy itself and the cast runs only once per sample() call.
            for cop in p.ops[n_before:]:
                if cop.kind == cabi.OP_CAST and cop.u.cast.in_ == self.x.data_ptr() + fo and cop.u.cast.batch == sub:
                    cop.flags |= cabi.OPF_ONCE
                    u.x_cast, u.cast_C_in, u.cast_C_out = cop.u.cast.out, cop.u.cast.C_in, cop.u.cast.C_out
                    u.x_cast_dtype = cop.u.cast.out_dtype
            self._fillers += [(fn, sl) for fn in p.per_call]
            if p is not root:
                for o in p.ops:
                    o.flags |= k << cabi.OPF_BRANCH_SHIFT
                root.ops += p.ops
                root.keep += p.keep + [p]
                root.packers += p.packers

    def _resident(self, device, net, batch, x_shape, n_iters, n_slots, *, cfg_mode, has_mask, has_min, has_max, keep_history,
                  aux_history, math):
        """The buffers every program of the plan shares (x_t, prior and mask, clip bounds, coefficient rows, noise tape, solver
        history), owned by the root program."""
        self.device, self.net, self.batch, self.x_shape = device, net, batch, tuple(x_shape)
        row = 1
        for s in x_shape:
            row *= s
        self.row, self.n_iters, self.cfg_mode = row, n_iters, cfg_mode
        root = Program(device, batch * (2 if cfg_mode == 2 else 1), n_iters, math)
        self.program, self.back = root, None             # back: the backward program of a differentiable plan
        self.classifier = None
        self.x = root.buf(batch, *x_shape)
        self.prior = root.buf(batch, *x_shape) if has_mask else None
        self.mask = root.buf(row) if has_mask else None
        self.x_min = root.buf(row) if has_min else None
        self.x_max = root.buf(row) if has_max else None
        self.coef = root.buf(n_iters, cabi.ROW_FLOATS)
        self.noise = root.buf(max(n_slots, 1), batch, row) if n_slots > 0 else None
        self.xhat_prev = root.buf(batch, row) if keep_history else None
        self.aux = root.buf(batch, row) if (keep_history and aux_history) else None
        self._update_ops = []
        self._fillers = []                 # (per-call table filler, sub-batch slice)
        self.handle: Optional[cabi.Plan] = None
        self.back_handle: Optional[cabi.Plan] = None
        self.version = None              # set by the first refresh_weights()

    def _prep_op(self, p, sub, fo):
        """Append the consistency model's re-noise and c_in scaling of ``sub`` trajectories at byte offset ``fo`` (x_t in place,
        the network's input into ``self.xin``) to ``p``."""
        op = cabi.Op()
        op.kind = cabi.OP_PREP
        q = op.u.prep
        q.batch, q.row, q.x, q.xin, q.coef = sub, self.row, self.x.data_ptr() + fo, self.xin.data_ptr() + fo, self.coef.data_ptr()
        q.noise = self.noise.data_ptr() if self.noise is not None else None
        p.ops.append(op)

    def _update_op(self, p, pred, sub, fo, predict_noise, consistency=False):
        """Append the solver update of ``sub`` trajectories at byte offset ``fo`` of the resident buffers to ``p`` (``pred``:
        address of their prediction, the unconditional half after it under two-branch CFG)."""
        op = cabi.Op()
        op.kind = cabi.OP_UPDATE
        u = op.u.update
        u.batch, u.row, u.x = sub, self.row, self.x.data_ptr() + fo
        u.pred = pred
        if self.cfg_mode == 2:
            u.pred_uncond = pred + 4 * sub * self.row
        if self.noise is not None:
            u.noise, u.noise_slot_stride = self.noise.data_ptr() + fo, self.batch * self.row
        u.prior = self.prior.data_ptr() + fo if self.prior is not None else None
        u.mask = self.mask.data_ptr() if self.mask is not None else None
        u.x_min = self.x_min.data_ptr() if self.x_min is not None else None
        u.x_max = self.x_max.data_ptr() if self.x_max is not None else None
        u.xhat_prev = self.xhat_prev.data_ptr() + fo if self.xhat_prev is not None else None
        u.aux = self.aux.data_ptr() + fo if self.aux is not None else None
        u.coef = self.coef.data_ptr()
        u.predict_noise = 1 if predict_noise else 0
        u.final_clip = 1 if consistency else 0
        self._update_ops.append(op)
        p.ops.append(op)
        return u

    def build(self, w_cfg: float):
        for op in self._update_ops:
            op.u.update.w_cfg, op.u.update.w_uncond = float(w_cfg), float(1 - w_cfg)
        self.w_cfg = w_cfg
        self.handle = _make_handle(self.device, self.program.ops, self.n_iters)
        if self.back is not None:
            self.back_handle = _make_handle(self.device, self.back.ops, self.n_iters)

    def refresh_weights(self, epoch: int = 0):
        v = _weights_version(self.net, epoch)
        if self.classifier is not None:
            v = _weights_version(self.classifier.model_ema, v * 1000003 + getattr(self.classifier, "weights_epoch", 0))
        if self.version is None:         # packed at construction
            self.version = v
        elif v != self.version:
            for prog in (self.program, self.back):
                if prog is not None:
                    for fn in prog.packers:
                        fn()
            self.version = v

    def close(self):
        for h in (self.handle, self.back_handle):
            if h is not None:
                h.close()
        self.handle = self.back_handle = None

    def fill_tables(self, t_all, cond_emb, t_key=None, cond_cg=None, cg_t=None):
        """Per-call tables (time-conditioning rows, per-trajectory condition terms of the denoiser and of a lowered
        classifier), once per ``sample()``.  ``cg_t``: the lowered classifier's time per iteration when it is not the
        denoiser's (ContinuousEDM: log(sigma) / 4 evaluated on the device; those tables are then refilled every call)."""
        # table fillers that depend on (weights, timesteps) only are skipped when neither changed since the last call
        fresh = t_key is None or (t_key, self.version) != getattr(self, "_time_tables_key", None)
        with torch.no_grad():
            for fn, sl in self._fillers:             # every branch fills its own tables from its slice of the condition
                own_t = cg_t is not None and id(fn) in self._cg_fillers
                if fresh or own_t or not getattr(fn, "time_only", False):
                    fn(_Ctx(cg_t if own_t else t_all, _cond_rows(self.cfg_mode, None if cond_emb is None else cond_emb[sl]),
                            None if cond_cg is None else cond_cg[sl]))
        self._time_tables_key = (t_key, self.version) if t_key is not None else None

    def run_guided(self, t_all, cond_emb, xt, noise_slots, guide, t_key=None, last_input=None):
        """The loop with a host callback between the denoiser and the update of every iteration (classifier guidance,
        diffusionsde.py:153-173): per iteration the denoiser operators are enqueued through the single-step entry
        (cds_plan_run_range), ``guide(n, x_t, out)`` works with ordinary PyTorch ops on the same stream, then the update operator
        runs.  ``out`` is the prediction, which the callback edits in place, or, when the update has a guidance operand
        (ContinuousEDM), that operand, into which the callback writes the classifier's gradient.  ``noise_slots[n]`` = 1 + tape
        slot of iteration n's draw, 0 = none.  ``last_input(x_t)``: called with the last iteration's input before it runs."""
        assert self.n_branches == 1 and self.pred is not None
        ops = self.program.ops
        upd = max(i for i, op in enumerate(ops) if op.kind == cabi.OP_UPDATE)
        assert upd == len(ops) - 1, "the update must be the program's last operator"
        self.fill_tables(t_all, cond_emb, t_key)
        stream = torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else 0
        x_view = self.x.view(self.batch, *self.x_shape)
        out_view = self.cg_grad if hasattr(self, "cg_grad") else self.pred.view(-1, *self.x_shape)[:self.batch]
        self.handle.run(0, 0, stream, False)                       # the CDS_OPF_ONCE operators (x_t hand-over cast)
        for n in range(self.n_iters):
            slot = int(noise_slots[n]) - 1
            if slot >= 0:
                with torch.no_grad():
                    _draw_noise(self.noise[slot], xt)
            if last_input is not None and n == self.n_iters - 1:
                last_input(x_view)
            self.handle.run_range(n, 0, upd, stream)
            guide(n, x_view, out_view)
            self.handle.run_range(n, upd, 1, stream)
        STATS["launches"] = (self.handle.launches_per_iter() + 2) * self.n_iters + 1

    def run_chunked(self, t_all, cond_emb, xt, noise_rows, t_key=None, cond_cg=None, cg_t=None, last_input=None):
        """The whole loop, with the noise tape refilled between chunks when it is shorter than the number of draws
        (``noise_rows[n]`` = does iteration n draw?).  The draws are taken in loop order, so a seeded run consumes the
        generator like the reference loop; everything is enqueued on one stream, so a refill cannot overtake its readers.
        ``last_input(x_t)``: called with the last iteration's input (the loop is then split before that iteration)."""
        cap = self.noise.shape[0] if self.noise is not None else 0
        split = self.n_iters - 1 if last_input is not None else None
        self.fill_tables(t_all, cond_emb, t_key, cond_cg, cg_t)
        stream = torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else 0
        use_graph = os.environ.get("CDS_GRAPH", "1") != "0"
        timed = STATS.get("time_loop") and self.device.type == "cuda"
        if timed:           # bench.py: device time of the reverse loop alone (noise draws + replayed iterations; events on the
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)    # launching stream)
            e0.record()
        first, used = 0, 0
        with torch.no_grad():
            for n in range(self.n_iters + 1):
                draws = n < self.n_iters and bool(noise_rows[n])
                if n == self.n_iters or (draws and used == cap) or n == split:
                    if n > first:
                        self.handle.run(first, n - first, stream, use_graph)
                    first = n
                    if n != split or (draws and used == cap):
                        used = 0
                    if n == split:
                        last_input(self.x.view(self.batch, *self.x_shape))
                if draws:
                    _draw_noise(self.noise[used], xt)
                    used += 1
        STATS["launches"] = self.handle.launches_per_iter() * self.n_iters + 1
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


def _screen(agent, xt, w_cfg, cond_emb, n_samples, decline=None):
    """The request screen of every entry point -> ``(device, cfg_mode)`` when the engine serves the call, else None: quietly
    under CDS_BACKEND=torch, on a device the engine does not serve and for a non-fp32 x_t (the caller's PyTorch loop runs), through
    ``_fallback`` for a request the engine declines -- the caller's own ``decline(cfg_mode)`` reason first."""
    if _backend() == "torch":
        return None
    device = _device_of(agent)
    if not _device_ok(device) or xt.dtype != torch.float32:
        return None
    cfg_mode = _cfg_mode(w_cfg, cond_emb)
    reason = decline(cfg_mode) if decline is not None else None
    if reason is None and cfg_mode is None:
        reason = "two-branch CFG without condition"
    if reason is None and n_samples != xt.shape[0]:
        reason = "n_samples != prior.shape[0]"
    return (device, cfg_mode) if reason is None else _fallback(reason)


def _get_plan(agent, key, factory):
    """Plan cache of one agent: least-recently-used order, at most CDS_MAX_PLANS entries (each pins device buffers).  A backbone
    the lowering declines (``Unsupported``) or an option set the library refuses (``CdsError`` -3) is a fallback -> None."""
    plans = agent._engine_plans
    plan = plans.pop(key, None)
    if plan is None:
        try:
            plan = factory()
        except Unsupported as e:
            return _fallback(str(e))
        except cabi.CdsError as e:
            if e.code == -3:
                return _fallback(str(e))
            raise
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


# One schedule of an agent's table cache: the coefficient rows (noise slots numbered 1, 2, ...), the number of noise slots, the
# time of every iteration on the device, and that column's bytes (``fill_tables`` skips the time-only fillers when they match).
_Table = collections.namedtuple("_Table", "rows n_slots t t_key")


def _schedule(agent, device, *, solver, sample_steps, order, step_values, alphas, sigmas, hs, stds, table, sched_id):
    """The coefficient table of one ``sample()`` call, from the agent's table cache (cleared once it passes 16 entries).

    ``table``: ``(rows, n_slots, time per iteration)``, or a zero-argument builder of it, or None for the SDE solvers (rows from
    ``alphas`` / ``sigmas`` / ``hs`` / ``stds`` / ``step_values``).  ``sched_id``: a hashable the caller vouches for --
    everything the table is a function of.  With it a hit skips the builder: no device->host read (each one a stream
    synchronisation, which would keep the host from preparing call n + 1 while call n runs; 1-step samplers spend a quarter of
    their wall time on the host), no per-step Python arithmetic (~10 ms for 100 SDE steps, more than a tenth of a cfg2
    sample() on the engine), no host->device copy.  Without one, or for a table given by value, the cache is keyed on what the
    table is built from."""
    key = ("id", sched_id)
    if table is None:                                  # the SDE solvers: the rows are a function of the schedule tensors
        if sched_id is None:
            key = ("content",) + tuple(z.detach().cpu().numpy().tobytes() for z in (step_values, alphas, sigmas, hs, stds))
        table = lambda: _step_table(solver, sample_steps, order, step_values, alphas, sigmas, hs, stds)    # noqa: E731
    elif sched_id is None or not callable(table):
        rows, n_slots, t = table() if callable(table) else table
        key, table = ("content", rows.numpy().tobytes(), t.detach().cpu().numpy().tobytes()), lambda: (rows, n_slots, t)
    key += (solver, sample_steps, tuple(order), str(device))
    cache = agent.__dict__.setdefault("_engine_tables", {})
    entry = cache.get(key)
    if entry is None:
        rows, n_slots, t = table()
        t = t.detach().cpu()
        entry = _Table(rows, int(n_slots), t.to(device), t.numpy().tobytes())
        if len(cache) > 16:
            cache.clear()
        cache[key] = entry
    return entry


def _step_table(solver, sample_steps, order, step_values, alphas, sigmas, hs, stds):
    """The SDE solvers' rows (per-iteration scalars on the host, reference op order) -> ``(rows, n_slots, time per iteration)``."""
    alphas, sigmas, hs, stds = (z.detach().float().cpu() for z in (alphas, sigmas, hs, stds))
    step_values = step_values.detach().cpu()
    table = S.coeff_table(solver, order, sample_steps, alphas, sigmas, hs, stds, step_values.double())
    n_slots = 0
    for n in range(len(order)):
        if table[n, S.R_NOISE] > 0:
            n_slots += 1
            table[n, S.R_NOISE] = float(n_slots)       # 1 + slot index
    return table, n_slots, step_values[torch.as_tensor(order, dtype=torch.long)]


def _tape_slots(n_slots, batch, row):
    """Noise tape: all draws of the loop up front when they fit CDS_NOISE_TAPE_MB (default 4096), else as many slots as fit (the
    loop then runs in chunks with the tape refilled in between -- O(budget) memory instead of O(sample_steps x batch x row))."""
    budget = int(float(os.environ.get("CDS_NOISE_TAPE_MB", "4096")) * (1 << 20))
    return min(n_slots, max(1, budget // (4 * batch * row))) if n_slots > 0 else 0


def _load_resident(agent, plan, xt, prior, tab: _Table, tape_slots):
    """Fill the plan's resident buffers: x_t, the coefficient rows (when the schedule changed), prior and mask, clip bounds."""
    with torch.no_grad():
        plan.x.copy_(xt)
        if getattr(plan, "_coef_of", None) is not tab:
            rows = tab.rows
            if tape_slots and tape_slots < tab.n_slots:      # slots are reused chunk by chunk: k-th draw -> slot k mod tape_slots
                rows = rows.clone()
                draws = rows[:, S.R_NOISE] > 0
                rows[draws, S.R_NOISE] = (rows[draws, S.R_NOISE] - 1) % tape_slots + 1
            plan.coef.copy_(rows)
            plan._coef_of = tab
        if plan.mask is not None:
            plan.prior.copy_(prior)
            plan.mask.copy_(_row(agent.fix_mask, plan.x_shape, plan.device))
        if plan.x_min is not None:
            plan.x_min.copy_(_row(agent.x_min, plan.x_shape, plan.device))
        if plan.x_max is not None:
            plan.x_max.copy_(_row(agent.x_max, plan.x_shape, plan.device))


def try_sample(agent, *, model, xt, prior, solver, sample_steps, order, step_values, alphas, sigmas, hs, stds,
               cond_emb, w_cfg, n_samples, guide=None, table=None, clip_in_loop=True, predict_noise=None, sched_id=None,
               classifier=None, w_cg=0.0, cond_cg=None, consistency=False, aux_history=False, cg_scale=None, cg_time=None,
               last_input=None):
    """One ``sample()`` call of any sampler family on the engine -> x0, or None when the caller's PyTorch loop must run.

    ``table``: the coefficient rows for samplers that are "the same update kernel with another coefficient table" (the legacy
    DDPM and EDM classes, RectifiedFlow's Euler step, ContinuousConsistencyModel, ContinuousEDM), see ``_schedule``;
    ``solver`` / ``alphas`` / ``sigmas`` / ``hs`` / ``stds`` / ``step_values`` then serve only as keys or are unused.
    ``clip_in_loop=False``: the sampler clips only its final sample (RectifiedFlow, legacy EDM); ``predict_noise``: overrides
    ``agent.predict_noise`` (classes without that attribute).  ``consistency``: the EDM-preconditioned family (CDS_OP_PREP in
    front of the denoiser, c_skip / c_out combine and final clip in the update); ``aux_history``: the EDM Heun corrector's
    history buffers.
    ``guide``: optional host callback ``guide(n, i, x_t, pred)`` (n = iteration, i = its loop index) run between the denoiser
    and the update of every iteration (classifier guidance); the loop then runs step by step instead of as a replayed graph --
    unless ``classifier`` (the one ``guide`` evaluates, with weight ``w_cg`` and condition ``cond_cg``) is one ``lower.guidable``
    accepts (a CumRewClassifier over HalfJannerUNet1d or an out_dim-1 MLPNNClassifier, an MSEClassifier over MLPNNClassifier
    or a QGPOClassifier over QGPONNClassifier with a condition) under
    CDS_MATH = fp32 | tf32 with one sub-batch chain: its input gradient and the guidance term are then operators of the replayed
    program, and ``guide`` is not called.
    A guided table-driven family gives its own guidance terms: ``cg_scale``, the per-iteration scale on the device (the SDE
    classes' is derived from ``sigmas`` / ``alphas``); ``cg_time``, the classifier's time per iteration when it is not the
    table's time column.  In a consistency program (ContinuousEDM) the guidance term enters the update as its guidance
    operand, and ``guide(n, i, x_t, g)`` writes the classifier's gradient into ``g`` instead of editing the prediction.
    ``last_input(x_t)``: called with the input of the last iteration before it runs (the legacy DDPM's log p)."""
    def decline(cfg_mode):
        if guide is not None and cfg_mode == 2:
            # the update operator combines the two CFG branches itself; a guidance term would have to enter after that combine
            return "classifier guidance together with two-branch classifier-free guidance"
        return None
    screened = _screen(agent, xt, w_cfg, cond_emb, n_samples, decline)
    if screened is None:
        return None
    device, cfg_mode = screened
    net = model["diffusion"]
    batch, x_shape = xt.shape[0], tuple(xt.shape[1:])
    keep_history = aux_history or (table is None and S.solver_keeps_history(solver))     # multistep SDE solvers, EDM Heun
    tab = _schedule(agent, device, solver=solver, sample_steps=sample_steps, order=order, step_values=step_values, alphas=alphas,
                    sigmas=sigmas, hs=hs, stds=stds, table=table, sched_id=sched_id)
    n_iters = tab.rows.shape[0]
    has_mask = isinstance(agent.fix_mask, torch.Tensor)
    has_min = clip_in_loop and getattr(agent, "x_min", None) is not None
    has_max = clip_in_loop and getattr(agent, "x_max", None) is not None
    pn = bool(agent.predict_noise) if predict_noise is None else bool(predict_noise)
    math = _math_mode()
    row_elems = 1
    for s_ in x_shape:
        row_elems *= s_
    cg_reason = None                       # why a guided call keeps the host callback (None: the graph serves it)
    if guide is not None:
        cg_reason = "no classifier" if classifier is None else guidable(classifier, x_shape, cond_cg)
        if cg_reason is None and cond_cg is not None and cond_cg.shape[0] != batch:
            cg_reason = "classifier condition rows != batch"
        if cg_reason is None and math == cabi.MATH_BF16_TC:
            cg_reason = "CDS_MATH=bf16"
        if cg_reason is None and _n_branches(batch, row_elems, False) != 1:
            cg_reason = "more than one sub-batch chain (CDS_BRANCHES)"
    lowered_cg = guide is not None and cg_reason is None
    operand = guide is not None and consistency and not lowered_cg      # the EDM callback writes the update's guidance operand
    tape_slots = _tape_slots(tab.n_slots, batch, row_elems)
    key = (id(net), batch, x_shape, n_iters, tape_slots, cfg_mode, pn, has_mask, has_min, has_max, keep_history, aux_history,
           consistency, math, float(w_cfg) if cfg_mode == 2 else 0.0,
           id(classifier.model_ema) if lowered_cg else ("operand" if operand else None))

    def factory():
        plan = SamplerPlan(device, net, batch, x_shape, n_iters, tape_slots, cfg_mode=cfg_mode, predict_noise=pn,
                           has_mask=has_mask, has_min=has_min, has_max=has_max, keep_history=keep_history, math=math,
                           consistency=consistency, aux_history=aux_history, classifier=classifier if lowered_cg else None,
                           guide_operand=operand)
        plan.build(w_cfg)
        return plan

    plan = _get_plan(agent, key, factory)
    if plan is None:
        return None
    _load_resident(agent, plan, xt, prior, tab, tape_slots)
    STATS["guidance_path"], STATS["guidance_reason"] = None, cg_reason
    if lowered_cg or operand:
        # the guidance scale of every iteration, the reference's own expression (classifier_guidance), evaluated on the device
        with torch.no_grad():
            if cg_scale is None:
                idx = torch.as_tensor(order, dtype=torch.long).to(device)
                sig = sigmas.to(device)[idx]
                cg_scale = -(w_cg * sig) if pn else w_cg * ((sig ** 2) / alphas.to(device)[idx])
            plan.cg_scale.copy_(cg_scale)
    if lowered_cg:
        STATS["guidance_path"] = "graph"
        guide = None
    if guide is not None:
        STATS["guidance_path"] = "callback"
        if plan.n_branches != 1 or getattr(plan, "pred", None) is None:
            return _fallback("guided sampling needs a single-branch program with a dense prediction buffer")
        slots = plan.coef[:, S.R_NOISE].cpu().tolist()              # tape slot per iteration as the update kernel sees it
        plan.run_guided(tab.t, cond_emb, xt, slots, lambda n, x, p: guide(n, order[n], x, p), t_key=tab.t_key,
                        last_input=last_input)
    else:
        # the loop's draws: same calls, same order, same shapes as the reference loop's (diffusionsde.py:548,571,...)
        plan.run_chunked(tab.t, cond_emb, xt, (tab.rows[:, S.R_NOISE] > 0).tolist(), t_key=tab.t_key,
                         cond_cg=cond_cg if lowered_cg else None, cg_t=cg_time if lowered_cg else None,
                         last_input=last_input)
    STATS["engine_calls"] += 1
    return plan.x.clone()


# ============================================================================ differentiable sampling (requires_grad=True)
class GradSamplerPlan(SamplerPlan):
    """The resident state of ``sample(requires_grad=True)`` over DQLMlp: a forward program (``lower.DQLGrad``'s network
    operators, which stash x_n, the hidden pre-activations and the raw prediction of every iteration, then the solver update)
    and a backward program that walks the iterations in reverse.  Each is one cds_plan replayed from a CUDA graph.  One branch,
    no CFG combine, no solver history.

    consistency: the consistency model's program -- a CDS_OP_PREP (re-noise, c_in scaling) in front of the network, the CM
    combine with its final clip in the update, and at the end of every backward iteration the PREP's backward mode, which adds
    c_in * d xin to the direct part of d x_n.  Rectified flow needs nothing of its own: its Euler step is the EPS update."""

    def __init__(self, device, net, batch, x_shape, n_iters, n_slots, *, predict_noise, has_mask, has_min, has_max, math,
                 consistency=False):
        self._resident(device, net, batch, x_shape, n_iters, n_slots, cfg_mode=1, has_mask=has_mask, has_min=has_min,
                       has_max=has_max, keep_history=False, aux_history=False, math=math)
        self.n_branches, row = 1, self.row
        self.back = back = Program(device, batch, n_iters, math)
        xin = None
        if consistency:
            self.xin = self.program.buf(batch, *x_shape)
            self._prep_op(self.program, batch, 0)
            xin = View(self.xin, 1, row)
        self.grad = g = DQLGrad(self.program, back, net, View(self.x, 1, row), xin)
        self.pred = g.pred.t
        u = self._update_op(self.program, g.pred.ptr, batch, 0, predict_noise, consistency)

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
        if consistency:                                      # gx += c_in * d xin closes every backward iteration
            pop = cabi.Op()
            pop.kind = cabi.OP_PREP
            q = pop.u.prep
            q.batch, q.row, q.x, q.gxin = batch, row, g.gx.data_ptr(), g.gxin.data_ptr()
            q.coef, q.coef_iter_stride = _rev(self.coef)
            back.ops.append(pop)
        self.generation = 0                # forward runs so far: a backward must belong to the latest one

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


def guidance_declined(agent, reason):
    """A guided ``sample()`` that keeps its PyTorch loop (ContinuousEDM and the legacy DDPM under two-branch CFG,
    ``requires_grad=True`` or ``preserve_history=True``): recorded in ``STATS["guidance_reason"]`` on a device the engine
    serves, without counting a fallback."""
    if _backend() != "torch" and _device_ok(_device_of(agent)):
        STATS["guidance_path"], STATS["guidance_reason"] = None, reason


def grad_fallback(agent):
    """``requires_grad=True`` on a sampler class that has no differentiable engine program: recorded (raised under
    CDS_BACKEND=cuda) like every other fallback; the caller then runs its PyTorch loop, which autograd differentiates."""
    if _backend() != "torch" and _device_ok(_device_of(agent)):
        return _fallback(f"requires_grad=True: {type(agent).__name__} has no differentiable engine program")
    return None


# the update kinds CDS_OP_UPDATE_BWD differentiates (csrc/grad.cuh): a table with any other kind keeps the PyTorch loop
_GRAD_KINDS = frozenset((S.UPD_DDPM, S.UPD_DDIM, S.UPD_EPS, S.UPD_X, S.UPD_CM))


def try_sample_grad(agent, *, model, xt, prior, solver, sample_steps, order, step_values, alphas, sigmas, hs, stds,
                    cond_emb, w_cfg, n_samples, guided=False, table=None, clip_in_loop=True, predict_noise=None, sched_id=None,
                    consistency=False):
    """``sample(requires_grad=True)`` on the engine: x0 connected to autograd through ``_GradSampleFn``.  Covers DQLMlp with
    one CFG branch and CDS_MATH = fp32 | tf32 under the DDPM / DDIM / first-order DPM-Solver updates, ContinuousConsistencyModel
    (``consistency``) and RectifiedFlow's Euler step; everything else takes the PyTorch loop (which autograd differentiates)
    through ``_fallback``.  ``table`` / ``clip_in_loop`` / ``predict_noise`` / ``sched_id`` / ``consistency``: as in
    ``try_sample``; the table's time column is what the network sees (c_noise for the consistency model)."""
    net = model["diffusion"]

    def decline(cfg_mode):
        name = type(net).__name__
        if name != "DQLMlp" or xt.dim() != 2:
            return f"requires_grad=True: backbone {name} has no differentiable engine program (DQLMlp only)"
        if S.solver_keeps_history(solver):
            return f"requires_grad=True with the multistep solver {solver} (history)"
        if cfg_mode is None or cfg_mode == 2:
            return "requires_grad=True with two-branch classifier-free guidance"
        if guided:
            return "requires_grad=True with classifier guidance"
        if _math_mode() == cabi.MATH_BF16_TC:
            return "requires_grad=True with CDS_MATH=bf16 (fp32 and tf32 only)"
        return None
    screened = _screen(agent, xt, w_cfg, cond_emb, n_samples, decline)
    if screened is None:
        return None
    device, cfg_mode = screened
    batch, x_shape = xt.shape[0], tuple(xt.shape[1:])
    tab = _schedule(agent, device, solver=solver, sample_steps=sample_steps, order=order, step_values=step_values, alphas=alphas,
                    sigmas=sigmas, hs=hs, stds=stds, table=table, sched_id=sched_id)
    kinds = {int(k) for k in tab.rows[:, S.R_KIND].tolist()} - _GRAD_KINDS
    if kinds:
        return _fallback(f"requires_grad=True: update kind {sorted(kinds)} has no backward operator")
    n_iters = tab.rows.shape[0]
    has_mask = isinstance(agent.fix_mask, torch.Tensor)
    has_min = clip_in_loop and getattr(agent, "x_min", None) is not None
    has_max = clip_in_loop and getattr(agent, "x_max", None) is not None
    pn = bool(agent.predict_noise) if predict_noise is None else bool(predict_noise)
    math = _math_mode()
    tape_slots = _tape_slots(tab.n_slots, batch, x_shape[0])
    key = (id(net), batch, x_shape, n_iters, tape_slots, cfg_mode, pn, has_mask, has_min, has_max, False, False,
           bool(consistency), math, 0.0, None, "grad")

    def factory():
        plan = GradSamplerPlan(device, net, batch, x_shape, n_iters, tape_slots, predict_noise=pn, has_mask=has_mask,
                               has_min=has_min, has_max=has_max, math=math, consistency=consistency)
        plan.build(1.0)
        return plan

    plan = _get_plan(agent, key, factory)
    if plan is None:
        return None
    _load_resident(agent, plan, xt, prior, tab, tape_slots)
    lin1, fl = net.mid_layer[0], net.final_layer
    a, e = x_shape[0], net.time_mlp[2].out_features
    with torch.enable_grad():
        # the per-call tables with autograd: Linear over cat[x, time_mlp(map_noise(t)), obs] = W_x x + (W_t temb + b) + W_o obs
        step_tab = F.linear(net.time_mlp(net.map_noise(tab.t)), lin1.weight[:, a:a + e], lin1.bias)
        if cfg_mode == 1:
            samp_tab = F.linear(_cond_rows(cfg_mode, cond_emb), lin1.weight[:, a + e:])
        else:
            samp_tab = torch.zeros((batch, lin1.out_features), device=device)
        noise_rows = (tab.rows[:, S.R_NOISE] > 0).tolist()
        run = lambda: plan.run_chunked(tab.t, None, xt, noise_rows)  # noqa: E731
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
