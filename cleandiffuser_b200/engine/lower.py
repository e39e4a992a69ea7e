"""Lower a denoiser ``nn.Module`` to the fused-operator program libcds executes.

The module tree (same names/shapes as the reference's, so user checkpoints load) is walked once per
(model, batch, option set); the result is a ``Program``:

* ``ops``        -- ``cabi.Op`` list for ONE reverse iteration (denoiser + solver update)
* ``packers``    -- re-run when parameter versions change (training mutates weights between calls):
                    copy/transpose parameters into the K-major layouts the kernels read
* ``per_call``   -- run at every ``sample()``: fill the per-iteration tables (time-conditioning rows evaluated
                    with the model's OWN ``map_noise`` / ``map_emb`` / ``emb_mlp`` modules on one row per
                    iteration -- inside ``sample()`` t is batch-constant, diffusionsde.py:528/:874 -- and the
                    per-trajectory condition terms)
* ``keep``       -- every device tensor the ops point into (workspace, packed weights, tables)

What is hoisted out of the iteration loop (SURVEY 8a quirk 5):
  JannerUNet1d w/o condition : the whole map_noise -> map_emb -> emb_mlp chain is a [n_iters, sum C_out] table.
  ChiUNet1d                  : cond_encoder = Linear(Mish(cat[time, obs])) splits exactly into a per-iteration
                               row plus a per-trajectory, iteration-invariant row (Mish is elementwise).
  DQLMlp                     : the first Linear over cat[x, time_mlp(t), obs] splits the same way.
  DiT1d / Janner + condition : map_emb(map_noise(t) + cond) is nonlinear in the sum -> small per-trajectory
                               GEMMs stay inside the iteration (0.5 % of the FLOPs).
  ChiTransformer             : the cross-attention memory is encoder(token + position) per token: token 0 (the time) depends
                               on the iteration only, tokens 1..To (the observations) on the trajectory only -> every layer's
                               cross-attention keys / values are a per-iteration table plus a per-trajectory table.
"""
import ctypes as C
from typing import Callable, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import cabi


class Unsupported(Exception):
    """The module / option set is outside what the kernels cover -> caller uses the PyTorch path."""


class View:
    """A channels-last activation: element (b, l, c) at base + b*bstride + l*lstride + c (elements of its dtype)."""

    def __init__(self, tensor: torch.Tensor, L: int, Cn: int, offset: int = 0, bstride: Optional[int] = None,
                 lstride: Optional[int] = None, tf32: bool = False):
        assert tensor.dtype in (torch.float32, torch.bfloat16)
        # tf32: fp32 storage that feeds a TF32 tensor-core operator -> producers round to TF32 when they write it (cds_dtype
        # CDS_TF32); readers treat it as fp32
        self.tf32 = bool(tf32) and tensor.dtype == torch.float32
        # module dims may be numpy ints (np.cumprod(dim_mult)); ctypes wants python ints
        self.t, self.L, self.C, self.offset = tensor, int(L), int(Cn), int(offset)
        self.lstride = self.C if lstride is None else int(lstride)
        self.bstride = self.L * self.lstride if bstride is None else int(bstride)

    @property
    def ptr(self):
        return self.t.data_ptr() + self.t.element_size() * self.offset

    @property
    def dtype(self):
        return cabi.BF16 if self.t.dtype == torch.bfloat16 else (cabi.TF32 if self.tf32 else cabi.F32)

    def channels(self, start: int, count: int) -> "View":
        return View(self.t, self.L, count, self.offset + int(start), self.bstride, self.lstride, self.tf32)


def _vec(step: Optional[torch.Tensor] = None, sample: Optional[torch.Tensor] = None, col: int = 0) -> cabi.Vec:
    """step: [n_iters, W] table, sample: [rows, W] table; the vector is columns col.. of both."""
    v = cabi.Vec()
    col = int(col)
    if step is not None:
        v.step, v.step_stride = step.data_ptr() + 4 * col, step.stride(0)
    if sample is not None:
        v.sample, v.sample_stride = sample.data_ptr() + 4 * col, sample.stride(0)
    return v


def _const_vec(t: Optional[torch.Tensor]) -> cabi.Vec:
    v = cabi.Vec()
    if t is not None:
        v.step, v.step_stride = t.data_ptr(), 0
    return v


class WSpec:
    """Where a GEMM weight comes from; packed lazily in the layout of the kernel that ends up running the op.

    kn() -> fp32 [K = taps*C_in, N = C_out*phases]   (CUDA-core kernel: K rows, N contiguous)
    nk() -> [taps, C_out, C_in]                      (tensor-core kernel: K contiguous; cast to bf16 / rounded to TF32), or None"""

    def __init__(self, kn: Callable[[], torch.Tensor], nk: Optional[Callable[[], torch.Tensor]] = None):
        self.kn, self.nk = kn, nk


def _pad_cin(w: torch.Tensor, cin: Optional[int]) -> torch.Tensor:
    """Zero-pad dim 1 (input channels) of a [Cout, Cin, ...] weight up to ``cin`` (x_t is fed 32-channel padded)."""
    if cin is None or cin == w.shape[1]:
        return w
    out = torch.zeros((w.shape[0], cin, *w.shape[2:]), device=w.device, dtype=w.dtype)
    out[:, :w.shape[1]] = w
    return out


def w_conv(conv: nn.Conv1d, cin: Optional[int] = None) -> WSpec:           # [Cout, Cin, k]
    return WSpec(lambda: _pad_cin(conv.weight, cin).permute(2, 1, 0).reshape(-1, conv.weight.shape[0]),
                 lambda: _pad_cin(conv.weight, cin).permute(2, 0, 1))


def w_linear(weight: torch.Tensor, cols: Optional[slice] = None) -> WSpec:    # [out, in]
    pick = (lambda: weight) if cols is None else (lambda: weight[:, cols])
    return WSpec(lambda: pick().t(), lambda: pick()[None])


def w_rows(make_out_in: Callable[[], torch.Tensor]) -> WSpec:                 # callable -> [out, in]
    return WSpec(lambda: make_out_in().t(), lambda: make_out_in()[None])


def w_convT(conv: nn.ConvTranspose1d) -> WSpec:
    """ConvTranspose1d(k=4, s=2, p=1) as a 3-tap conv with two output phases:
    out[2m]   = x[m-1] W[..,3] + x[m] W[..,1]        out[2m+1] = x[m] W[..,2] + x[m+1] W[..,0]"""
    def make():
        w = conv.weight                                      # [Cin, Cout, 4]
        cin, cout, _ = w.shape
        p = torch.zeros(3, cin, 2 * cout, device=w.device, dtype=w.dtype)
        p[0, :, :cout] = w[:, :, 3]
        p[1, :, :cout] = w[:, :, 1]
        p[1, :, cout:] = w[:, :, 2]
        p[2, :, cout:] = w[:, :, 0]
        return p.reshape(3 * cin, 2 * cout)

    def make_nk():                                           # [3][2*Cout][Cin]
        return make().reshape(3, conv.weight.shape[0], -1).permute(0, 2, 1)
    return WSpec(make, make_nk)


def round_tf32(w: torch.Tensor) -> torch.Tensor:
    """fp32 -> nearest TF32-representable fp32 (10-bit mantissa, ties away from zero like cvt.rna.tf32.f32).  wgmma
    .tf32 ignores the low 13 mantissa bits of its operands, i.e. truncates; weights are rounded once here so that
    their part of the error is unbiased."""
    bits = w.detach().to(torch.float32).contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


class Program:
    def __init__(self, device: torch.device, rows: int, n_iters: int, math: int = cabi.MATH_FP32):
        self.device, self.rows, self.n_iters, self.math = device, rows, n_iters, math
        self.ops: List[cabi.Op] = []
        self.keep: List[torch.Tensor] = []
        self.packers: List[Callable[[], None]] = []
        self.per_call: List[Callable[[object], None]] = []

    # ---- memory ---------------------------------------------------------------------------
    def buf(self, *shape, dtype=torch.float32) -> torch.Tensor:
        t = torch.zeros(tuple(int(s) for s in shape), device=self.device, dtype=dtype)
        self.keep.append(t)
        return t

    @property
    def act_dtype(self):
        """Intermediate activations: bf16 on CDS_MATH_BF16_TC programs, fp32 otherwise (CUDA-core and TF32 programs)."""
        return torch.bfloat16 if self.math == cabi.MATH_BF16_TC else torch.float32

    @property
    def tc(self) -> bool:
        """Does this program ask for the tensor-core kernels?"""
        return self.math in cabi.TC_MODES

    @property
    def k_align(self) -> int:
        """Channel granularity of a tensor-core operand row (64 bytes): what x_t is padded to."""
        return 16 if self.math == cabi.MATH_TF32_TC else 32

    def act(self, L: int, Cn: int, dtype=None) -> View:
        """A (rows, L, Cn) activation.  Without an explicit dtype it is an inter-layer activation in the program's activation
        type (bf16 / TF32-rounded fp32 / fp32); an explicit torch.float32 is kept exact (predictions, DiT's residual stream)."""
        return View(self.buf(self.rows, L, Cn, dtype=self.act_dtype if dtype is None else dtype), L, Cn,
                    tf32=dtype is None and self.math == cabi.MATH_TF32_TC)

    def packed(self, make: Callable[[], torch.Tensor], dtype=torch.float32) -> torch.Tensor:
        """Persistent packed copy of parameters; ``make`` is re-evaluated into it when weights change."""
        with torch.no_grad():
            t = make().detach().to(device=self.device, dtype=dtype).contiguous().clone()
        self.keep.append(t)

        def refresh():
            with torch.no_grad():
                t.copy_(make())
        self.packers.append(refresh)
        return t

    # ---- operator emitters --------------------------------------------------------------------
    def conv(self, x: View, w: WSpec, out: View, *, taps=1, stride=1, pad=0, phases=1, L_out=None,
             bias: Optional[cabi.Vec] = None, gn: Optional[nn.Module] = None, act=cabi.ACT_NONE,
             scale: Optional[cabi.Vec] = None, shift: Optional[cabi.Vec] = None, res: Optional[View] = None,
             res_conv=None, in_batch_mod=0, res_batch_mod=0, rows=None, sample_row_div=0):
        """Emit one CDS_OP_CONV.  ``res_conv`` = (View, WSpec of the 1x1 weight, bias tensor maker)."""
        op = cabi.Op()
        op.kind = cabi.OP_CONV
        c = op.u.conv
        c.batch = self.rows if rows is None else rows
        c.L_in, c.L_out = x.L, int(out.L // phases if L_out is None else L_out)
        c.C_in, c.C_out = x.C, out.C
        c.taps, c.stride, c.pad, c.phases = int(taps), int(stride), int(pad), int(phases)
        c.in_batch_mod = int(in_batch_mod)
        c.sample_row_div = int(sample_row_div)
        c.in_, c.in_bstride, c.in_lstride, c.in_dtype = x.ptr, x.bstride, x.lstride, x.dtype
        if bias is not None:
            c.bias = bias
        if gn is not None:
            gamma, beta = self.packed(lambda: gn.weight), self.packed(lambda: gn.bias)
            c.groups, c.gn_gamma, c.gn_beta, c.gn_eps = int(gn.num_groups), gamma.data_ptr(), beta.data_ptr(), gn.eps
        c.act = act
        if scale is not None:
            c.scale = scale
        if shift is not None:
            c.shift = shift
        if res is not None:
            c.res, c.res_bstride, c.res_lstride, c.res_dtype = res.ptr, res.bstride, res.lstride, res.dtype
        c.res_batch_mod = int(res_batch_mod)
        if res_conv is not None:
            rx = res_conv[0]
            c.res_in, c.res_in_bstride, c.res_in_lstride, c.res_C = rx.ptr, rx.bstride, rx.lstride, rx.C
            c.res_in_dtype = rx.dtype
            c.res_w = 1          # placeholder so that eligibility sees a shortcut conv; real pointer set below
        c.out, c.out_bstride, c.out_lstride, c.out_dtype = out.ptr, out.bstride, out.lstride, out.dtype

        # kernel family: tensor cores when the program asks for them AND this op qualifies, else CUDA cores
        use_tc = False
        if self.tc and w.nk is not None and (res_conv is None or res_conv[1].nk is not None):
            c.math = self.math
            use_tc = bool(cabi.load().cds_conv_tc_supported(C.byref(c)))
        c.math = self.math if use_tc else cabi.MATH_FP32
        tf32 = self.math == cabi.MATH_TF32_TC
        wdt = torch.float32 if tf32 else torch.bfloat16            # tensor-core weight element
        wfix = round_tf32 if tf32 else (lambda t: t)
        if use_tc:
            wt = self.packed(lambda: wfix(w.nk().reshape(taps * out.C * phases, x.C)), wdt)
        else:
            wt = self.packed(w.kn)
            assert wt.shape == (taps * x.C, out.C * phases), (wt.shape, taps, x.C, out.C, phases)
        c.w = wt.data_ptr()
        if res_conv is not None:
            rw = res_conv[1]
            rwt = self.packed(lambda: wfix(rw.nk().reshape(out.C, rx.C)), wdt) if use_tc else self.packed(rw.kn)
            c.res_w, c.res_bias = rwt.data_ptr(), self.packed(res_conv[2]).data_ptr()
        self.ops.append(op)
        return out

    def token_linear(self, x: View, w: WSpec, out: View, **kw):
        """Linear layer over a dense token stream (rows, L, C): on tensor-core programs the tokens are flattened to rows*L
        length-1 sequences (any L, e.g. DiT1d's 100), per-trajectory vectors follow through ``sample_row_div = L`` and a
        residual stream is flattened alongside; if the flattened operator is not tensor-core material it is emitted as is."""
        L = x.L
        dense = (x.lstride == x.C and x.bstride == L * x.C and out.lstride == out.C and out.bstride == L * out.C)
        res = kw.get("res")
        res_period = 0                       # > 0: the residual repeats every L rows (a (L, C) table broadcast over the batch)
        if res is not None:
            if res.bstride == 0 and res.lstride == res.C:
                res_period = L
            else:
                dense = dense and res.lstride == res.C and res.bstride == L * res.C
        if self.tc and dense and x.t.dtype == self.act_dtype and w.nk is not None and kw.get("res_conv") is None:
            flat = lambda v: View(v.t, 1, v.C, v.offset, v.C, v.C, v.tf32)
            probe = cabi.Op()
            c = probe.u.conv
            c.batch, c.L_in, c.L_out, c.C_in, c.C_out, c.taps, c.stride, c.pad, c.phases = self.rows * L, 1, 1, x.C, out.C, 1, 1, 0, 1
            c.in_, c.in_bstride, c.in_lstride, c.in_dtype = x.ptr, x.C, x.C, x.dtype
            c.out, c.out_bstride, c.out_lstride, c.out_dtype = out.ptr, out.C, out.C, out.dtype
            c.act = kw.get("act", cabi.ACT_NONE)
            c.sample_row_div = L
            c.in_batch_mod = int(kw.get("in_batch_mod", 0)) * L
            c.math = self.math
            if res is not None:
                c.res, c.res_bstride, c.res_lstride, c.res_dtype = res.ptr, res.C, res.C, res.dtype
                c.res_batch_mod = res_period
            if cabi.load().cds_conv_tc_supported(C.byref(c)):
                kw2 = dict(kw)
                kw2["in_batch_mod"] = c.in_batch_mod
                if res is not None:
                    kw2["res"] = flat(res)
                    kw2["res_batch_mod"] = res_period
                return self.conv(flat(x), w, flat(out), rows=self.rows * L, sample_row_div=L, **kw2)
        return self.conv(x, w, out, **kw)

    def cast_pad(self, x: View, width: int, rows: Optional[int] = None) -> View:
        """fp32 dense (rows, L, C) -> dense (rows, L, width) of the program's activation dtype with zero channels appended
        (rows: of the VIEW, which may be a sub-batch of its tensor)."""
        assert x.t.dtype == torch.float32 and x.lstride == x.C and x.bstride == x.L * x.C
        rows = x.t.shape[0] if rows is None else int(rows)
        out = View(self.buf(rows, x.L, width, dtype=self.act_dtype), x.L, width, tf32=self.math == cabi.MATH_TF32_TC)
        op = cabi.Op()
        op.kind = cabi.OP_CAST
        k = op.u.cast
        k.batch, k.L, k.C_in, k.C_out, k.in_, k.out, k.out_dtype = rows, x.L, x.C, int(width), x.ptr, out.ptr, out.dtype
        self.ops.append(op)
        return out

    def lnmod(self, x: View, out: View, mod: torch.Tensor, shift_col: int, scale_col: int, eps: float):
        op = cabi.Op()
        op.kind = cabi.OP_LNMOD
        m = op.u.lnmod
        m.batch, m.L, m.C, m.eps = self.rows, x.L, x.C, eps
        m.in_, m.out, m.out_dtype = x.ptr, out.ptr, out.dtype
        m.shift, m.scale = mod.data_ptr() + 4 * int(shift_col), mod.data_ptr() + 4 * int(scale_col)
        m.mod_bstride = mod.stride(0)
        self.ops.append(op)

    def mha(self, q: View, kv_step: Optional[View], kv_sample: Optional[View], out: View, heads: int,
            diag: Optional[int] = None):
        """CDS_OP_MHA.  kv_step: (n_iters, Lk, 2C) view (bstride = the iteration stride), kv_sample: (rows, Lk, 2C) view, either
        may be None; diag: key j is visible to query i iff j <= i + diag, None = no mask."""
        kv = kv_sample if kv_sample is not None else kv_step
        op = cabi.Op()
        op.kind = cabi.OP_MHA
        m = op.u.mha
        m.batch, m.Lq, m.Lk, m.C, m.heads = self.rows, q.L, kv.L, q.C, int(heads)
        m.masked, m.diag = (0, 0) if diag is None else (1, int(diag))
        m.q, m.q_bstride, m.q_lstride = q.ptr, q.bstride, q.lstride
        if kv_step is not None:
            m.kv_step, m.kv_step_stride, m.kv_step_lstride = kv_step.ptr, kv_step.bstride, kv_step.lstride
        if kv_sample is not None:
            m.kv_sample, m.kv_sample_bstride, m.kv_sample_lstride = kv_sample.ptr, kv_sample.bstride, kv_sample.lstride
        m.out, m.out_bstride, m.out_lstride = out.ptr, out.bstride, out.lstride
        m.in_dtype, m.out_dtype = q.dtype, out.dtype
        self.ops.append(op)

    def attn(self, qkv: View, out: View, heads: int):
        op = cabi.Op()
        op.kind = cabi.OP_ATTN
        a = op.u.attn
        a.batch, a.L, a.C, a.heads = self.rows, out.L, out.C, int(heads)
        a.qkv, a.out, a.out_dtype, a.qkv_dtype = qkv.ptr, out.ptr, out.dtype, qkv.dtype
        self.ops.append(op)


# =============================================================================== UNets
def _is_groupnorm(m) -> bool:
    """GroupNorm1d recognised structurally (class name + the attributes the kernels need), so that modules built from the
    reference's own classes (cleandiffuser/utils/building_blocks.py:60-76) lower exactly like this package's."""
    return (type(m).__name__ in ("GroupNorm1d", "GroupNorm") and hasattr(m, "num_groups") and hasattr(m, "eps")
            and isinstance(getattr(m, "weight", None), torch.Tensor) and isinstance(getattr(m, "bias", None), torch.Tensor))


def _lower_conv_block(p: Program, seq: nn.Sequential, x: View, out: View, k: int, **kw):
    """Conv1d -> GroupNorm1d -> Mish as ONE operator."""
    conv, gn = seq[0], seq[1]
    if not _is_groupnorm(gn):
        raise Unsupported("norm_type other than groupnorm")
    return p.conv(x, w_conv(conv, x.C), out, taps=k, pad=k // 2, bias=_const_vec(p.packed(lambda: conv.bias)),
                  gn=gn, act=cabi.ACT_MISH, **kw)


def _lower_resblock(p: Program, blk, x: View, out: View, k: int, cond: dict):
    """(Chi)ResidualBlock = 2 operators: conv1+GN+Mish+FiLM, then conv2+GN+Mish+shortcut."""
    h = p.act(out.L, out.C)
    _lower_conv_block(p, blk.conv1, x, h, k, **cond)
    if isinstance(blk.residual_conv, nn.Conv1d):
        rc = blk.residual_conv
        shortcut = dict(res_conv=(x, w_rows(lambda: _pad_cin(rc.weight, x.C)[:, :, 0]), lambda: rc.bias))
    else:
        shortcut = dict(res=x)
    return _lower_conv_block(p, blk.conv2, h, out, k, **shortcut)


def _unet_body(p: Program, net, x: View, horizon: int, k: int, film_of: Callable, stage_len: int, final_k: int):
    """Shared down / mid / up walk of both UNets.  ``film_of(block)`` gives the conditioning kwargs.
    Skip connections are never copied: the producer writes straight into one half of the (b, L, 2C)
    buffer the up-stage reads as its concatenated input."""
    n = len(net.downs)
    chans = [net.downs[s][0].conv1[0].out_channels for s in range(n)]
    lens = [horizon >> s for s in range(n)]
    if lens[-1] < 1:
        raise Unsupported("horizon too short for the number of stages")
    # cat buffer of up-stage u holds [x | skip h[n-1-u]] at resolution n-1-u
    cats = [View(p.buf(p.rows, lens[n - 1 - u], 2 * chans[n - 1 - u], dtype=p.act_dtype), lens[n - 1 - u],
                 2 * chans[n - 1 - u], tf32=p.math == cabi.MATH_TF32_TC) for u in range(n - 1)]

    def skip_slot(s):     # where h[s] lives
        if s == 0 or n == 1:
            return p.act(lens[s], chans[s])
        u = n - 1 - s
        return cats[u].channels(chans[s], chans[s])

    for s in range(n):
        stage = net.downs[s]
        mid = _lower_resblock(p, stage[0], x, p.act(lens[s], chans[s]), k, film_of(stage[0]))
        h = _lower_resblock(p, stage[1], mid, skip_slot(s), k, film_of(stage[1]))
        down = stage[stage_len - 1]
        if isinstance(down, nn.Identity):
            x = h
        else:
            x = p.conv(h, w_conv(down.conv), p.act(lens[s + 1], chans[s]), taps=3, stride=2, pad=1,
                       bias=_const_vec(p.packed(lambda d=down: d.conv.bias)))

    mids = [net.mid_block1, net.mid_block2] if hasattr(net, "mid_block1") else list(net.mids)
    x = _lower_resblock(p, mids[0], x, p.act(lens[-1], chans[-1]), k, film_of(mids[0]))
    dst = cats[0].channels(0, chans[-1]) if n > 1 else p.act(lens[-1], chans[-1])
    x = _lower_resblock(p, mids[1], x, dst, k, film_of(mids[1]))

    for u in range(n - 1):
        stage = net.ups[u]
        s = n - 1 - u                          # resolution index of this up stage
        c_out = stage[0].conv1[0].out_channels
        y = _lower_resblock(p, stage[0], cats[u], p.act(lens[s], c_out), k, film_of(stage[0]))
        y = _lower_resblock(p, stage[1], y, p.act(lens[s], c_out), k, film_of(stage[1]))
        up = stage[stage_len - 1]
        if isinstance(up, nn.Identity):
            raise Unsupported("up stage without Upsample1d")
        dst = cats[u + 1].channels(0, c_out) if u + 1 < n - 1 else p.act(lens[s - 1], c_out)
        x = p.conv(y, w_convT(up.conv), dst, taps=3, stride=1, pad=1, phases=2, L_out=lens[s],
                   bias=_const_vec(p.packed(lambda m=up: m.conv.bias)))

    fc = net.final_conv
    if fc[0].in_channels != x.C:
        # dim_mult[0] != 1 (a single-stage UNet included): the module's final_conv cannot take the last stage's channels
        # and its forward raises; the weight packing would zero-pad them instead
        raise Unsupported(f"final_conv takes {fc[0].in_channels} channels, the last stage gives {x.C}")
    y = _lower_conv_block(p, fc, x, p.act(horizon, fc[0].out_channels), final_k)
    last = fc[3]
    return p.conv(y, w_rows(lambda: last.weight[:, :, 0]), p.act(horizon, last.out_channels, dtype=torch.float32),
                  bias=_const_vec(p.packed(lambda: last.bias)))


def _all_resblocks(net):
    blocks = []
    for stage in net.downs:
        blocks += [stage[0], stage[1]]
    blocks += [net.mid_block1, net.mid_block2] if hasattr(net, "mid_block1") else list(net.mids)
    for stage in net.ups:
        blocks += [stage[0], stage[1]]
    return blocks


def lower_janner(p: Program, net: nn.Module, x: View, horizon: int, has_cond: bool, in_batch_mod: int) -> View:
    if any(not isinstance(s[2], nn.Identity) for s in list(net.downs) + list(net.ups)) or \
            not isinstance(net.mid_attn, nn.Identity):
        raise Unsupported("JannerUNet1d(attention=True)")
    if horizon & (horizon - 1):
        raise Unsupported("horizon must be 2^n")
    blocks = _all_resblocks(net)
    widths = [b.emb_mlp[1].out_features for b in blocks]
    offs = [sum(widths[:i]) for i in range(len(widths))]
    total = sum(widths)
    k = blocks[0].conv1[0].kernel_size[0]

    if not has_cond:
        # time conditioning is batch-constant: one row per iteration, evaluated by the model's own modules
        table = p.buf(p.n_iters, total)

        def fill(ctx):
            e = net.map_noise(ctx.t_all)
            e = net.map_emb(e + torch.zeros_like(e))
            table.copy_(torch.cat([b.emb_mlp(e) for b in blocks], dim=1))
        fill.time_only = True      # depends on (weights, timesteps) only: the runtime skips it when neither changed
        p.per_call.append(fill)
        film = {id(b): dict(shift=_vec(step=table, col=o)) for b, o in zip(blocks, offs)}
    else:
        # emb = map_emb(map_noise(t) + cond_b): per trajectory AND per iteration -> tiny GEMMs in the loop.
        md, e_dim = net.map_emb[2].out_features, net.map_emb[0].in_features
        t_rows = p.buf(p.n_iters, net.map_emb[0].out_features)       # W0 map_noise(t) + b0, per iteration
        c_rows = p.buf(p.rows, net.map_emb[0].out_features)          # W0 cond_b, per trajectory
        dummy_in, dummy_w = p.buf(p.rows, 1), p.buf(1, net.map_emb[0].out_features)

        def fill(ctx):
            t_rows.copy_(net.map_emb[0](net.map_noise(ctx.t_all)))
            c_rows.copy_(F.linear(ctx.cond_rows, net.map_emb[0].weight))
        p.per_call.append(fill)
        h1 = View(p.buf(p.rows, 1, net.map_emb[0].out_features), 1, net.map_emb[0].out_features)
        p.conv(View(dummy_in, 1, 1), WSpec(lambda: dummy_w), h1, bias=_vec(step=t_rows, sample=c_rows), act=cabi.ACT_MISH)
        emb_m = View(p.buf(p.rows, 1, md), 1, md)                      # Mish(map_emb(.)): every consumer starts with Mish
        p.conv(h1, w_linear(net.map_emb[2].weight), emb_m, bias=_const_vec(p.packed(lambda: net.map_emb[2].bias)),
               act=cabi.ACT_MISH)
        tb = View(p.buf(p.rows, 1, total), 1, total)
        p.conv(emb_m, w_rows(lambda: torch.cat([b.emb_mlp[1].weight for b in blocks], 0)), tb,
               bias=_const_vec(p.packed(lambda: torch.cat([b.emb_mlp[1].bias for b in blocks], 0))))
        film = {id(b): dict(shift=_vec(sample=tb.t.view(p.rows, total), col=o)) for b, o in zip(blocks, offs)}

    x = View(x.t, x.L, x.C, x.offset, x.bstride, x.lstride, x.tf32)
    # first conv reads x_t; under two-branch CFG both halves of the doubled batch read the same rows
    first = blocks[0]
    pred = _unet_body_with_mod(p, net, x, horizon, k, lambda b: film[id(b)], 4, 5, in_batch_mod, first)
    return pred


def _unet_body_with_mod(p, net, x, horizon, k, film_of, stage_len, final_k, in_batch_mod, first_block):
    """``_unet_body`` with ``in_batch_mod`` applied to the operators that read x_t directly (the first block's
    conv1 and its shortcut)."""
    n_before = len(p.ops)
    pred = _unet_body(p, net, x, horizon, k, film_of, stage_len, final_k)
    if in_batch_mod:
        x_ptr = x.ptr
        for op in p.ops[n_before:]:
            c = op.u.conv
            if op.kind == cabi.OP_CONV and c.in_ == x_ptr:
                c.in_batch_mod = in_batch_mod
            if op.kind == cabi.OP_CONV and (c.res_in == x_ptr or c.res == x_ptr):
                c.res_batch_mod = in_batch_mod
    return pred


def _fixed_shape_rows(fn, x: torch.Tensor, chunk: int = 1024) -> torch.Tensor:
    """``fn`` over the rows of ``x`` in chunks of ``chunk`` rows (the last one zero-padded): every row goes through GEMMs of
    the same shape whatever the batch, so a trajectory's conditioning rows do not depend on how many trajectories share the
    call (BLAS libraries pick their algorithm, and with it the summation order, by problem size).  Pinned by the sub-batch
    check of tests/test_baseline_configs_gpu.py::test_cfg5_consistency_one_step_per_gpu_batch (8192 vs 256 trajectories)."""
    n = x.shape[0]
    pad = (-n) % chunk
    if pad:
        x = torch.cat([x, x.new_zeros((pad,) + tuple(x.shape[1:]))])
    return torch.cat([fn(c) for c in x.split(chunk)])[:n]


def lower_chi(p: Program, net: nn.Module, x: View, horizon: int, has_cond: bool, in_batch_mod: int) -> View:
    if not net.obs_as_global_cond:
        raise Unsupported("ChiUNet1d(obs_as_global_cond=False)")
    if not has_cond:
        raise Unsupported("ChiUNet1d needs a condition")       # the reference raises too (chiunet.py:149)
    if horizon & (horizon - 1):
        raise Unsupported("horizon must be 2^n")
    blocks = _all_resblocks(net)
    widths = [b.cond_encoder[1].out_features for b in blocks]
    offs = [sum(widths[:i]) for i in range(len(widths))]
    total = sum(widths)
    e_dim = net.emb_dim
    k = blocks[0].conv1[0].kernel_size[0]
    step_tab, samp_tab = p.buf(p.n_iters, total), p.buf(p.rows, total)

    def fill(ctx):
        # cond_encoder(cat[time, obs]) = W_t Mish(time) + b  (per iteration)  +  W_o Mish(obs)  (per trajectory)
        te = F.mish(net.map_emb(net.map_noise(ctx.t_all)))
        step_tab.copy_(torch.cat([F.linear(te, b.cond_encoder[1].weight[:, :e_dim], b.cond_encoder[1].bias)
                                  for b in blocks], 1))

        def per_traj(c):
            oe = F.mish(net.global_cond_encoder(c))
            return torch.cat([F.linear(oe, b.cond_encoder[1].weight[:, e_dim:]) for b in blocks], 1)
        samp_tab.copy_(_fixed_shape_rows(per_traj, torch.flatten(ctx.cond_rows, 1)))
    p.per_call.append(fill)

    def film_of(b):
        o = offs[[id(z) for z in blocks].index(id(b))]
        if b.cond_predict_scale:
            return dict(scale=_vec(step_tab, samp_tab, o), shift=_vec(step_tab, samp_tab, o + b.out_dim))
        return dict(shift=_vec(step_tab, samp_tab, o))
    return _unet_body_with_mod(p, net, x, horizon, k, film_of, 3, k, in_batch_mod, blocks[0])


# =============================================================================== DQLMlp
def lower_dql(p: Program, net: nn.Module, x: View, has_cond: bool, in_batch_mod: int) -> View:
    act_dim = x.C
    lin1 = net.mid_layer[0]
    e_dim = net.time_mlp[2].out_features
    hidden = lin1.out_features
    step_tab, samp_tab = p.buf(p.n_iters, hidden), p.buf(p.rows, hidden)

    def fill(ctx):
        # Linear over cat[x, time_mlp(map_noise(t)), obs] = W_x x + (W_t temb + b) + W_o obs
        temb = net.time_mlp(net.map_noise(ctx.t_all))
        step_tab.copy_(F.linear(temb, lin1.weight[:, act_dim:act_dim + e_dim], lin1.bias))
        if has_cond:
            samp_tab.copy_(F.linear(ctx.cond_rows, lin1.weight[:, act_dim + e_dim:]))
        else:
            samp_tab.zero_()
    p.per_call.append(fill)
    h = View(p.buf(p.rows, 1, hidden), 1, hidden)
    p.conv(x, w_linear(lin1.weight, slice(0, act_dim)), h, bias=_vec(step_tab, samp_tab), act=cabi.ACT_MISH,
           in_batch_mod=in_batch_mod)
    for idx in (2, 4):
        lin = net.mid_layer[idx]
        h2 = View(p.buf(p.rows, 1, lin.out_features), 1, lin.out_features)
        p.conv(h, w_linear(lin.weight), h2, bias=_const_vec(p.packed(lambda m=lin: m.bias)), act=cabi.ACT_MISH)
        h = h2
    out = View(p.buf(p.rows, 1, act_dim), 1, act_dim)
    fl = net.final_layer
    return p.conv(h, w_linear(fl.weight), out, bias=_const_vec(p.packed(lambda: fl.bias)))


# =============================================================================== DQLMlp, differentiable
def _rev(stash: torch.Tensor):
    """(pointer, signed stride) that walks the [n_iters, ...] stash from its last slot to its first: backward iteration m reads
    the slot of forward iteration n_iters - 1 - m."""
    per = stash[0].numel()
    return stash.data_ptr() + 4 * per * (stash.shape[0] - 1), -per


class DQLGrad:
    """DQLMlp under ``sample(requires_grad=True)``: a forward program that keeps what the backward needs and the backward
    program over the same buffers.

    Forward, per iteration n (the reverse loop's network evaluation; the runtime appends the solver update):
        stash x_n;  z1 = W_x x_n + step_tab[n] + samp_tab[b]  (Linear, no activation);  stash z1, h1 = Mish(z1)  (one operator);
        z2, z3 alike;  pred = W_f h3 + b_f;  stash pred  (raw: clip_prediction happens in the update)
    Backward, per iteration m = n_iters-1 .. 0 walking the stashes in reverse (the runtime puts the update's backward first; it
    turns d x_{n+1} in ``gx`` into d pred in ``gpred`` and the direct part of d x_n in ``gx``):
        d W_f, d b_f += Mish(z3)^T gpred;  dz3 = (gpred W_f) Mish'(z3);  ... layer 3, layer 2 alike ... ;
        d step_tab[n] = sum_rows dz1 (with d W_x += x_n^T dz1: W_x's "bias" is the per-iteration table row);
        d samp_tab += dz1;  gx += dz1 W_x
    ``step_tab`` / ``samp_tab`` are filled by the caller (they are autograd inputs: d step_tab carries into time_mlp, the time
    columns of mid_layer[0] and its bias, d samp_tab into the observation columns and the condition).

    Consistency form (``xin`` given: the consistency model, whose network reads xin = c_in x written by the CDS_OP_PREP the
    runtime puts in front): x_n (the re-noised x_t the update reads) and xin_n are both stashed, the first layer reads xin and
    its weight gradient the stashed xin, and the last data gradient writes d xin into its own buffer ``gxin`` (overwritten,
    not accumulated): the runtime's CDS_OP_PREP in backward mode then adds c_in * gxin to ``gx``."""

    def __init__(self, p: Program, bp: Program, net: nn.Module, x: View, xin: Optional[View] = None):
        R, n, a = p.rows, p.n_iters, x.C
        lins = [net.mid_layer[0], net.mid_layer[2], net.mid_layer[4], net.final_layer]
        widths = [lin.out_features for lin in lins[:3]]
        self.step_tab, self.samp_tab = p.buf(n, widths[0]), p.buf(R, widths[0])
        self.xs, self.ps = p.buf(n, R, a), p.buf(n, R, a)
        self.xins = p.buf(n, R, a) if xin is not None else None
        self.zs = [p.buf(n, R, w) for w in widths]

        def stash(src: View, dst: torch.Tensor, act_out: Optional[View] = None):
            op = cabi.Op()
            op.kind = cabi.OP_STASH
            s = op.u.stash
            s.n, s.src, s.dst, s.dst_iter_stride = R * src.C, src.ptr, dst.data_ptr(), dst[0].numel()
            if act_out is not None:
                s.act_out, s.act = act_out.ptr, cabi.ACT_MISH
            p.ops.append(op)

        stash(x, self.xs)
        if xin is not None:
            stash(xin, self.xins)
        net_in = x if xin is None else xin
        h = net_in
        for k, lin in enumerate(lins[:3]):
            z = View(p.buf(R, 1, widths[k]), 1, widths[k])
            if k == 0:
                p.conv(net_in, w_linear(lin.weight, slice(0, a)), z, bias=_vec(self.step_tab, self.samp_tab))
            else:
                p.conv(h, w_linear(lin.weight), z, bias=_const_vec(p.packed(lambda m=lin: m.bias)))
            h = View(p.buf(R, 1, widths[k]), 1, widths[k])
            stash(z, self.zs[k], h)
        fl = lins[3]
        self.pred = View(p.buf(R, 1, a), 1, a)
        p.conv(h, w_linear(fl.weight), self.pred, bias=_const_vec(p.packed(lambda: fl.bias)))
        stash(self.pred, self.ps)

        # ---- backward program
        self.gx, self.gpred = bp.buf(R, a), bp.buf(R, a)
        dz = [bp.buf(R, w) for w in widths]
        wts = [bp.packed(lambda: lins[0].weight[:, :a])] + [bp.packed(lambda m=lin: m.weight) for lin in lins[1:]]
        self.g_w = [bp.buf(*w.shape) for w in wts]                        # d W_x, d W2, d W3, d W_f
        self.g_b = [None] + [bp.buf(lin.out_features) for lin in lins[1:]]
        self.g_step, self.g_samp = bp.buf(n, widths[0]), bp.buf(R, widths[0])
        self.accumulators = self.g_w + self.g_b[1:] + [self.g_step, self.g_samp]

        def wgrad(k: int, dzk: torch.Tensor, h_src: torch.Tensor, act: int):
            op = cabi.Op()
            op.kind = cabi.OP_WGRAD
            g = op.u.wgrad
            N, K = wts[k].shape
            g.rows, g.N, g.K, g.dz, g.ldz = R, N, K, dzk.data_ptr(), N
            g.h, g.h_iter_stride = _rev(h_src)
            g.ldh, g.act = K, act
            g.dw, g.lddw, g.accumulate = self.g_w[k].data_ptr(), K, 1
            if k == 0:
                g.db, g.db_iter_stride = _rev(self.g_step)
            else:
                g.db, g.db_iter_stride = self.g_b[k].data_ptr(), 0
            bp.ops.append(op)

        def dgrad(k: int, dzk: torch.Tensor, out: torch.Tensor, z_src: Optional[torch.Tensor], accumulate=0, out_sum=None):
            op = cabi.Op()
            op.kind = cabi.OP_DGRAD
            d = op.u.dgrad
            N, K = wts[k].shape
            d.rows, d.N, d.K, d.dz, d.ldz, d.w, d.ldw = R, N, K, dzk.data_ptr(), N, wts[k].data_ptr(), K
            if z_src is not None:
                d.z, d.z_iter_stride = _rev(z_src)
                d.act = cabi.ACT_MISH
            d.accumulate, d.out, d.ldo = accumulate, out.data_ptr(), K
            if out_sum is not None:
                d.out_sum = out_sum.data_ptr()
            bp.ops.append(op)

        upstream = self.gpred
        for k in (3, 2, 1):
            wgrad(k, upstream, self.zs[k - 1], cabi.ACT_MISH)
            dgrad(k, upstream, dz[k - 1], self.zs[k - 1], out_sum=self.g_samp if k == 1 else None)
            upstream = dz[k - 1]
        if xin is None:
            wgrad(0, upstream, self.xs, cabi.ACT_NONE)
            dgrad(0, upstream, self.gx, None, accumulate=1)
        else:
            self.gxin = bp.buf(R, a)
            wgrad(0, upstream, self.xins, cabi.ACT_NONE)
            dgrad(0, upstream, self.gxin, None)


# =============================================================================== IDQLMlp
def lower_idql(p: Program, net: nn.Module, x: View, has_cond: bool, in_batch_mod: int) -> View:
    """idqlmlp.py:21-65.  affine_in over cat[x, time_mlp(t), obs] splits like DQLMlp's first Linear (per-iteration row +
    per-trajectory row); each residual block is LayerNorm (affine folded into the LN+modulate operator: scale = gamma - 1,
    shift = beta, broadcast over the batch) -> Linear + Mish -> Linear + identity residual.  Dropout is inactive in eval mode."""
    if net.training and any(blk.net[0].p > 0 for blk in net.ln_resnet):
        raise Unsupported("IDQLMlp in train mode (dropout)")
    act_dim = x.C
    lin_in = net.affine_in
    e_dim = net.time_mlp[2].out_features
    hidden = lin_in.out_features
    step_tab, samp_tab = p.buf(p.n_iters, hidden), p.buf(p.rows, hidden)

    def fill(ctx):
        temb = net.time_mlp(net.map_noise(ctx.t_all))
        step_tab.copy_(F.linear(temb, lin_in.weight[:, act_dim:act_dim + e_dim], lin_in.bias))
        if has_cond:
            samp_tab.copy_(F.linear(ctx.cond_rows, lin_in.weight[:, act_dim + e_dim:]))
        else:
            samp_tab.zero_()
    p.per_call.append(fill)
    f32 = torch.float32
    h = View(p.buf(p.rows, 1, hidden), 1, hidden)                       # the residual stream stays exact fp32
    p.conv(x, w_linear(lin_in.weight, slice(0, act_dim)), h, bias=_vec(step_tab, samp_tab), in_batch_mod=in_batch_mod)
    for blk in net.ln_resnet:
        ln, fc1, fc2 = blk.net[1], blk.net[2], blk.net[4]
        if not ln.elementwise_affine:
            raise Unsupported("LayerNorm without affine")
        mod = p.buf(1, 2 * hidden)                                    # [gamma - 1 | beta]: LN(x) * (1 + scale) + shift
        p.packers.append(lambda m=mod, l=ln: m.copy_(torch.cat([l.weight - 1., l.bias])[None]))
        p.packers[-1]()
        y = p.act(1, hidden)
        op = cabi.Op()
        op.kind = cabi.OP_LNMOD
        m = op.u.lnmod
        m.batch, m.L, m.C, m.eps = p.rows, 1, hidden, ln.eps
        m.in_, m.out, m.out_dtype = h.ptr, y.ptr, y.dtype
        m.scale, m.shift, m.mod_bstride = mod.data_ptr(), mod.data_ptr() + 4 * hidden, 0
        p.ops.append(op)
        mid = p.act(1, fc1.out_features)
        p.conv(y, w_linear(fc1.weight), mid, bias=_const_vec(p.packed(lambda f=fc1: f.bias)), act=cabi.ACT_MISH)
        h2 = View(p.buf(p.rows, 1, hidden), 1, hidden)
        p.conv(mid, w_linear(fc2.weight), h2, bias=_const_vec(p.packed(lambda f=fc2: f.bias)), res=h)
        h = h2
    out = View(p.buf(p.rows, 1, act_dim), 1, act_dim)
    fo = net.affine_out
    return p.conv(h, w_linear(fo.weight), out, bias=_const_vec(p.packed(lambda: fo.bias)))


# =============================================================================== SfBCUNet
def lower_sfbc(p: Program, net: nn.Module, x: View, has_cond: bool, in_batch_mod: int) -> View:
    """sfbc_unet.py:9-82.  Every residual block is two fused operators:
    ``h = silu(W1 x + b1) + linearc(c)`` (the conditioning enters as the post-activation shift: one row per iteration for the
    time part, one per trajectory for the condition part, both evaluated once per call for all blocks) and
    ``out = silu(W2 h + b2) + skip(x)`` (skip = the operator's shortcut GEMM, or an identity residual).
    ``torch.cat([x, kept.pop()])`` costs nothing: the down block whose output is kept writes straight into the right-hand
    channels of the up block's input buffer, the previous block into the left-hand ones."""
    downs, ups = list(net.down_blocks), list(net.up_blocks)
    blocks = downs + [net.mid_block] + ups
    widths = [b.linearc.out_features for b in blocks]
    offs = [sum(widths[:i]) for i in range(len(widths))]
    total = sum(widths)
    step_tab, samp_tab = p.buf(p.n_iters, total), p.buf(p.rows, total)

    def fill(ctx):
        wc = torch.cat([b.linearc.weight for b in blocks], 0)
        bc = torch.cat([b.linearc.bias for b in blocks], 0)
        step_tab.copy_(F.linear(net.t_layer(net.map_noise(ctx.t_all)), wc, bc))
        if has_cond:
            samp_tab.copy_(F.linear(ctx.cond_rows, wc))
        else:
            samp_tab.zero_()
    p.per_call.append(fill)

    n = len(downs)
    # input buffers of the up blocks: [ x from below | kept down activation ]
    cat_in = []
    for j, b in enumerate(ups):
        left = b.linear1[0].in_features - downs[n - 1 - j].linear1[0].out_features
        cat_in.append((p.act(1, b.linear1[0].in_features), left))

    def out_view(width, dest):
        """Where a block's output goes: a fresh activation, or a channel range of an up block's input buffer."""
        if dest is None:
            return p.act(1, width)
        buf, start = dest
        return buf.channels(start, width)

    def block(b, xin, o, dest, first=False):
        width = b.linear1[0].out_features
        h = p.act(1, width)
        ibm = in_batch_mod if first else 0
        p.conv(xin, w_linear(b.linear1[0].weight), h, bias=_const_vec(p.packed(lambda: b.linear1[0].bias)), act=cabi.ACT_SILU,
               shift=_vec(step=step_tab, sample=samp_tab, col=o), in_batch_mod=ibm)
        out = out_view(width, dest)
        kw = dict(bias=_const_vec(p.packed(lambda: b.linear2[0].bias)), act=cabi.ACT_SILU, res_batch_mod=ibm)
        if isinstance(b.skip, nn.Linear):
            kw["res_conv"] = (xin, w_linear(b.skip.weight), lambda: b.skip.bias)
        else:
            kw["res"] = xin
        return p.conv(h, w_linear(b.linear2[0].weight), out, **kw)

    h = x
    for i, b in enumerate(downs):
        j = n - 1 - i                              # the up block that pops this activation (none for the first down block)
        dest = (cat_in[j][0], cat_in[j][1]) if 0 <= j < len(ups) else None
        h = block(b, h, offs[i], dest, first=(i == 0))
    h = block(net.mid_block, h, offs[n], (cat_in[0][0], 0) if ups else None)
    for j, b in enumerate(ups):
        dest = (cat_in[j + 1][0], 0) if j + 1 < len(ups) else None
        h = block(b, cat_in[j][0], offs[n + 1 + j], dest)
    out = View(p.buf(p.rows, 1, x.C), 1, x.C)
    return p.conv(h, w_linear(net.out_layer.weight), out, bias=_const_vec(p.packed(lambda: net.out_layer.bias)))


# =============================================================================== PearceMlp
def lower_pearce(p: Program, net: nn.Module, x: View, has_cond: bool, in_batch_mod: int) -> View:
    """pearcemlp.py:35-79.  Every Linear over a concatenation splits by column blocks, like DQLMlp's first layer:
      fcs[0]  W [x_e | t_e | cond]      = W_xe x_e  + (W_te map_noise(t) + b: one row per iteration) + (W_c cond: one row per trajectory)
      fcs[k]  W [nn/1.414 | x | t]      = (W_h / c) v + (x W_x^T: one row per trajectory AND iteration, a small GEMM ahead of the
                                          blocks, all three layers at once) + (w_t t + b: one row per iteration)
    The residual chain ``nn_{k+1} = FC_k(nn_k / 1.414, ..) + nn_k / 1.414`` is carried as ``v_k = 1.414^(k-1) nn_k`` so that every
    residual has coefficient one: ``v_{k+1} = 1.414^k FC_k + v_k`` (a constant output scale), the 1 / 1.414^k go into the packed
    weights of the Linear that reads ``v_k``.  FCBlock = Linear + GroupNorm1d + exact GELU = one operator."""
    act_dim, emb, To = x.C, net.emb_dim, net.To
    fc0, fc1, fc2, head = net.fcs[0], net.fcs[1], net.fcs[2], net.fcs[3]
    for fc in (fc0, fc1, fc2):
        if not _is_groupnorm(fc.model[1]) or type(fc.model[2]).__name__ != "GELU" or getattr(fc.model[2], "approximate", "none") != "none":
            raise Unsupported("PearceMlp FCBlock other than Linear -> GroupNorm1d -> GELU")
    hidden = fc0.model[0].out_features
    lins = [fc1.model[0], fc2.model[0], head]
    s = 1.414
    inv = [1.0 / s, 1.0 / (s * s), 1.0 / (s * s)]       # what the Linear reading v_1, v_2, v_3 folds into its weights
    widths = [l.out_features for l in lins]
    offs = [sum(widths[:i]) for i in range(3)]
    xw = p.buf(p.rows, sum(widths))                                     # x W_x^T of the three layers
    step0, samp0 = p.buf(p.n_iters, hidden), p.buf(p.rows, hidden)
    steps = [p.buf(p.n_iters, w) for w in widths]

    def fill(ctx):
        w0 = fc0.model[0]
        step0.copy_(F.linear(net.map_noise(ctx.t_all), w0.weight[:, emb:2 * emb], w0.bias))
        if has_cond:
            samp0.copy_(F.linear(torch.flatten(ctx.cond_rows, 1), w0.weight[:, 2 * emb:]))
        else:
            samp0.zero_()
        tr = ctx.t_all.to(torch.float32)[:, None]
        for lin, tab in zip(lins, steps):
            tab.copy_(tr * lin.weight[:, hidden + act_dim][None, :] + lin.bias[None, :])
    p.per_call.append(fill)

    p.conv(x, w_rows(lambda: torch.cat([l.weight[:, hidden:hidden + act_dim] for l in lins], 0)), View(xw, 1, xw.shape[1]),
           in_batch_mod=in_batch_mod)
    ae = net.act_emb
    e1 = p.act(1, ae[0].out_features)
    p.conv(x, w_linear(ae[0].weight), e1, bias=_const_vec(p.packed(lambda: ae[0].bias)), act=cabi.ACT_LEAKY_RELU, in_batch_mod=in_batch_mod)
    x_e = p.act(1, emb)
    p.conv(e1, w_linear(ae[2].weight), x_e, bias=_const_vec(p.packed(lambda: ae[2].bias)))
    f32 = torch.float32
    v = View(p.buf(p.rows, 1, hidden), 1, hidden)                        # the residual chain stays exact fp32
    p.conv(x_e, w_linear(fc0.model[0].weight, slice(0, emb)), v, bias=_vec(step0, samp0), gn=fc0.model[1], act=cabi.ACT_GELU_ERF)
    for k, fc in enumerate((fc1, fc2)):
        lin = fc.model[0]
        v2 = View(p.buf(p.rows, 1, hidden), 1, hidden)
        scale = p.buf(1, hidden)
        scale.fill_(s ** (k + 1))
        p.conv(v, w_rows(lambda l=lin, c=inv[k]: l.weight[:, :hidden] * c), v2, bias=cabi_vec2(steps[k], xw, offs[k]), gn=fc.model[1], act=cabi.ACT_GELU_ERF, scale=_const_vec(scale[0]), res=v)
        v = v2
    out = View(p.buf(p.rows, 1, act_dim), 1, act_dim)
    return p.conv(v, w_rows(lambda: head.weight[:, :hidden] * inv[2]), out, bias=cabi_vec2(steps[2], xw, offs[2]))


def cabi_vec2(step: torch.Tensor, sample: torch.Tensor, sample_col: int) -> cabi.Vec:
    """step: [n_iters, W] table from column 0; sample: [rows, Wtot] table from column ``sample_col``."""
    v = cabi.Vec()
    v.step, v.step_stride = step.data_ptr(), step.stride(0)
    v.sample, v.sample_stride = sample.data_ptr() + 4 * int(sample_col), sample.stride(0)
    return v


# =============================================================================== DiT1d
def _embed_tokens(p: Program, x: View, lin: nn.Linear, pos: View, X: View, in_batch_mod: int):
    """X = lin(x_t) + pos (a (L, d) table broadcast over the batch)."""
    L = X.L
    if p.tc and x.t.dtype == torch.float32 and x.lstride == x.C and x.bstride == L * x.C:
        # x_t enters as a channel-padded copy in the activation dtype (kept fresh by the solver update, like the UNets' hand-over)
        kin = p.k_align * ((x.C + p.k_align - 1) // p.k_align)
        xb = p.cast_pad(x, kin, rows=in_batch_mod or p.rows)
        w_in = w_rows(lambda: F.pad(lin.weight, (0, kin - lin.weight.shape[1])))
        p.token_linear(xb, w_in, X, bias=_const_vec(p.packed(lambda: lin.bias)), res=pos, in_batch_mod=in_batch_mod)
    else:
        p.conv(x, w_linear(lin.weight), X, bias=_const_vec(p.packed(lambda: lin.bias)), res=pos, in_batch_mod=in_batch_mod)


def _dit_conditioning(p: Program, net: nn.Module, L: int, has_cond: bool):
    """DiT1d's conditioning inside the program -> (the per-trajectory adaLN table [rows, sum of the adaLN widths] of every block
    and the final layer, the (L, d) position table): emb = Mish(W2 Mish(W0 (map_noise(t) + cond_b) + b0) + b2), every consumer
    applies SiLU first"""
    d, R = net.d_model, p.rows
    w0 = net.map_emb[0]
    t_rows, c_rows = p.buf(p.n_iters, d), p.buf(R, d)
    pos = p.buf(L, d)
    dummy_in, dummy_w = p.buf(R, 1), p.buf(1, d)

    def fill(ctx):
        t_rows.copy_(w0(net.map_noise(ctx.t_all)))
        if has_cond:
            c_rows.copy_(F.linear(ctx.cond_rows, w0.weight))
        else:
            c_rows.zero_()
        pos.copy_(net.pos_emb(torch.arange(L, device=pos.device)))      # int64 positions: degenerate table, by design
    p.per_call.append(fill)
    h1 = View(p.buf(R, 1, d), 1, d)
    p.conv(View(dummy_in, 1, 1), WSpec(lambda: dummy_w), h1, bias=_vec(step=t_rows, sample=c_rows), act=cabi.ACT_MISH)
    emb_s = View(p.buf(R, 1, d), 1, d)
    p.conv(h1, w_linear(net.map_emb[2].weight), emb_s, bias=_const_vec(p.packed(lambda: net.map_emb[2].bias)),
           act=cabi.ACT_MISH_SILU)
    mods = [blk.adaLN_modulation[1] for blk in net.blocks] + [net.final_layer.adaLN_modulation[1]]
    total = sum(m.out_features for m in mods)
    mod = View(p.buf(R, 1, total), 1, total)
    p.conv(emb_s, w_rows(lambda: torch.cat([m.weight for m in mods], 0)), mod,
           bias=_const_vec(p.packed(lambda: torch.cat([m.bias for m in mods], 0))))
    return mod.t.view(R, total), pos


def _dit_block(p: Program, blk: nn.Module, mod2d: torch.Tensor, o: int, heads: int, X: View, Y: View, QKV: View, ATT: View,
               HID: View, X1: View, X2: View, hpre: Optional[View] = None):
    """One DiTBlock: X (block input) -> X1 (after the attention residual) -> X2 (block output); the adaLN chunks of the block
    start at column ``o`` of ``mod2d`` in the order shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp.  The denoiser
    passes one buffer for X, X1 and X2 (the residual stream updated in place) and fuses the GELU into the first MLP Linear; a
    classifier's input gradient passes one X / X1 per block (the LayerNorm inputs its backward reads), and ``hpre``: the first MLP
    Linear then writes the GELU's pre-activation there and CDS_OP_STASH forms HID = gelu_tanh(hpre)."""
    d = X.C
    p.lnmod(X, Y, mod2d, o, o + d, blk.norm1.eps)
    at = blk.attn
    p.token_linear(Y, w_linear(at.in_proj_weight), QKV, bias=_const_vec(p.packed(lambda a=at: a.in_proj_bias)))
    p.attn(QKV, ATT, heads)
    # reference quirk (dit.py:33-34): the residual wraps the MODULATED tokens Y, not the block input
    p.token_linear(ATT, w_linear(at.out_proj.weight), X1, bias=_const_vec(p.packed(lambda a=at: a.out_proj.bias)),
                   scale=_vec(sample=mod2d, col=o + 2 * d), res=Y)
    p.lnmod(X1, Y, mod2d, o + 3 * d, o + 4 * d, blk.norm2.eps)
    b1 = _const_vec(p.packed(lambda b=blk: b.mlp[0].bias))
    if hpre is None:
        p.token_linear(Y, w_linear(blk.mlp[0].weight), HID, bias=b1, act=cabi.ACT_GELU_TANH)
    else:
        p.token_linear(Y, w_linear(blk.mlp[0].weight), hpre, bias=b1)
        _act_stash(p, hpre, HID, cabi.ACT_GELU_TANH)
    p.token_linear(HID, w_linear(blk.mlp[3].weight), X2, bias=_const_vec(p.packed(lambda b=blk: b.mlp[3].bias)),
                   scale=_vec(sample=mod2d, col=o + 5 * d), res=X1)


def lower_dit(p: Program, net: nn.Module, x: View, horizon: int, has_cond: bool, in_batch_mod: int) -> View:
    d = net.d_model
    depth = len(net.blocks)
    heads = net.blocks[0].attn.num_heads
    if net.blocks[0].attn.dropout != 0.0 and net.training:
        raise Unsupported("attention dropout in train mode")
    L = horizon
    mod2d, pos = _dit_conditioning(p, net, L, has_cond)

    # ---- tokens
    # residual stream X and the attention operands QKV stay fp32; what feeds a Linear layer (the modulated tokens Y, the
    # attention output, the MLP hidden) has the program's activation dtype: bf16 on tensor-core programs, where those Linear
    # layers (97 % of DiT1d's FLOPs outside attention) run on wgmma over the flattened token stream
    f32 = torch.float32
    X = p.act(L, d, f32)
    # head_dim 32 (every pipeline) and L <= 128: attention runs on tensor cores (mma.sync, bf16 q/k/v); otherwise fp32 CUDA cores
    QKV = p.act(L, 3 * d) if (d // heads == 32 and L <= 128) else p.act(L, 3 * d, f32)
    Y, ATT, HID = p.act(L, d), p.act(L, d), p.act(L, 4 * d)
    _embed_tokens(p, x, net.x_proj, View(pos, L, d, bstride=0), X, in_batch_mod)
    for i, blk in enumerate(net.blocks):
        _dit_block(p, blk, mod2d, 6 * d * i, heads, X, Y, QKV, ATT, HID, X, X)
    o = 6 * d * depth
    fl = net.final_layer
    p.lnmod(X, Y, mod2d, o, o + d, fl.norm_final.eps)
    out = p.act(L, net.in_dim, f32)
    p.token_linear(Y, w_linear(fl.linear.weight), out, bias=_const_vec(p.packed(lambda: fl.linear.bias)))
    return out                 # shaped (rows, L, in_dim): CDS_OP_GUIDE reads it per token


# =============================================================================== ChiTransformer
def _layernorm(p: Program, ln: nn.LayerNorm, x: View, out: View):
    """Affine nn.LayerNorm as CDS_OP_LNMOD: LN(x) * (1 + (gamma - 1)) + beta, the same vectors for every trajectory."""
    mod = p.packed(lambda: torch.cat([ln.weight - 1., ln.bias]))
    p.lnmod(x, out, mod.expand(p.rows, 2 * x.C), x.C, 0, ln.eps)


def lower_chitransformer(p: Program, net: nn.Module, x: View, horizon: int, has_cond: bool, in_batch_mod: int) -> View:
    """chitransformer.py.  Per decoder layer (norm_first): LN -> QKV Linear -> causal CDS_OP_MHA -> out-projection onto the
    residual stream; LN -> Q Linear -> CDS_OP_MHA over the memory (mask t >= s - 1) -> out-projection; LN -> Linear + exact
    GELU -> Linear.  The memory's keys / values never enter the loop: token 0 = encoder(map_noise(t) + cond_pos_emb[0]) is a
    per-iteration row, tokens 1..To = encoder(obs_emb(cond) + cond_pos_emb[1:]) are per-trajectory rows, each projected by
    every layer's K / V weights once per sample() call into [n_iters | rows, layers, 1 + To, 2 d] tables (the other part's
    rows are zero, so the operator's step + sample sum picks each token from its own table)."""
    from ..nn_diffusion.chitransformer import causal_mask, memory_mask
    if not isinstance(net.encoder, nn.Sequential):
        raise Unsupported("ChiTransformer(n_cond_layers > 0)")
    layers = list(net.decoder.layers)
    if net.training and (net.drop.p > 0 or any(l.dropout.p > 0 for l in layers)):
        raise Unsupported("ChiTransformer in train mode (dropout)")
    if net.decoder.norm is not None or any(not l.norm_first or l.activation is not F.gelu for l in layers):
        raise Unsupported("ChiTransformer decoder other than norm_first with exact GELU")
    To, L = net.To, horizon
    if net.mask.shape != (L, L) or not torch.equal(net.mask.detach().cpu(), causal_mask(L)) or \
            not torch.equal(net.memory_mask.detach().cpu(), memory_mask(L, To)):
        raise Unsupported("ChiTransformer with other attention masks or horizon != Ta")
    d, heads, Lk, n = net.pos_emb.shape[2], layers[0].self_attn.num_heads, 1 + To, len(layers)
    obs_dim, R = net.obs_dim, p.rows
    xattn = [l.multihead_attn for l in layers]

    kv_step = p.buf(p.n_iters, n, Lk, 2 * d, dtype=p.act_dtype)
    kv_samp = p.buf(R, n, Lk, 2 * d, dtype=p.act_dtype)

    def kv_of(m, a):                        # memory tokens -> [k | v] of one layer's cross-attention
        return F.linear(m, a.in_proj_weight[d:], a.in_proj_bias[d:])

    def fill_step(ctx):
        m0 = net.encoder(net.map_noise(ctx.t_all) + net.cond_pos_emb[0, 0])
        kv_step[:, :, 0].copy_(torch.stack([kv_of(m0, a) for a in xattn], 1))
    fill_step.time_only = True
    p.per_call.append(fill_step)

    def fill_samp(ctx):
        c = ctx.cond_rows
        c = torch.zeros(R, To * obs_dim, device=kv_samp.device) if c is None else c.reshape(R, To * obs_dim)

        def per_traj(rows):
            m = net.encoder(net.obs_emb(rows.view(-1, To, obs_dim)) + net.cond_pos_emb[0, 1:])
            return torch.stack([kv_of(m, a) for a in xattn], 1)
        kv_samp[:, :, 1:].copy_(_fixed_shape_rows(per_traj, c))
    p.per_call.append(fill_samp)

    f32 = torch.float32
    X = p.act(L, d, f32)                     # the residual stream stays exact fp32
    Y, Q, ATT, QKV, HID = p.act(L, d), p.act(L, d), p.act(L, d), p.act(L, 3 * d), p.act(L, 4 * d)
    pos = p.packed(lambda: net.pos_emb[0, :L])
    _embed_tokens(p, x, net.act_emb, View(pos, L, d, bstride=0), X, in_batch_mod)
    bias = lambda get: _const_vec(p.packed(get))     # noqa: E731
    for i, layer in enumerate(layers):
        sa, xa = layer.self_attn, layer.multihead_attn
        _layernorm(p, layer.norm1, X, Y)
        p.token_linear(Y, w_linear(sa.in_proj_weight), QKV, bias=bias(lambda a=sa: a.in_proj_bias))
        p.mha(QKV.channels(0, d), None, QKV.channels(d, 2 * d), ATT, heads, diag=0)
        p.token_linear(ATT, w_linear(sa.out_proj.weight), X, bias=bias(lambda a=sa: a.out_proj.bias), res=X)
        _layernorm(p, layer.norm2, X, Y)
        p.token_linear(Y, w_rows(lambda a=xa: a.in_proj_weight[:d]), Q, bias=bias(lambda a=xa: a.in_proj_bias[:d]))
        at = i * Lk * 2 * d
        p.mha(Q, View(kv_step, Lk, 2 * d, at, n * Lk * 2 * d), View(kv_samp, Lk, 2 * d, at, n * Lk * 2 * d), ATT, heads, diag=1)
        p.token_linear(ATT, w_linear(xa.out_proj.weight), X, bias=bias(lambda a=xa: a.out_proj.bias), res=X)
        _layernorm(p, layer.norm3, X, Y)
        p.token_linear(Y, w_linear(layer.linear1.weight), HID, bias=bias(lambda m=layer: m.linear1.bias), act=cabi.ACT_GELU_ERF)
        p.token_linear(HID, w_linear(layer.linear2.weight), X, bias=bias(lambda m=layer: m.linear2.bias), res=X)
    _layernorm(p, net.ln_f, X, Y)
    out = p.act(L, net.head.out_features, f32)
    p.token_linear(Y, w_linear(net.head.weight), out, bias=bias(lambda: net.head.bias))
    return out                 # shaped (rows, L, C): CDS_OP_GUIDE reads it per token


def lower_denoiser(p: Program, net: nn.Module, x: View, x_shape, has_cond: bool, in_batch_mod: int) -> View:
    """Dispatch on the backbone type (reference instances are recognised structurally by class name)."""
    name = type(net).__name__
    if name in ("JannerUNet1d", "ChiUNet1d") and len(x_shape) == 2 and p.tc:
        # TMA/wgmma want K in whole 64-byte rows: 32 bf16 / 16 fp32 channels
        x = p.cast_pad(x, p.k_align * ((x.C + p.k_align - 1) // p.k_align), rows=in_batch_mod or p.rows)
    if name == "JannerUNet1d" and len(x_shape) == 2:
        return lower_janner(p, net, x, x_shape[0], has_cond, in_batch_mod)
    if name == "ChiUNet1d" and len(x_shape) == 2:
        return lower_chi(p, net, x, x_shape[0], has_cond, in_batch_mod)
    if name == "DiT1d" and len(x_shape) == 2:
        return lower_dit(p, net, x, x_shape[0], has_cond, in_batch_mod)
    if name == "ChiTransformer" and len(x_shape) == 2:
        return lower_chitransformer(p, net, x, x_shape[0], has_cond, in_batch_mod)
    if name == "DQLMlp" and len(x_shape) == 1:
        return lower_dql(p, net, x, has_cond, in_batch_mod)
    if name == "DVInvMlp" and len(x_shape) == 1:
        if not has_cond:
            raise Unsupported("DVInvMlp needs a condition")         # the reference raises too (dvinvmlp.py:44)
        return lower_dql(p, net, x, has_cond, in_batch_mod)         # same graph: cat[x, time_mlp(t), cond] -> 3 x (Linear + Mish) -> Linear
    if name == "SfBCUNet" and len(x_shape) == 1:
        return lower_sfbc(p, net, x, has_cond, in_batch_mod)
    if name == "PearceMlp" and len(x_shape) == 1:
        return lower_pearce(p, net, x, has_cond, in_batch_mod)
    if name == "IDQLMlp" and len(x_shape) == 1:
        return lower_idql(p, net, x, has_cond, in_batch_mod)
    raise Unsupported(f"backbone {name} with x_shape {tuple(x_shape)}")


# =============================================================================== classifier guidance: the classifier's input gradient
def guidable(clf, x_shape, cond_cg=None) -> Optional[str]:
    """None when ``lower_classifier_grad`` can put the input gradient of ``clf`` at x_t into the loop, else the reason it cannot.
    The classifiers are recognised structurally (class names and the attributes the lowering reads), so that the reference's own
    instances qualify: a CumRewClassifier over a HalfJannerUNet1d, a HalfDiT1d or an out_dim-1 MLPNNClassifier, an
    MSEClassifier over an MLPNNClassifier guided with a per-trajectory target ``cond_cg``, or a QGPOClassifier over a
    QGPONNClassifier guided with a per-trajectory condition ``cond_cg`` (the observations)."""
    name = type(clf).__name__
    net_name = type(getattr(clf, "model_ema", None)).__name__
    if name == "CumRewClassifier":
        if net_name == "MLPNNClassifier":
            return _mlp_classifier_reason(clf, x_shape, cond_cg, mse=False)
        if net_name == "HalfDiT1d":
            return _half_dit_reason(clf, x_shape)
        return _half_janner_reason(clf, x_shape)
    if name == "MSEClassifier":
        if net_name != "MLPNNClassifier":
            return f"classifier network {net_name} (MLPNNClassifier only)"
        return _mlp_classifier_reason(clf, x_shape, cond_cg, mse=True)
    if name == "QGPOClassifier":
        return _qgpo_reason(clf, x_shape, cond_cg)
    return f"classifier {name} (CumRewClassifier, MSEClassifier or QGPOClassifier only)"


def lower_classifier_grad(p: Program, clf, x: View) -> View:
    """Append the input gradient d sum(logp) / d x of a classifier ``guidable`` accepted to the iteration program -> the gradient
    as a view shaped like ``x`` (its channels may include x's zero padding)"""
    if type(clf).__name__ == "QGPOClassifier":
        return lower_qgpo_grad(p, clf, x)
    if type(clf.model_ema).__name__ == "MLPNNClassifier":
        return lower_mlp_classifier_grad(p, clf, x)
    if type(clf.model_ema).__name__ == "HalfDiT1d":
        return lower_half_dit_grad(p, clf, x)
    return lower_half_janner_grad(p, clf, x)


def _half_janner_reason(clf, x_shape) -> Optional[str]:
    net = getattr(clf, "model_ema", None)
    if type(net).__name__ != "HalfJannerUNet1d":
        return f"classifier network {type(net).__name__} (HalfJannerUNet1d or MLPNNClassifier only)"
    if net.training:
        return "classifier model_ema in train mode"
    if len(x_shape) != 2 or x_shape[0] & (x_shape[0] - 1):
        return "classifier horizon must be 2^n"
    blocks = [b for s in net.downs for b in (s[0], s[1])] + [net.mid_block1[0], net.mid_block2[0]]
    if not all(_is_groupnorm(b.conv1[1]) and _is_groupnorm(b.conv2[1]) for b in blocks):
        return "classifier norm_type other than groupnorm"
    if blocks[0].conv1[0].in_channels != x_shape[1]:
        return "classifier in_dim does not match x"
    L = max(x_shape[0] >> (len(net.downs) + 1), 1)
    if net.final_block[0].in_features != L * blocks[-1].conv1[0].out_channels + net.map_emb[2].out_features:
        return "classifier final_block does not match its feature map"
    return None


def _qgpo_layers(net):
    """(hidden Linears, output Linear) of QGPONNClassifier.mlp when it is Linear + SiLU stages under an out_dim-1 Linear and an
    identity, else None"""
    seq = getattr(getattr(net, "mlp", None), "mlp", None)
    if not isinstance(seq, nn.Sequential) or len(seq) < 3 or type(seq[-1]).__name__ != "Identity":
        return None
    stages, out = list(seq)[:-2], seq[-2]
    if not isinstance(out, nn.Linear) or out.out_features != 1:
        return None
    if not all(isinstance(s, nn.Sequential) and len(s) == 2 and isinstance(s[0], nn.Linear) and type(s[1]).__name__ == "SiLU"
               for s in stages):
        return None
    return [s[0] for s in stages], out


def _qgpo_reason(clf, x_shape, cond_cg) -> Optional[str]:
    net = getattr(clf, "model_ema", None)
    if type(net).__name__ != "QGPONNClassifier":
        return f"classifier network {type(net).__name__} (QGPONNClassifier only)"
    if net.training:
        return "classifier model_ema in train mode"
    obs, act = getattr(net, "obs_proj", None), getattr(net, "act_proj", None)
    if not isinstance(obs, nn.Linear) or not isinstance(act, nn.Linear) or obs.out_features != act.out_features:
        return "classifier obs_proj / act_proj are not Linears of one width"
    layers = _qgpo_layers(net)
    if layers is None:
        return "classifier mlp is not Linear + SiLU layers under an out_dim-1 Linear"
    if layers[0][0].in_features <= 2 * act.out_features:
        return "classifier mlp input has no time-embedding columns"
    if len(x_shape) != 1 or x_shape[0] != act.in_features:
        return "classifier act_proj does not match x"
    if cond_cg is None:
        return "no classifier condition (condition_cg=None)"
    if cond_cg.dim() != 2 or cond_cg.shape[1] != obs.in_features:
        return "classifier condition does not match obs_proj"
    return None


# hidden activations the lowered Linear stacks fuse into CDS_OP_STASH / CDS_OP_DGRAD
_STACK_ACTS = {"ReLU": cabi.ACT_RELU, "SiLU": cabi.ACT_SILU, "Mish": cabi.ACT_MISH}


def _mlp_classifier_layers(net):
    """(hidden Linears, activation module type name, output Linear, out_activation type name) of MLPNNClassifier.mlp, or a
    string saying which part is not an Mlp of Linear + activation stages under a Linear and an output activation"""
    seq = getattr(getattr(net, "mlp", None), "mlp", None)
    if not isinstance(seq, nn.Sequential) or len(seq) < 2 or not isinstance(seq[-2], nn.Linear):
        return "classifier mlp is not an Mlp"
    stages = list(seq)[:-2]
    if not stages:
        return "classifier mlp has no hidden layer"
    if not all(isinstance(s, nn.Sequential) and len(s) == 2 and isinstance(s[0], nn.Linear) for s in stages):
        return "classifier mlp hidden stages are not Linear + activation"
    acts = sorted({type(s[1]).__name__ for s in stages})
    if len(acts) != 1:
        return f"classifier hidden activations differ ({', '.join(acts)})"
    return [s[0] for s in stages], acts[0], seq[-2], type(seq[-1]).__name__


def _emb_width(net) -> int:
    """width of net.map_noise's output (the time-embedding columns of the first Linear)"""
    dev = next(net.parameters()).device
    with torch.no_grad():
        return int(net.map_noise(torch.zeros(1, device=dev)).shape[-1])


def _mlp_classifier_reason(clf, x_shape, cond_cg, mse: bool) -> Optional[str]:
    net = clf.model_ema
    if net.training:
        return "classifier model_ema in train mode"
    layers = _mlp_classifier_layers(net)
    if isinstance(layers, str):
        return layers
    hidden, act, lin_o, out_act = layers
    if act not in _STACK_ACTS:
        return f"classifier activation {act} (ReLU, SiLU or Mish only)"
    if out_act != "Identity":
        return f"classifier out_activation {out_act} (Identity only)"
    if any(a.out_features != b.in_features for a, b in zip(hidden, hidden[1:] + [lin_o])):
        return "classifier mlp widths do not chain"
    if len(x_shape) != 1 or hidden[0].in_features != x_shape[0] + _emb_width(net):
        return "classifier x_dim does not match x"
    if not mse:
        return None if lin_o.out_features == 1 else f"classifier out_dim {lin_o.out_features} (1 only under CumRewClassifier)"
    if cond_cg is None:
        return "no classifier condition (condition_cg=None)"
    if cond_cg.dim() != 2 or cond_cg.shape[1] != lin_o.out_features:
        return "classifier condition is not (batch, out_dim)"
    return None


def _gn(p: Program, h: View, gn: nn.Module, out: View, vec: Optional[cabi.Vec] = None, res: Optional[View] = None):
    """CDS_OP_GN: out = Mish(GroupNorm(h) gamma + beta) [+ vec] [+ res]"""
    op = cabi.Op()
    op.kind = cabi.OP_GN
    g = op.u.gn
    g.batch, g.L, g.C, g.groups, g.eps, g.act = p.rows, h.L, h.C, int(gn.num_groups), float(gn.eps), cabi.ACT_MISH
    g.h, g.h_bstride, g.h_lstride = h.ptr, h.bstride, h.lstride
    g.gamma, g.beta = p.packed(lambda: gn.weight).data_ptr(), p.packed(lambda: gn.bias).data_ptr()
    if vec is not None:
        g.vec = vec
    if res is not None:
        g.res, g.res_bstride, g.res_lstride = res.ptr, res.bstride, res.lstride
    g.out, g.out_bstride, g.out_lstride, g.out_dtype = out.ptr, out.bstride, out.lstride, out.dtype
    p.ops.append(op)
    return out


def _gn_bwd(p: Program, h: View, gn: nn.Module, dout: View, dh: View):
    """CDS_OP_GN_BWD: dh = d h of Mish(GroupNorm(h) gamma + beta) given the output gradient dout"""
    op = cabi.Op()
    op.kind = cabi.OP_GN_BWD
    g = op.u.gn_bwd
    g.batch, g.L, g.C, g.groups, g.eps, g.act = p.rows, h.L, h.C, int(gn.num_groups), float(gn.eps), cabi.ACT_MISH
    g.h, g.h_bstride, g.h_lstride = h.ptr, h.bstride, h.lstride
    g.gamma, g.beta = p.packed(lambda: gn.weight).data_ptr(), p.packed(lambda: gn.bias).data_ptr()
    g.dout, g.dout_bstride, g.dout_lstride = dout.ptr, dout.bstride, dout.lstride
    g.dh, g.dh_bstride, g.dh_lstride, g.dh_dtype = dh.ptr, dh.bstride, dh.lstride, dh.dtype
    p.ops.append(op)
    return dh


def _as_conv(make: Callable[[], torch.Tensor]) -> WSpec:
    """WSpec of a weight given as a Conv1d weight [C_out, C_in, taps] (packed like ``w_conv``)"""
    return WSpec(lambda: (lambda w: w.permute(2, 1, 0).reshape(-1, w.shape[0]))(make()), lambda: make().permute(2, 0, 1))


def w_conv_dgrad(conv: nn.Conv1d, cin: Optional[int] = None) -> WSpec:
    """Data gradient of a stride-1 Conv1d(k, padding k // 2) as a conv of the output gradient with the same padding:
    W'[c_in][c_out][tap] = W[c_out][c_in][k - 1 - tap] (input channels zero-padded to ``cin``: their gradient is zero)."""
    return _as_conv(lambda: _pad_cin(conv.weight, cin).permute(1, 0, 2).flip(2))


def w_down_dgrad(conv: nn.Conv1d) -> WSpec:
    """Data gradient of Downsample1d (k = 3, stride 2, padding 1, L_in = 2 L_out) as ``w_convT``'s two-phase 3-tap form:
    dx[2m] = W1^T d[m]  (phase 0, tap 1),   dx[2m+1] = W2^T d[m] + W0^T d[m+1]  (phase 1, taps 1 and 2)."""
    def make():                                              # [3][C_out of the conv = gradient input][2 * C_in]
        w = conv.weight                                      # [Cout, Cin, 3]
        cout, cin, _ = w.shape
        q = torch.zeros(3, cout, 2 * cin, device=w.device, dtype=w.dtype)
        q[1, :, :cin] = w[:, :, 1]
        q[1, :, cin:] = w[:, :, 2]
        q[2, :, cin:] = w[:, :, 0]
        return q
    return WSpec(lambda: make().reshape(-1, 2 * conv.weight.shape[1]), lambda: make().permute(0, 2, 1))


def lower_half_janner_grad(p: Program, clf, x: View) -> View:
    """Append the input gradient d sum(logp) / d x of ``clf.model_ema`` (a HalfJannerUNet1d; ``guidable``) at x_t
    to the iteration program -> the gradient as a (rows, horizon, x.C) fp32 view (x.C may include zero padding channels).

    Forward, per ResidualBlock: conv1 -> h1;  m = CDS_OP_GN(h1) + time row;  conv2 -> h2;  [1x1 shortcut conv -> s];
    out = CDS_OP_GN(h2) + shortcut.  The Downsample convs as in the denoiser.  z1 = W1 [flatten(x), emb] + b1 (the emb half and
    b1 are a per-iteration table row; the columns of W1 permuted from the channel-major flatten(1) to the (l, c) order).
    Backward: dz1 = (1 W2) Mish'(z1) and d flatten = dz1 W1 (CDS_OP_DGRAD), then per block in reverse CDS_OP_GN_BWD, conv2's
    data gradient, CDS_OP_GN_BWD, conv1's data gradient with the shortcut's added in the same CDS_OP_CONV.  Final Linear2's
    value is not needed for the gradient."""
    net = clf.model_ema
    R = p.rows
    stages = [(s[0], s[1], s[2]) for s in net.downs] + [(net.mid_block1[0], None, net.mid_block1[1]),
                                                         (net.mid_block2[0], None, net.mid_block2[1])]
    blocks = [b for st in stages for b in st[:2] if b is not None]
    widths = [b.emb_mlp[1].out_features for b in blocks]
    offs = [sum(widths[:i]) for i in range(len(widths))]
    lin1, lin2 = net.final_block[0], net.final_block[2]
    f2 = lin1.out_features
    table = p.buf(p.n_iters, sum(widths) + f2)

    def fill(ctx):
        emb = net.map_emb(net.map_noise(ctx.t_all))
        fc = lin1.in_features - emb.shape[1]
        table.copy_(torch.cat([b.emb_mlp(emb) for b in blocks] + [F.linear(emb, lin1.weight[:, fc:], lin1.bias)], dim=1))
    fill.time_only = True
    p.per_call.append(fill)
    row_of = {id(b): _vec(step=table, col=o) for b, o in zip(blocks, offs)}

    # ---- forward
    tape = []                                    # ("block", blk, x, h1, h2, k) / ("down", conv, x) in forward order
    h = x
    for res1, res2, down in stages:
        for blk in (res1, res2):
            if blk is None:
                continue
            k = blk.conv1[0].kernel_size[0]
            c1, c2, C = blk.conv1[0], blk.conv2[0], blk.conv1[0].out_channels
            h1, m, h2, out = p.act(h.L, C), p.act(h.L, C), p.act(h.L, C), p.act(h.L, C)
            p.conv(h, w_conv(c1, h.C), h1, taps=k, pad=k // 2, bias=_const_vec(p.packed(lambda c=c1: c.bias)))
            _gn(p, h1, blk.conv1[1], m, vec=row_of[id(blk)])
            p.conv(m, w_conv(c2), h2, taps=k, pad=k // 2, bias=_const_vec(p.packed(lambda c=c2: c.bias)))
            if isinstance(blk.residual_conv, nn.Conv1d):
                rc = blk.residual_conv
                res = p.conv(h, w_rows(lambda r=rc, cin=h.C: _pad_cin(r.weight, cin)[:, :, 0]), p.act(h.L, C),
                           bias=_const_vec(p.packed(lambda r=rc: r.bias)))
            else:
                res = h
            _gn(p, h2, blk.conv2[1], out, res=res)
            tape.append(("block", blk, h, h1, h2, k))
            h = out
        if not isinstance(down, nn.Identity):
            out = p.act((h.L + 1) // 2, h.C)
            p.conv(h, w_conv(down.conv), out, taps=3, stride=2, pad=1, bias=_const_vec(p.packed(lambda d=down: d.conv.bias)))
            tape.append(("down", down.conv, h))
            h = out
    fc = h.L * h.C
    z1 = View(p.buf(R, 1, f2), 1, f2)
    w1 = lambda: lin1.weight[:, :fc].reshape(f2, h.C, h.L).permute(0, 2, 1).reshape(f2, fc)     # noqa: E731
    p.conv(View(h.t, 1, fc, h.offset, h.bstride, fc, h.tf32), w_rows(w1), z1, bias=_vec(step=table, col=sum(widths)))

    # ---- backward
    ones = p.buf(R, lin2.out_features)
    ones.fill_(1.0)
    dz1, dflat = p.buf(R, f2), p.buf(R, h.L, h.C)
    for dz, w, n, k, z, out in ((ones, p.packed(lambda: lin2.weight), lin2.out_features, f2, z1, dz1),
                                (dz1, p.packed(w1), f2, fc, None, dflat)):
        op = cabi.Op()
        op.kind = cabi.OP_DGRAD
        d = op.u.dgrad
        d.rows, d.N, d.K, d.dz, d.ldz, d.w, d.ldw = R, n, k, dz.data_ptr(), n, w.data_ptr(), k
        if z is not None:
            d.z, d.z_iter_stride, d.act = z.ptr, 0, cabi.ACT_MISH
        d.out, d.ldo = out.data_ptr(), k
        p.ops.append(op)
    g = View(dflat, h.L, h.C)
    for i in range(len(tape) - 1, -1, -1):
        entry = tape[i]
        if entry[0] == "down":
            _, dconv, xin = entry
            dx = p.act(xin.L, xin.C)
            if xin.L == 1:                           # length 1 -> 1: only the centre tap sees the input
                p.conv(g, w_rows(lambda c=dconv: c.weight[:, :, 1].t()), dx)
            else:
                p.conv(g, w_down_dgrad(dconv), dx, taps=3, stride=1, pad=1, phases=2, L_out=g.L)
            g = dx
            continue
        _, blk, xin, h1, h2, k = entry
        C = h1.C
        d2, dm, d1 = p.act(h1.L, C), p.act(h1.L, C), p.act(h1.L, C)
        _gn_bwd(p, h2, blk.conv2[1], g, d2)
        p.conv(d2, w_conv_dgrad(blk.conv2[0]), dm, taps=k, pad=k // 2)
        _gn_bwd(p, h1, blk.conv1[1], dm, d1)
        first = i == 0
        dx = p.act(xin.L, xin.C, torch.float32 if first else None)      # the input gradient itself stays exact fp32
        if isinstance(blk.residual_conv, nn.Conv1d):
            rc = blk.residual_conv
            short = dict(res_conv=(g, w_rows(lambda r=rc, cin=xin.C: _pad_cin(r.weight, cin)[:, :, 0].t()),
                                   lambda cin=xin.C: torch.zeros(cin)))
        else:
            short = dict(res=g)
        p.conv(d1, w_conv_dgrad(blk.conv1[0], xin.C), dx, taps=k, pad=k // 2, **short)
        g = dx
    return g


def _act_stash(p: Program, z: View, out: View, act: int):
    """CDS_OP_STASH without a slot: out = act(z) (dense (rows, L, C) fp32 views)"""
    op = cabi.Op()
    op.kind = cabi.OP_STASH
    s = op.u.stash
    s.n, s.act, s.src, s.act_out = p.rows * z.L * z.C, act, z.ptr, out.ptr
    p.ops.append(op)


def _dgrad(p: Program, dz: torch.Tensor, w: torch.Tensor, out: torch.Tensor, z: Optional[View] = None, act: int = cabi.ACT_NONE):
    """CDS_OP_DGRAD: out = (dz W) act'(z), dz (rows, N), W (N, K) dense, out (rows, K) dense"""
    op = cabi.Op()
    op.kind = cabi.OP_DGRAD
    d = op.u.dgrad
    n, k = w.shape
    d.rows, d.N, d.K, d.dz, d.ldz, d.w, d.ldw = p.rows, n, k, dz.data_ptr(), n, w.data_ptr(), k
    if z is not None:
        d.z, d.z_iter_stride, d.act = z.ptr, 0, act
    d.out, d.ldo = out.data_ptr(), k
    p.ops.append(op)


class _LinearActStack:
    """A stack of hidden Linears z_k = W_k h_{k-1} + b_k, h_k = act(z_k) inside a classifier's input gradient, forward and
    backward, for one activation ``act`` (CDS_ACT_RELU / SILU / MISH).  The pre-activations z_k stay in dense fp32 buffers for
    the backward; every h_k is CDS_OP_STASH without a slot."""

    def __init__(self, p: Program, hidden: List[nn.Linear], act: int):
        self.p, self.hidden, self.act = p, hidden, act
        self.zs: List[View] = []

    def dense(self, width: int) -> View:
        """an exact fp32 (rows, 1, width) activation"""
        return View(self.p.buf(self.p.rows, 1, width), 1, width)

    def forward(self, h: View, first_w: WSpec, first_bias: cabi.Vec, act_last: bool) -> View:
        """z_1 = first_w h + first_bias (the first Linear's columns that read h, its other columns and bias folded into the
        bias rows), z_k (CDS_OP_CONV), h_k = act(z_k) (CDS_OP_STASH) between them and, when ``act_last``, after the last:
        -> h_n, or z_n when not ``act_last``"""
        p = self.p
        for k, lin in enumerate(self.hidden):
            z = self.dense(lin.out_features)
            if k == 0:
                p.conv(h, first_w, z, bias=first_bias)
            else:
                p.conv(h, w_linear(lin.weight), z, bias=_const_vec(p.packed(lambda m=lin: m.bias)))
            self.zs.append(z)
            h = z
            if act_last or k + 1 < len(self.hidden):
                h = self.dense(lin.out_features)
                _act_stash(p, z, h, self.act)
        return h

    def backward(self, seed: torch.Tensor, w_out: torch.Tensor) -> torch.Tensor:
        """dz_n = (seed W_out) act'(z_n), dz_k = (dz_{k+1} W_{k+1}) act'(z_k) (CDS_OP_DGRAD) -> dz_1 (rows, width of z_1)"""
        p = self.p
        up, w_up = seed, w_out
        for k in range(len(self.hidden) - 1, -1, -1):
            dz = p.buf(p.rows, self.hidden[k].out_features)
            _dgrad(p, up, w_up, dz, self.zs[k], self.act)
            up = dz
            if k:
                w_up = p.packed(lambda m=self.hidden[k]: m.weight)
        return up


def lower_qgpo_grad(p: Program, clf, x: View) -> View:
    """Append the input gradient d sum(logp) / d x of ``clf.model_ema`` (a QGPONNClassifier; ``guidable``) at x_t (rows, act_dim)
    to the iteration program -> the gradient as a dense (rows, 1, act_dim) fp32 view.

    logp = 10 tanh(z / 10),  z = W_o h_n + b_o,  h_k = silu(z_k),  z_k = W_k h_{k-1} + b_k,
    z_1 = W_1 [obs_proj(c) | act_proj(x) | map_noise(t)] + b_1 = W_1a act_proj(x) + (W_1e map_noise(t) + b_1) + W_1y obs_proj(c)
    Forward: a = act_proj(x) (CDS_OP_CONV);  z_1 (CDS_OP_CONV, its bias the per-iteration row W_1e e(t) + b_1 plus the
    per-trajectory row W_1y obs_proj(c), both filled once per call);  per hidden layer h_k = silu(z_k) (CDS_OP_STASH without a
    slot) and z_{k+1} (CDS_OP_CONV): the pre-activations stay for the backward (``_LinearActStack``).
    Backward: the seed d logp / d z (CDS_OP_HEAD_GRAD over silu(z_n)), dz_n = (seed W_o) silu'(z_n), ..., dz_1 (CDS_OP_DGRAD
    with SiLU), da = dz_1 W_1a, dx = da W_act (CDS_OP_DGRAD): the reference's factorisation through act_proj, kept so that the
    gradient's summation error stays that of the two products autograd forms."""
    net = clf.model_ema
    R = p.rows
    hidden, lin_o = _qgpo_layers(net)
    lin1 = hidden[0]
    E = net.act_proj.out_features
    step_tab, samp_tab = p.buf(p.n_iters, lin1.out_features), p.buf(R, lin1.out_features)

    def fill_time(ctx):
        step_tab.copy_(F.linear(net.map_noise(ctx.t_all), lin1.weight[:, 2 * E:], lin1.bias))
    fill_time.time_only = True

    def fill_cond(ctx):
        samp_tab.copy_(F.linear(net.obs_proj(ctx.cond_cg.to(torch.float32)), lin1.weight[:, :E]))
    p.per_call += [fill_time, fill_cond]

    stack = _LinearActStack(p, hidden, cabi.ACT_SILU)
    a = p.conv(x, w_linear(net.act_proj.weight), stack.dense(E), bias=_const_vec(p.packed(lambda: net.act_proj.bias)))
    z_n = stack.forward(a, w_linear(lin1.weight, slice(E, 2 * E)), _vec(step_tab, samp_tab), act_last=False)

    seed = p.buf(R, 1)
    op = cabi.Op()
    op.kind = cabi.OP_HEAD_GRAD
    q = op.u.head_grad
    q.rows, q.K, q.h, q.ldh, q.act = R, z_n.C, z_n.ptr, z_n.C, cabi.ACT_SILU
    q.w, q.b = p.packed(lambda: lin_o.weight.reshape(-1)).data_ptr(), p.packed(lambda: lin_o.bias).data_ptr()
    q.scale, q.seed = 10.0, seed.data_ptr()
    p.ops.append(op)

    dz1 = stack.backward(seed, p.packed(lambda: lin_o.weight))
    da = p.buf(R, E)
    _dgrad(p, dz1, p.packed(lambda: lin1.weight[:, E:2 * E]), da)
    dx = View(p.buf(R, 1, x.C), 1, x.C)
    _dgrad(p, da, p.packed(lambda: net.act_proj.weight), dx.t)
    return dx


def lower_mlp_classifier_grad(p: Program, clf, x: View) -> View:
    """Append the input gradient d sum(logp) / d x of ``clf.model_ema`` (an MLPNNClassifier under an MSEClassifier or an
    out_dim-1 CumRewClassifier; ``guidable``) at x_t (rows, x_dim) to the iteration program -> the gradient as a dense
    (rows, 1, x.C) fp32 view (x.C may include zero padding channels, whose gradient is zero).

    y = W_o h_n + b_o,  h_k = act(z_k),  z_k = W_k h_{k-1} + b_k,  z_1 = W_1 [x | map_noise(t)] + b_1 = W_1x x + (W_1e e(t) + b_1)
    Forward (``_LinearActStack``): z_1 (CDS_OP_CONV, its bias the per-iteration row W_1e map_noise(t) + b_1 filled once per
    call), h_k = act(z_k) (CDS_OP_STASH) and z_{k+1} (CDS_OP_CONV).
      CumRew head, logp = y (out_dim 1):  the seed d logp / d y = 1, so y itself is not evaluated and h_n not formed.
      MSE head, logp = -T mean_j (y_j - c_j)^2:  r = W_o h_n + (b_o - c) (CDS_OP_CONV, the per-trajectory bias row b_o - c filled
      per call from condition_cg) and d logp / d y = -(2 T / out_dim) r.  The factor goes into a copy of W_o that every call
      refills (T = clf.temperature, read per call): dz_n = (r (-(2 T / out_dim) W_o)) act'(z_n).
    Backward: dz_n, ..., dz_1 (CDS_OP_DGRAD with act'), dx = dz_1 W_1x (CDS_OP_DGRAD)."""
    net = clf.model_ema
    R = p.rows
    hidden, act, lin_o, _ = _mlp_classifier_layers(net)
    lin1 = hidden[0]
    X = lin1.in_features - _emb_width(net)
    mse = type(clf).__name__ == "MSEClassifier"
    step_tab = p.buf(p.n_iters, lin1.out_features)

    def fill_time(ctx):
        step_tab.copy_(F.linear(net.map_noise(ctx.t_all), lin1.weight[:, X:], lin1.bias))
    fill_time.time_only = True
    p.per_call.append(fill_time)

    w_1x = lambda: _pad_cin(lin1.weight[:, :X], x.C)                                      # noqa: E731
    stack = _LinearActStack(p, hidden, _STACK_ACTS[act])
    h_n = stack.forward(x, w_rows(w_1x), _vec(step=step_tab), act_last=mse)
    if mse:
        D = lin_o.out_features
        target, w_seed = p.buf(R, D), p.buf(D, lin_o.in_features)

        def fill_target(ctx):
            target.copy_(lin_o.bias[None, :] - ctx.cond_cg.to(torch.float32))
            w_seed.copy_(lin_o.weight * (-(2.0 * float(clf.temperature) / D)))
        p.per_call.append(fill_target)
        r = stack.dense(D)
        p.conv(h_n, w_linear(lin_o.weight), r, bias=_vec(sample=target))
        seed = r.t.view(R, D)
    else:
        seed, w_seed = p.buf(R, 1), p.packed(lambda: lin_o.weight)
        seed.fill_(1.0)
    dz1 = stack.backward(seed, w_seed)
    dx = stack.dense(x.C)
    _dgrad(p, dz1, p.packed(w_1x), dx.t.view(R, x.C))
    return dx


# =============================================================================== HalfDiT1d's input gradient
HALF_DIT_HEAD_DIMS = (16, 32, 64)          # the head_dim CDS_OP_ATTN's backward mode covers
HALF_DIT_MAX_L = 128                       # the longest horizon CDS_OP_ATTN's backward mode covers


def _affine_ln(m) -> bool:
    return isinstance(m, nn.LayerNorm) and m.elementwise_affine and m.bias is not None and len(m.normalized_shape) == 1


def _half_dit_reason(clf, x_shape) -> Optional[str]:
    net = clf.model_ema
    if net.training:
        return "classifier model_ema in train mode"
    if len(x_shape) != 2 or x_shape[1] != net.x_proj.in_features:
        return "classifier in_dim does not match x"
    d, heads = net.d_model, net.blocks[0].attn.num_heads
    if d % heads or d // heads not in HALF_DIT_HEAD_DIMS:
        return f"classifier head_dim {d / heads:g} (16, 32 or 64 only)"
    if x_shape[0] > HALF_DIT_MAX_L:
        return f"classifier horizon {x_shape[0]} (at most {HALF_DIT_MAX_L})"
    fl, proj = getattr(net, "final_layer", None), getattr(net, "proj", None)
    ok = isinstance(proj, nn.Sequential) and len(proj) == 6 and \
        [type(m).__name__ for m in proj] == ["LayerNorm", "SiLU", "Linear", "LayerNorm", "SiLU", "Linear"] and \
        _affine_ln(proj[0]) and _affine_ln(proj[3]) and isinstance(getattr(fl, "linear", None), nn.Linear) and \
        isinstance(getattr(fl, "norm_final", None), nn.LayerNorm) and not fl.norm_final.elementwise_affine and \
        fl.linear.in_features == d and proj[0].normalized_shape[0] == fl.linear.out_features == proj[2].in_features and \
        proj[3].normalized_shape[0] == proj[2].out_features == proj[5].in_features
    return None if ok else "classifier proj / final_layer without the reference's structure"


def _lnmod_bwd(p: Program, x: View, scale: torch.Tensor, scale_col: int, eps: float, dout: View, dx: View,
               res: Optional[View] = None, gate_col: Optional[int] = None, gated: Optional[View] = None,
               mod_bstride: Optional[int] = None):
    """CDS_OP_LNMOD in backward mode: dx = d x of LN(x) (1 + scale) + shift given dout [+ res]; gated = gate * dx (gate: column
    ``gate_col`` of the same table).  ``scale``: a [rows, W] table (mod_bstride = its row stride) or one row (mod_bstride 0)."""
    op = cabi.Op()
    op.kind = cabi.OP_LNMOD
    m = op.u.lnmod
    m.batch, m.L, m.C, m.eps = p.rows, x.L, x.C, float(eps)
    m.in_ = x.ptr
    m.scale = scale.data_ptr() + 4 * int(scale_col)
    m.mod_bstride = scale.stride(0) if mod_bstride is None else mod_bstride
    m.dout, m.dout_bstride, m.dout_lstride = dout.ptr, dout.bstride, dout.lstride
    if res is not None:
        m.res = res.ptr
    m.out, m.out_dtype = dx.ptr, dx.dtype
    if gated is not None:
        m.gate, m.gate_bstride = scale.data_ptr() + 4 * int(gate_col), m.mod_bstride
        m.gated, m.gated_dtype = gated.ptr, gated.dtype
    p.ops.append(op)
    return dx


def lower_half_dit_grad(p: Program, clf, x: View) -> View:
    """Append the input gradient d sum(logp) / d x of ``clf.model_ema`` (a HalfDiT1d; ``guidable``) at x_t (rows, horizon, x.C)
    to the iteration program -> the gradient as a (rows, horizon, x.C) fp32 view (x.C may include zero padding channels).

    logp = proj(mean_L(FinalLayer1d(X_D, emb))),  X_{i+1} = DiTBlock_i(X_i, emb),  X_0 = x_proj(x) + pos;  emb depends on t only
    (CumRewClassifier.logp passes no condition), so the adaLN table is DiT1d's conditioning path with a zero condition.
    Forward: the blocks of ``lower_dit`` (``_dit_block``), each keeping X_i, X1_i, QKV_i and the GELU pre-activation H_i;
    the final LN + modulate; mean_L and the final Linear as one GEMM over the flattened tokens (the weight tiled L times, / L);
    proj's LayerNorms as CDS_OP_LNMOD with the [gamma - 1 | beta] table, SiLU as CDS_OP_STASH.
    Backward, seeded with ones for every out_dim: proj through CDS_OP_DGRAD (SiLU') and CDS_OP_LNMOD's backward mode; the final
    Linear's data gradient is one row per trajectory (CDS_OP_DGRAD with W / L), which the final LayerNorm backward reads
    broadcast over the horizon.  Per block, in reverse (g = the gated copy the LayerNorm backward before it wrote):
        dH  = (g_m dX2) W2 (token GEMM);  dH' = dH gelu_tanh'(H) (CDS_OP_STASH, backward mode);  dY2 = dH' W1 (token GEMM)
        dX1 = dX2 + LNmod_bwd(X1; dY2), and g_a dX1           (CDS_OP_LNMOD, backward mode)
        dA  = (g_a dX1) W_out;  dQKV = attn_bwd(QKV; dA) (CDS_OP_ATTN, backward mode)
        dY1 = dX1 + dQKV W_in (token GEMM + residual)
        dX  = LNmod_bwd(X; dY1), and g_m of the block before times dX
    then dx = dX_0 W_x.  The token GEMMs are ``Program.token_linear`` with the transposed weights (wgmma on tensor-core programs
    where the kernel takes them)."""
    net = clf.model_ema
    R, L, d = p.rows, x.L, net.d_model
    heads, depth = net.blocks[0].attn.num_heads, len(net.blocks)
    fl, proj = net.final_layer, net.proj
    f32 = torch.float32
    mod2d, pos = _dit_conditioning(p, net, L, False)

    # ---- forward, keeping what the backward reads
    Xs = [p.act(L, d, f32) for _ in range(depth + 1)]
    X1s = [p.act(L, d, f32) for _ in range(depth)]
    QKVs = [p.act(L, 3 * d) for _ in range(depth)]                   # fp32 storage on fp32 / TF32 programs
    Hs = [p.act(L, 4 * d, f32) for _ in range(depth)]
    Y, ATT, HID = p.act(L, d), p.act(L, d), p.act(L, 4 * d)
    pos_v = View(pos, L, d, bstride=0)
    if x.C != net.x_proj.in_features or x.tf32 or not p.tc:
        # x_t as the denoiser reads it (the channel-padded copy of a tensor-core program, else x_t itself)
        p.token_linear(x, w_rows(lambda: _pad_cin(net.x_proj.weight, x.C)), Xs[0],
                       bias=_const_vec(p.packed(lambda: net.x_proj.bias)), res=pos_v)
    else:
        _embed_tokens(p, x, net.x_proj, pos_v, Xs[0], 0)
    for i, blk in enumerate(net.blocks):
        _dit_block(p, blk, mod2d, 6 * d * i, heads, Xs[i], Y, QKVs[i], ATT, HID, X1s[i], Xs[i + 1], hpre=Hs[i])
    o = 6 * d * depth
    p.lnmod(Xs[depth], Y, mod2d, o, o + d, fl.norm_final.eps)
    d2, d4 = fl.linear.out_features, proj[2].out_features

    def dense(width):
        return View(p.buf(R, 1, width), 1, width)
    feat = dense(d2)                                                 # mean_L(final_layer(X_D))
    p.conv(View(Y.t, 1, L * d, Y.offset, Y.bstride, L * d, Y.tf32), w_rows(lambda: fl.linear.weight.repeat(1, L) / L), feat,
           bias=_const_vec(p.packed(lambda: fl.linear.bias)))
    ln_tabs = [p.packed(lambda m=m: torch.cat([m.weight - 1., m.bias])[None]) for m in (proj[0], proj[3])]
    z0, h0, z1, z1n = dense(d2), dense(d2), dense(d4), dense(d4)
    p.lnmod(feat, z0, ln_tabs[0].expand(R, 2 * d2), d2, 0, proj[0].eps)
    _act_stash(p, z0, h0, cabi.ACT_SILU)
    p.conv(h0, w_linear(proj[2].weight), z1, bias=_const_vec(p.packed(lambda: proj[2].bias)))
    p.lnmod(z1, z1n, ln_tabs[1].expand(R, 2 * d4), d4, 0, proj[3].eps)

    # ---- backward
    ones = p.buf(R, proj[5].out_features)
    ones.fill_(1.0)
    dz1n, dz1, dz0, dfeat, drow = p.buf(R, d4), dense(d4), p.buf(R, d2), dense(d2), dense(d)
    _dgrad(p, ones, p.packed(lambda: proj[5].weight), dz1n, z1n, cabi.ACT_SILU)
    _lnmod_bwd(p, z1, ln_tabs[1], 0, proj[3].eps, View(dz1n, 1, d4), dz1, mod_bstride=0)
    _dgrad(p, dz1.t.view(R, d4), p.packed(lambda: proj[2].weight), dz0, z0, cabi.ACT_SILU)
    _lnmod_bwd(p, feat, ln_tabs[0], 0, proj[0].eps, View(dz0, 1, d2), dfeat, mod_bstride=0)
    _dgrad(p, dfeat.t.view(R, d2), p.packed(lambda: fl.linear.weight / L), drow.t.view(R, d))

    G = p.act(L, d)                                                  # a gated gradient: the input of a data-gradient GEMM
    dH, dHp, dY = p.act(L, 4 * d, f32), p.act(L, 4 * d, f32), p.act(L, d, f32)
    dXa, dXb, dA, dQKV = p.act(L, d, f32), p.act(L, d, f32), p.act(L, d, f32), p.act(L, 3 * d)
    g_m = lambda i: 6 * d * i + 5 * d                                # noqa: E731
    _lnmod_bwd(p, Xs[depth], mod2d, o + d, fl.norm_final.eps, View(drow.t, L, d, bstride=d, lstride=0), dXa,
               gate_col=g_m(depth - 1), gated=G)
    for i in range(depth - 1, -1, -1):
        blk, at, ob = net.blocks[i], net.blocks[i].attn, 6 * d * i
        p.token_linear(G, w_rows(lambda b=blk: b.mlp[3].weight.t()), dH)
        op = cabi.Op()
        op.kind = cabi.OP_STASH                                      # backward mode: dH' = dH gelu_tanh'(H)
        a = op.u.stash
        a.n, a.act, a.src, a.grad, a.act_out = R * L * 4 * d, cabi.ACT_GELU_TANH, Hs[i].ptr, dH.ptr, dHp.ptr
        p.ops.append(op)
        p.token_linear(dHp, w_rows(lambda b=blk: b.mlp[0].weight.t()), dY)
        _lnmod_bwd(p, X1s[i], mod2d, ob + 4 * d, blk.norm2.eps, dY, dXb, res=dXa, gate_col=ob + 2 * d, gated=G)
        p.token_linear(G, w_rows(lambda m=at: m.out_proj.weight.t()), dA)
        op = cabi.Op()
        op.kind = cabi.OP_ATTN                                       # backward mode: d q|k|v from q|k|v and d out
        b = op.u.attn
        b.batch, b.L, b.C, b.heads = R, L, d, heads
        b.qkv, b.qkv_dtype, b.dout, b.out, b.out_dtype = QKVs[i].ptr, QKVs[i].dtype, dA.ptr, dQKV.ptr, dQKV.dtype
        p.ops.append(op)
        p.token_linear(dQKV, w_rows(lambda m=at: m.in_proj_weight.t()), dY, res=dXb)
        gate = dict(gate_col=g_m(i - 1), gated=G) if i else {}
        _lnmod_bwd(p, Xs[i], mod2d, ob + d, blk.norm1.eps, dY, dXa, **gate)
    dx = p.act(L, x.C, f32)
    p.token_linear(dXa, w_rows(lambda: _pad_cin(net.x_proj.weight, x.C).t()), dx)
    return dx                  # (token_linear returns the flattened view of a tensor-core program)


def guide(p: Program, pred: View, g: View, scale: torch.Tensor):
    """CDS_OP_GUIDE: pred += scale[iter] * g  (pred dense fp32)"""
    assert pred.lstride == pred.C and pred.bstride == pred.L * pred.C and pred.t.dtype == torch.float32
    op = cabi.Op()
    op.kind = cabi.OP_GUIDE
    q = op.u.guide
    q.batch, q.L, q.C, q.pred = p.rows, pred.L, pred.C, pred.ptr
    q.g, q.g_bstride, q.g_lstride, q.s = g.ptr, g.bstride, g.lstride, scale.data_ptr()
    p.ops.append(op)
