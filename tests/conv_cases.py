"""TEST INFRASTRUCTURE: the operator-level case table of CDS_OP_CONV and the code that turns a case into a descriptor.

Every case is a plain dict that names the kernel instantiation it is meant to reach (``want``, in the form
``choice_key`` gives ``cabi.conv_choice``).  tests/test_conv_dispatch_cpu.py checks on the CPU that each case reaches
its variant and that the table covers every instantiation the dispatcher can select; tests/test_conv_kernels_gpu.py
runs every case through ``cds_run_op`` on the GPU against tests/opref.py.

Buffers: every tensor is a view into a larger buffer whose gaps hold NaN -- one extra trajectory past the rows the op
may read (or write), and for ``strided`` cases a 32-channel margin on both sides of the channel slice plus one spare
position per trajectory (bstride > L * lstride), which is how the UNet concatenations lay out their halves.
"""
import torch

from cleandiffuser_b200.engine import cabi

MATH = {"bf16": cabi.MATH_BF16_TC, "tf32": cabi.MATH_TF32_TC, "fp32": cabi.MATH_FP32}
_ACT_DT = {"bf16": cabi.BF16, "tf32": cabi.TF32, "fp32": cabi.F32}
TORCH_DT = {cabi.F32: torch.float32, cabi.TF32: torch.float32, cabi.BF16: torch.bfloat16}
MARGIN = 32                                # channels of NaN on each side of a strided view


def tc(kc, n, split, has_res, tf32):
    return ("tc", kc, n, split, bool(has_res), bool(tf32))


def ps(n, has_res, tf32):
    return ("ps", n, bool(has_res), bool(tf32))


def simt(bn):
    return ("simt", bn)


def choice_key(ch):
    """cabi.conv_choice() dict -> the tuple form of ``want``"""
    if ch["family"] == "simt":
        return simt(ch["bn"])
    if ch["family"] == "ps":
        return ps(ch["n"], ch["has_res"], ch["tf32"])
    return tc(ch["kc"], ch["n"], ch["split"], ch["has_res"], ch["tf32"])


def case(name, math, B, L, C_in, C_out, want, **kw):
    c = dict(name=name, math=math, B=B, L=L, C_in=C_in, C_out=C_out, want=want, taps=1, stride=1, phases=1, groups=0,
             act=cabi.ACT_NONE, bias="step", film=None, res=None, res_C=None, in_mod=0, res_mod=0, srd=0,
             in_dtype=_ACT_DT[math], out_dtype=_ACT_DT[math], strided=False, offset=0.0, seed=0)
    c.update(kw)
    if c["res"] == "conv" and c["res_C"] is None:
        c["res_C"] = C_in
    return c


GN = dict(groups=8, act=cabi.ACT_MISH)
TRAJ = dict(film="traj")                    # ChiUNet FiLM: per-trajectory scale and shift
M = cabi.ACT_MISH
R3 = 3 * 2 * 132                            # 3 tiles for each of at most 2 x 132 resident CTAs

CASES = [
    # ---- conv_tc, bf16: KC 64 (C_in % 64 == 0) / KC 32 --------------------------------------------------------------
    case("bf16_head3_k64", "bf16", 37, 32, 64, 3, tc(64, 16, 1, 0, 0), out_dtype=cabi.F32),
    case("bf16_head14_k32", "bf16", 37, 16, 32, 14, tc(32, 16, 1, 0, 0), out_dtype=cabi.F32, strided=True),
    case("bf16_head29_k64", "bf16", 21, 8, 128, 29, tc(64, 32, 1, 0, 0), out_dtype=cabi.F32, bias=None),
    case("bf16_head29_k32", "bf16", 5, 32, 96, 29, tc(32, 32, 1, 0, 0), out_dtype=cabi.F32),
    case("bf16_c32_gn_k64", "bf16", 77, 32, 64, 32, tc(64, 32, 1, 0, 0), taps=5, **GN),
    case("bf16_c32_gn_res_k32", "bf16", 77, 16, 32, 32, tc(32, 32, 1, 1, 0), taps=3, res="conv", res_C=32, **GN),
    case("bf16_c32_shortcut_k64", "bf16", 40, 32, 64, 32, tc(64, 32, 1, 1, 0), taps=5, res="conv", **GN, **TRAJ),
    case("bf16_c64_split_k64", "bf16", 99, 8, 64, 64, tc(64, 32, 2, 0, 0), taps=5, **GN, film="shift", strided=True),
    case("bf16_c64_split_res_k64", "bf16", 61, 16, 128, 64, tc(64, 32, 2, 1, 0), taps=5, res="conv", **GN, **TRAJ),
    case("bf16_c64_split_k32", "bf16", 50, 4, 32, 64, tc(32, 32, 2, 0, 0), taps=3, **GN, res="id"),
    case("bf16_c64_split_res_k32", "bf16", 50, 32, 96, 64, tc(32, 32, 2, 1, 0), taps=3, res="conv", **GN),
    case("bf16_c64_whole_k64_3tiles", "bf16", R3 * 128 // 32 + 7, 32, 64, 64, tc(64, 64, 1, 0, 0), taps=5, **GN, **TRAJ,
         res="id"),
    case("bf16_c64_whole_res_k64", "bf16", 2200, 16, 64, 64, tc(64, 64, 1, 1, 0), taps=5, res="conv", **GN),
    case("bf16_c64_whole_k32", "bf16", 9000, 4, 32, 64, tc(32, 64, 1, 0, 0), taps=3, **GN, res="id", strided=True),
    case("bf16_c64_whole_res_k32", "bf16", 4500, 8, 32, 64, tc(32, 64, 1, 1, 0), taps=1, res="conv", **GN),
    case("bf16_c128_k64", "bf16", 45, 8, 128, 128, tc(64, 64, 2, 0, 0), taps=5, **GN, **TRAJ, res="id"),
    case("bf16_c128_res_k64", "bf16", 45, 16, 64, 128, tc(64, 64, 2, 1, 0), taps=5, res="conv", **GN, **TRAJ),
    case("bf16_c128_k32", "bf16", 33, 2, 32, 128, tc(32, 64, 2, 0, 0), taps=3, **GN),
    case("bf16_c128_res_k32", "bf16", 33, 4, 128, 128, tc(32, 64, 2, 1, 0), taps=3, res="conv", res_C=32, **GN),
    case("bf16_c256_k64", "bf16", 45, 4, 256, 256, tc(64, 128, 2, 0, 0), taps=5, **GN, **TRAJ, res="id"),
    case("bf16_c256_res_k64", "bf16", 45, 8, 128, 256, tc(64, 128, 2, 1, 0), taps=5, res="conv", **GN, **TRAJ),
    case("bf16_c256_k32", "bf16", 17, 1, 32, 256, tc(32, 128, 2, 0, 0), taps=1, **GN),
    case("bf16_c256_res_k32", "bf16", 17, 2, 96, 256, tc(32, 128, 2, 1, 0), taps=3, res="conv", **GN),
    case("bf16_c512_gn", "bf16", 45, 4, 256, 512, tc(64, 256, 2, 0, 0), taps=5, **GN, **TRAJ, res="id"),
    case("bf16_c512_gn_res", "bf16", 45, 4, 256, 512, tc(64, 128, 4, 1, 0), taps=5, res="conv", **GN, **TRAJ),
    case("bf16_c1024_gn", "bf16", 30, 2, 512, 1024, tc(64, 256, 4, 0, 0), taps=5, **GN, **TRAJ, res="id"),
    case("bf16_c1024_gn_res", "bf16", 30, 2, 512, 1024, tc(64, 128, 8, 1, 0), taps=3, res="conv", **GN, **TRAJ),
    # transposed (phases 2), stride 2, runtime column tiles
    case("bf16_convT_c32", "bf16", 37, 8, 64, 32, tc(64, 64, 1, 0, 0), taps=3, phases=2, act=M),
    case("bf16_convT_c64", "bf16", 37, 4, 128, 64, tc(64, 128, 1, 0, 0), taps=3, phases=2, film="shift", strided=True),
    case("bf16_convT_c128", "bf16", 37, 16, 32, 128, tc(32, 256, 1, 0, 0), taps=3, phases=2),
    case("bf16_stride2_c64", "bf16", 37, 8, 64, 64, tc(64, 32, 2, 0, 0), taps=3, stride=2, **GN),
    case("bf16_stride2_c128_k32", "bf16", 37, 16, 32, 128, tc(32, 64, 2, 0, 0), taps=3, stride=2, **GN, strided=True),
    case("bf16_lin320", "bf16", 3700, 1, 128, 320, tc(64, 160, 1, 0, 0), srd=100, act=cabi.ACT_GELU_TANH, bias="both"),
    case("bf16_lin384", "bf16", 640, 1, 64, 384, tc(64, 192, 1, 0, 0), act=cabi.ACT_SILU),
    case("bf16_lin384_k32", "bf16", 640, 1, 96, 384, tc(32, 128, 1, 0, 0), act=cabi.ACT_GELU_ERF),
    case("bf16_lin384_res_k32", "bf16", 640, 1, 96, 384, tc(32, 128, 1, 1, 0), res="conv"),
    case("bf16_lin896_res_k64", "bf16", 300, 1, 64, 896, tc(64, 128, 1, 1, 0), res="conv"),
    case("bf16_lin960", "bf16", 3700, 1, 320, 960, tc(64, 192, 1, 0, 0), srd=100, act=cabi.ACT_MISH_SILU, film="traj"),
    case("bf16_lin960_k32", "bf16", 700, 1, 32, 960, tc(32, 64, 1, 0, 0), act=cabi.ACT_LEAKY_RELU),
    case("bf16_lin1280", "bf16", 3700, 1, 320, 1280, tc(64, 256, 1, 0, 0), srd=100, film="gate", res="id"),
    case("bf16_lin1280_k32", "bf16", 700, 1, 32, 1280, tc(32, 256, 1, 0, 0), srd=50, bias="sample"),
    case("bf16_lin640", "bf16", 500, 1, 64, 640, tc(64, 160, 1, 0, 0)),
    # ---- conv_tc, TF32: KC 64 (C_in % 32 == 0) / KC 32 (C_in % 16 == 0) ----------------------------------------------
    case("tf32_head3_k64", "tf32", 37, 32, 32, 3, tc(64, 16, 1, 0, 1), out_dtype=cabi.F32),
    case("tf32_head14_k32", "tf32", 37, 16, 16, 14, tc(32, 16, 1, 0, 1), out_dtype=cabi.F32, strided=True),
    case("tf32_head29_k64", "tf32", 21, 8, 64, 29, tc(64, 32, 1, 0, 1), out_dtype=cabi.F32),
    case("tf32_head29_k32", "tf32", 21, 32, 48, 29, tc(32, 32, 1, 0, 1), out_dtype=cabi.F32),
    case("tf32_c32_gn_k64", "tf32", 77, 32, 32, 32, tc(64, 32, 1, 0, 1), taps=5, **GN, **TRAJ, res="id"),
    case("tf32_c32_gn_k32", "tf32", 77, 16, 16, 32, tc(32, 32, 1, 0, 1), taps=5, **GN),
    case("tf32_c32_shortcut_k64", "tf32", 40, 32, 64, 32, tc(64, 32, 1, 1, 1), taps=5, res="conv", **GN, **TRAJ),
    case("tf32_c32_shortcut_k32", "tf32", 40, 8, 16, 32, tc(32, 32, 1, 1, 1), taps=5, res="conv", **GN),
    case("tf32_c64_k64_3tiles", "tf32", R3 * 128 // 32 + 5, 32, 32, 64, tc(64, 64, 1, 0, 1), taps=5, **GN, **TRAJ,
         res="id"),
    case("tf32_c64_res_k64", "tf32", 99, 16, 64, 64, tc(64, 64, 1, 1, 1), taps=5, res="conv", **GN, strided=True),
    case("tf32_c64_k32", "tf32", 99, 8, 48, 64, tc(32, 64, 1, 0, 1), taps=3, **GN, film="shift"),
    case("tf32_c64_res_k32", "tf32", 99, 4, 16, 64, tc(32, 64, 1, 1, 1), taps=3, res="conv", **GN),
    case("tf32_c128_k64", "tf32", 45, 8, 64, 128, tc(64, 64, 2, 0, 1), taps=5, **GN, **TRAJ, res="id"),
    case("tf32_c128_res_k64", "tf32", 45, 16, 64, 128, tc(64, 64, 2, 1, 1), taps=5, res="conv", **GN),
    case("tf32_c128_k32", "tf32", 45, 2, 16, 128, tc(32, 64, 2, 0, 1), taps=3, **GN),
    case("tf32_c128_res_k32", "tf32", 45, 4, 48, 128, tc(32, 64, 2, 1, 1), taps=3, res="conv", **GN),
    case("tf32_c256_k64", "tf32", 45, 8, 128, 256, tc(64, 128, 2, 0, 1), taps=5, **GN, **TRAJ, res="id"),
    case("tf32_c256_res_k64", "tf32", 45, 8, 128, 256, tc(64, 128, 2, 1, 1), taps=5, res="conv", **GN),
    case("tf32_c256_k32", "tf32", 45, 1, 16, 256, tc(32, 128, 2, 0, 1), taps=1, **GN),
    case("tf32_c256_res_k32", "tf32", 45, 2, 48, 256, tc(32, 128, 2, 1, 1), taps=3, res="conv", **GN),
    case("tf32_c512_gn", "tf32", 45, 4, 256, 512, tc(64, 256, 2, 0, 1), taps=5, **GN, **TRAJ, res="id"),
    case("tf32_c512_gn_res", "tf32", 45, 4, 256, 512, tc(64, 128, 4, 1, 1), taps=5, res="conv", **GN, **TRAJ),
    case("tf32_c1024_gn", "tf32", 30, 2, 512, 1024, tc(64, 256, 4, 0, 1), taps=5, **GN, **TRAJ, res="id"),
    case("tf32_c1024_gn_res", "tf32", 30, 2, 512, 1024, tc(64, 128, 8, 1, 1), taps=3, res="conv", **GN),
    case("tf32_convT_c32", "tf32", 37, 8, 32, 32, tc(64, 64, 1, 0, 1), taps=3, phases=2, act=M),
    case("tf32_convT_c64", "tf32", 37, 4, 64, 64, tc(64, 128, 1, 0, 1), taps=3, phases=2, strided=True),
    case("tf32_convT_c128", "tf32", 37, 16, 16, 128, tc(32, 256, 1, 0, 1), taps=3, phases=2, film="shift"),
    case("tf32_stride2_c64", "tf32", 37, 8, 32, 64, tc(64, 64, 1, 0, 1), taps=3, stride=2, **GN),
    case("tf32_lin320", "tf32", 3700, 1, 128, 320, tc(64, 160, 1, 0, 1), srd=100, act=cabi.ACT_GELU_TANH, bias="both"),
    case("tf32_lin384", "tf32", 640, 1, 32, 384, tc(64, 192, 1, 0, 1), act=cabi.ACT_SILU),
    case("tf32_lin384_k32", "tf32", 640, 1, 48, 384, tc(32, 128, 1, 0, 1), act=cabi.ACT_GELU_ERF),
    case("tf32_lin384_res_k32", "tf32", 640, 1, 48, 384, tc(32, 128, 1, 1, 1), res="conv"),
    case("tf32_lin896_res_k64", "tf32", 300, 1, 32, 896, tc(64, 128, 1, 1, 1), res="conv"),
    case("tf32_lin960", "tf32", 3700, 1, 320, 960, tc(64, 192, 1, 0, 1), srd=100, act=cabi.ACT_MISH_SILU, film="traj"),
    case("tf32_lin960_k32", "tf32", 700, 1, 16, 960, tc(32, 64, 1, 0, 1), act=cabi.ACT_LEAKY_RELU),
    case("tf32_lin1280", "tf32", 3700, 1, 320, 1280, tc(64, 256, 1, 0, 1), srd=100, film="gate", res="id",
         out_dtype=cabi.F32),
    case("tf32_lin1280_k32", "tf32", 700, 1, 16, 1280, tc(32, 256, 1, 0, 1), srd=50, bias="sample", out_dtype=cabi.BF16),
    case("tf32_lin640", "tf32", 500, 1, 32, 640, tc(64, 160, 1, 0, 1)),
    # operands that are NOT TF32-representable: wgmma .tf32 truncates them (include/cds.h), as the reference assumes
    case("tf32_unrounded_inputs", "tf32", 45, 8, 64, 128, tc(64, 64, 2, 0, 1), taps=5, **GN, in_dtype=cabi.F32),
    # GroupNorm over a common offset of 32 sigma: the tensor-core kernels compute var = E[x^2] - mean^2 in fp32
    case("tf32_gn_offset32", "tf32", 45, 8, 64, 64, tc(64, 64, 1, 0, 1), taps=3, **GN, offset=32.0),
    case("bf16_gn_offset32", "bf16", 45, 8, 64, 128, tc(64, 64, 2, 0, 0), taps=3, **GN, offset=32.0, out_dtype=cabi.F32),
    # CFG branches: in_batch_mod (x_t shared), res_batch_mod
    case("bf16_in_mod", "bf16", 96, 4, 64, 64, tc(64, 32, 2, 0, 0), taps=5, **GN, in_mod=32, res="id", res_mod=32),
    case("tf32_in_mod_shortcut", "tf32", 256, 8, 32, 32, tc(64, 32, 1, 1, 1), taps=5, **GN, in_mod=128, res="conv",
         res_mod=64),
    # ---- conv_ps (L = 4, GroupNorm + Mish, C_out 128 / 256) ---------------------------------------------------------
    case("ps_bf16_c128_k3", "bf16", 300, 4, 128, 128, ps(32, 0, 0), taps=3, **GN, film="shift", res="id"),
    case("ps_bf16_c128_k5_shortcut", "bf16", 300, 4, 256, 128, ps(32, 1, 0), taps=5, **GN, res="conv", res_C=64),
    case("ps_bf16_c256_k1", "bf16", 300, 4, 64, 256, ps(64, 0, 0), taps=1, **GN, res="id", strided=True),
    case("ps_bf16_c256_mods", "bf16", 512, 4, 256, 256, ps(64, 0, 0), taps=5, **GN, film="shift", in_mod=256, res="id",
         res_mod=128),
    case("ps_tf32_c128_k5", "tf32", 300, 4, 128, 128, ps(32, 0, 1), taps=5, **GN, res="id"),
    case("ps_tf32_c128_shortcut_mods", "tf32", 512, 4, 64, 128, ps(32, 1, 1), taps=3, **GN, film="shift", res="conv",
         in_mod=256, res_mod=256),
    case("ps_tf32_c256_k3", "tf32", 300, 4, 256, 256, ps(64, 0, 1), taps=3, **GN, res="id", strided=True),
    # (conv_ps is not persistent: one CTA per (128-trajectory tile, column quarter); this is a large grid, 1636 CTAs)
    case("ps_tf32_c256_large_grid", "tf32", 3 * 132 * 128 // 4 + 50, 4, 64, 256, ps(64, 0, 1), taps=1, **GN),
    # ---- conv_simt (CDS_MATH_FP32) ------------------------------------------------------------------------------------
    case("simt_bn32", "fp32", 41, 16, 14, 32, simt(32), taps=5, **GN, **TRAJ),
    case("simt_bn64_cpg8", "fp32", 41, 8, 32, 64, simt(64), taps=5, **GN, res="conv", res_C=14),
    case("simt_bn128_gn1", "fp32", 300, 32, 64, 128, simt(128), taps=3, groups=1, act=M, res="id", strided=True),
    case("simt_bn64_cpg32_4col", "fp32", 41, 16, 64, 256, simt(64), taps=3, **GN, bias="both"),
    case("simt_convT", "fp32", 41, 8, 64, 64, simt(128), taps=3, phases=2, act=M),
    case("simt_head", "fp32", 41, 32, 32, 14, simt(32), taps=5, act=cabi.ACT_GELU_ERF, in_dtype=cabi.BF16),
    case("simt_wide_nogn", "fp32", 82, 4, 64, 320, simt(128), act=cabi.ACT_SILU, film="traj", in_mod=41),
    # conv_simt storing TF32 / bf16: on tensor-core programs a Linear over the raw x_t (3..9 fp32 channels) is not
    # tensor-core material, runs here, and stores the program's activation type (SfBCUNet's first block, PearceMlp's act_emb)
    case("simt_c6_c512_tf32out", "fp32", 300, 1, 6, 512, simt(128), act=cabi.ACT_SILU, film="shift", out_dtype=cabi.TF32),
    case("simt_c6_c512_bf16out", "fp32", 300, 1, 6, 512, simt(128), act=cabi.ACT_SILU, film="shift", out_dtype=cabi.BF16),
    case("simt_c9_c128_bf16out", "fp32", 1000, 1, 9, 128, simt(128), act=cabi.ACT_LEAKY_RELU, out_dtype=cabi.BF16),
    case("simt_c9_c256_tf32out", "fp32", 1000, 1, 9, 256, simt(128), bias="both", out_dtype=cabi.TF32),
    case("simt_c6_c128_shortcut_tf32out", "fp32", 300, 1, 6, 128, simt(128), act=cabi.ACT_SILU, res="conv",
         out_dtype=cabi.TF32),
    # SfBCUNet's first block, second operator: h (the program's activation type) -> C_out, plus the 1x1 shortcut of x_t
    case("simt_c512_shortcut_c6_bf16", "fp32", 300, 1, 512, 512, simt(128), act=cabi.ACT_SILU, res="conv", res_C=6,
         in_dtype=cabi.BF16, out_dtype=cabi.BF16),
    case("simt_c512_shortcut_c6_tf32", "fp32", 300, 1, 512, 256, simt(128), act=cabi.ACT_SILU, res="conv", res_C=6,
         in_dtype=cabi.TF32, out_dtype=cabi.TF32),
    # the CFG form: both halves share x_t (in_batch_mod) and the shortcut's input (res_batch_mod)
    case("simt_cfg_c6_c256_bf16", "fp32", 600, 1, 6, 256, simt(128), act=cabi.ACT_SILU, film="shift", in_mod=300,
         res="conv", res_mod=300, out_dtype=cabi.BF16),
    case("simt_cfg_c6_c256_tf32", "fp32", 600, 1, 6, 256, simt(128), act=cabi.ACT_SILU, film="shift", in_mod=300,
         res="conv", res_mod=300, out_dtype=cabi.TF32),
    # PearceMlp's FCBlock on fp32 programs: Linear + GroupNorm(8) + exact GELU, a constant scale, an identity residual
    case("simt_gn_gelu_c512", "fp32", 300, 1, 512, 512, simt(64), groups=8, act=cabi.ACT_GELU_ERF, bias="both",
         film="const_scale", res="id"),
]

# ---- the persistent tile loop: a large-batch twin of one case per conv_tc instantiation, so that every CTA of the launch runs
# three or more tiles -- the producer running ahead into the next tile, the ring's phase wrap, the reuse of the accumulator
# tile and the residual prefetch of the next tile all happen.  A launch has at most 2 CTAs per SM resident
# (ConvTcCfg::kMinBlocks <= 2), so num_tiles >= 3 x 2 x 132 suffices on an H100.  The bf16 64-column layers split into two
# 32-column CTAs only while there are fewer than 264 row tiles (conv_tc_pick_split), i.e. fewer than 528 tiles: their twins
# run inside a plan with a second (trivial) branch, where every conv_tc launch is capped at one CTA per SM (cds_plan_finalize),
# so 396 tiles are three per CTA.
SMS = 132


def resident_ctas(c):
    return SMS * (1 if c.get("one_cta") else 2)


def tiles_per_row_tile(c):
    """column tiles of one 128-row tile for the tc variant c["want"]: SPLIT, or the runtime column tiles"""
    _, kc, n, split, _, _ = c["want"]
    return split if split > 1 else max(1, c["C_out"] * c["phases"] // n)


def num_tiles(c):
    return -(-c["B"] * c["L"] // 128) * tiles_per_row_tile(c)


def _twin(c):
    one_cta = c["math"] == "bf16" and c["want"][2] == 32 and c["want"][3] == 2
    t = dict(c, name=c["name"] + "_3tiles", one_cta=one_cta)
    m_tiles = -(-3 * resident_ctas(t) // tiles_per_row_tile(t))
    t["B"] = m_tiles * 128 // c["L"] + 1                      # + 1: a ragged last row tile
    return t


def _add_twins(cases):
    by_want = {}
    for c in cases:
        if c["want"][0] == "tc" and not (c["in_mod"] or c["res_mod"]):
            # prefer the two-phase transposed convs (their TMA store covers one phase of a tile: out_tma = 2)
            if c["want"] not in by_want or (c["phases"] == 2 and by_want[c["want"]]["phases"] == 1):
                by_want[c["want"]] = c
    done = {c["want"] for c in cases if c["want"][0] == "tc" and num_tiles(c) >= 3 * resident_ctas(c)}
    return cases + [_twin(c) for w, c in by_want.items() if w not in done]


CASES = {c["name"]: c for c in _add_twins(CASES)}


# ---------------------------------------------------------------------------------------------------- op construction
def _layout(rows, L, C, strided):
    """(buffer shape, channel offset) of a (rows, L, C) view with a NaN gap of one trajectory after it"""
    if strided:
        return (rows + 1, L + 1, C + 2 * MARGIN), MARGIN
    return (rows + 1, L, C), 0


def geometry(c):
    """dict of the views the op reads and writes: name -> (rows, L, C, dtype)"""
    B, L = c["B"], c["L"]
    g = {"in": (c["in_mod"] or B, L * c["stride"], c["C_in"], c["in_dtype"]),
         "out": (B, L * c["phases"], c["C_out"], c["out_dtype"])}
    res_dt = c["in_dtype"] if c["math"] != "fp32" else cabi.F32
    if c["res"] == "id":
        g["res"] = (c["res_mod"] or B, L, c["C_out"], cabi.F32 if c["math"] == "tf32" else res_dt)
    if c["res"] == "conv":
        g["res_in"] = (c["res_mod"] or B, L, c["res_C"], res_dt)
    return g


def _rnd(x, math):
    """data that the kernel family reads exactly: bf16 / TF32-representable values"""
    if math == "bf16":
        return x.to(torch.bfloat16).to(torch.float32)
    if math == "tf32":
        import opref
        return opref.tf32_round(x)
    return x


def make(c, device, it=1):
    """Allocate and fill every buffer of case ``c`` on ``device``.  Returns (op, data) where data holds the buffers
    ('buf/<name>', 'view/<name>'), the canonical weights and the resolved vectors that tests/opref.py takes."""
    g = torch.Generator().manual_seed(1000 + c["seed"] + sum(map(ord, c["name"])))
    math = c["math"]
    B, L, C_in, C_out, taps, phases = c["B"], c["L"], c["C_in"], c["C_out"], c["taps"], c["phases"]
    N = C_out * phases
    d = {}
    for name, (rows, Lv, C, dt) in geometry(c).items():
        shape, off = _layout(rows, Lv, C, c["strided"])
        buf = torch.full(shape, float("nan"), dtype=TORCH_DT[dt])
        view = buf[:rows, :Lv, off:off + C]
        if name != "out":
            v = torch.randn(rows, Lv, C, generator=g)
            if not (name == "in" and c["in_dtype"] == cabi.F32 and math == "tf32"):
                v = _rnd(v, math if name in ("in", "res_in") or math == "bf16" else "fp32")
            if dt == cabi.TF32:             # a CDS_TF32 tensor holds TF32 values, whichever kernel family reads it
                v = _rnd(v, "tf32")
            view.copy_(v.to(buf.dtype))
        d["buf/" + name] = buf.to(device)
        d["off/" + name] = off
    for name in list(geometry(c)):
        buf, off = d["buf/" + name], d["off/" + name]
        rows, Lv, C, _ = geometry(c)[name]
        d["view/" + name] = buf[:rows, :Lv, off:off + C]
    K = taps * C_in
    w = _rnd(torch.randn(taps, C_in, N, generator=g) / K ** 0.5, math)
    d["w"] = w.to(device)
    if math == "fp32":
        packed = w.reshape(K, N)
    else:
        packed = w.permute(0, 2, 1).reshape(taps * N, C_in)
    d["w_packed"] = packed.to(torch.bfloat16 if math == "bf16" else torch.float32).contiguous().to(device)
    owners = -(-B // c["srd"]) if c["srd"] > 1 else B

    def vec(step, sample, scale=0.1, center=0.0):
        st = (center + scale * torch.randn(3, C_out + 8, generator=g)) if step else None
        sa = ((0.0 if step else center) + scale * torch.randn(owners, C_out + 4, generator=g)) if sample else None
        resolved = None
        if st is not None:
            resolved = st[it, :C_out]
        if sa is not None:
            resolved = sa[:, :C_out] if resolved is None else sa[:, :C_out] + resolved
        dev = [None if t is None else t.to(device) for t in (st, sa)]
        v = cabi.Vec()
        if dev[0] is not None:
            v.step, v.step_stride = dev[0].data_ptr(), C_out + 8
        if dev[1] is not None:
            v.sample, v.sample_stride = dev[1].data_ptr(), C_out + 4
        d.setdefault("keep", []).extend(t for t in dev if t is not None)
        return v, None if resolved is None else resolved.to(device)

    bias = {None: (False, False), "step": (True, False), "sample": (False, True), "both": (True, True)}[c["bias"]]
    d["bias_vec"], d["bias"] = vec(*bias)
    if c["offset"]:                         # a common offset of the GroupNorm input: the conv output has std ~ 1
        d["keep"][0][it].add_(c["offset"])
        d["bias"] = d["bias"] + c["offset"]
    film = c["film"]
    d["scale_vec"], d["scale"] = vec(False, film in ("traj", "gate"), 0.3, 1.0) if film in ("traj", "gate") else (cabi.Vec(), None)
    if film == "const_scale":               # one (C_out,) vector for every row and iteration (step_stride 0)
        d["scale"] = (1.414 + 0.3 * torch.randn(C_out, generator=g)).to(device)
        d["scale_vec"] = cabi.Vec(d["scale"].data_ptr(), 0, 0, 0)
    d["shift_vec"], d["shift"] = vec(film == "shift", film == "traj") if film in ("shift", "traj") else (cabi.Vec(), None)
    if c["groups"]:
        d["gamma"] = (1 + 0.2 * torch.randn(C_out, generator=g)).to(device)
        d["beta"] = (0.2 * torch.randn(C_out, generator=g)).to(device)
    if c["res"] == "conv":
        rw = _rnd(torch.randn(c["res_C"], C_out, generator=g) / c["res_C"] ** 0.5, math)
        d["res_w"] = rw.to(device)
        d["res_w_packed"] = (rw if math == "fp32" else rw.t()).to(torch.bfloat16 if math == "bf16" else torch.float32).contiguous().to(device)
        d["res_bias"] = (0.1 * torch.randn(C_out, generator=g)).to(device)
    return d


def descriptor(c, d=None, ptr=None):
    """cabi.Op of case ``c`` over the buffers ``d`` (make()), or -- for the CPU dispatch test -- over fake, 16-byte aligned
    addresses (ptr=True): only the geometry, strides, dtypes and alignment matter to cds_conv_choice."""
    geo = geometry(c)
    op = cabi.Op()
    op.kind = cabi.OP_CONV
    o = op.u.conv
    o.batch, o.L_in, o.L_out, o.C_in, o.C_out = c["B"], c["L"] * c["stride"], c["L"], c["C_in"], c["C_out"]
    o.taps, o.stride, o.pad, o.phases = c["taps"], c["stride"], c["taps"] // 2, c["phases"]
    o.in_batch_mod, o.res_batch_mod, o.sample_row_div = c["in_mod"], c["res_mod"], c["srd"]
    o.math = MATH[c["math"]]
    fake = {"in": 1 << 28, "out": 2 << 28, "res": 3 << 28, "res_in": 4 << 28}

    def addr(name):
        rows, Lv, C, dt = geo[name]
        shape, off = _layout(rows, Lv, C, c["strided"])
        es = 2 if dt == cabi.BF16 else 4
        base = d["buf/" + name].data_ptr() if d is not None else fake[name]
        return base + off * es, shape[1] * shape[2], shape[2], dt

    o.in_, o.in_bstride, o.in_lstride, o.in_dtype = addr("in")
    o.out, o.out_bstride, o.out_lstride, o.out_dtype = addr("out")
    if "res" in geo:
        o.res, o.res_bstride, o.res_lstride, o.res_dtype = addr("res")
    if "res_in" in geo:
        o.res_in, o.res_in_bstride, o.res_in_lstride, o.res_in_dtype = addr("res_in")
        o.res_C = c["res_C"]
        o.res_w = d["res_w_packed"].data_ptr() if d is not None else 5 << 28
        o.res_bias = d["res_bias"].data_ptr() if d is not None else 6 << 28
    o.w = d["w_packed"].data_ptr() if d is not None else 7 << 28
    o.act = c["act"]
    if c["groups"]:
        o.groups, o.gn_eps = c["groups"], 1e-5
        o.gn_gamma = d["gamma"].data_ptr() if d is not None else 8 << 28
        o.gn_beta = d["beta"].data_ptr() if d is not None else 9 << 28
    if d is not None:
        o.bias, o.scale, o.shift = d["bias_vec"], d["scale_vec"], d["shift_vec"]
    else:                                   # presence (and shape) of the vectors is all that eligibility looks at
        fake_vec = lambda step, sample: cabi.Vec(10 << 28 if step else 0, 16, 11 << 28 if sample else 0, 16)
        o.bias = fake_vec(c["bias"] in ("step", "both"), c["bias"] in ("sample", "both"))
        o.scale = fake_vec(c["film"] == "const_scale", c["film"] in ("traj", "gate"))
        o.shift = fake_vec(c["film"] == "shift", c["film"] == "traj")
    return op


def reference(c, d):
    """tests/opref.py's fp64 result for case ``c`` over the operands ``d`` (on their device)"""
    import opref
    kw = dict(batch=c["B"], L_out=c["L"], taps=c["taps"], stride=c["stride"], pad=c["taps"] // 2, phases=c["phases"],
              math_mode=MATH[c["math"]], bias=d["bias"], act_kind=c["act"], scale=d["scale"], shift=d["shift"],
              sample_row_div=max(1, c["srd"]))
    if c["groups"]:
        kw.update(groups=c["groups"], gamma=d["gamma"], beta=d["beta"], eps=1e-5)
    if c["res"] == "id":
        kw["res"] = d["view/res"]
    if c["res"] == "conv":
        kw.update(res_in=d["view/res_in"], res_w=d["res_w"], res_bias=d["res_bias"])
    return opref.conv(d["view/in"], d["w"], **kw)


# ---------------------------------------------------------------------------------------------------- the checker
# |y - ref| <= ATOL * s + r * |ref|,  s = max(1, mean |ref|).  The operands are exactly representable in the kernel's
# operand type, so what is left is fp32 accumulation order (K <= 5 x 512 products of ~unit operands: ~1e-6 relative),
# the MUFU approximations of rsqrt / exp / rcp (~2^-22), and the rounding of the stored value: at most half an ulp of the
# output type plus that ulp's worth when the kernel's fp32 value and the exact one straddle a rounding boundary.
ATOL = 1e-4
RTOL = {cabi.F32: 0.0, cabi.TF32: 2.0 ** -10, cabi.BF16: 2.0 ** -8}
U = 2.0 ** -24


def pre_norm(c, d):
    """the fp64 conv + bias of case ``c``: the GroupNorm input"""
    import opref
    return opref.conv(d["view/in"], d["w"], batch=c["B"], L_out=c["L"], taps=c["taps"], stride=c["stride"],
                      pad=c["taps"] // 2, math_mode=MATH[c["math"]], bias=d["bias"])


def gn_offset_atol(pre, groups, gamma):
    """Extra absolute error allowed by the fp32 statistics var = E[x^2] - mean^2 of the tensor-core kernels, per output
    element, for the GroupNorm input ``pre`` (batch, L, C) in fp64: with d = summation depth (a thread's columns of the
    group + the shuffle rounds over L + 4), E[x^2] carries a relative error <= (d + 2) u, i.e. var an absolute one
    <= (d + 2) u (mu^2 + sigma^2): rstd is off by half that over sigma^2, the normalised value z by |z| times it; the mean
    is off by <= d u |mu|, z by d u |mu| / sigma.  gamma and the Mish slope (<= 1.1) scale both."""
    B, L, C = pre.shape
    G = groups
    g = pre.reshape(B, L, G, C // G)
    mu = g.mean(dim=(1, 3), keepdim=True)
    sig = ((g - mu) ** 2).mean(dim=(1, 3), keepdim=True).sqrt()
    z = ((g - mu) / sig).abs()
    depth = C // G + max(1, L).bit_length() + 4
    ratio = mu.abs() / sig
    dz = 0.5 * (depth + 2) * U * (1 + ratio ** 2) * z + depth * U * ratio
    return (1.1 * dz * gamma.abs().to(dz.dtype).reshape(1, 1, G, C // G)).reshape(B, L, C)


def check(c, y, ref, extra_atol=0.0, s=None):
    """(ok, largest error as a fraction of the bound, message) for the stored output ``y`` (fp32, bf16 widened) of case
    ``c`` against the exact result ``ref``; ``s``: max(1, mean |ref|) of the whole output when ``ref`` is a part of it"""
    ref = ref.to(torch.float64)
    yd = y.to(torch.float64)
    if not torch.isfinite(yd).all():
        return False, float("inf"), "non-finite output"
    s = max(1.0, ref.abs().mean().item()) if s is None else s
    bound = ATOL * s + extra_atol + RTOL[c["out_dtype"]] * ref.abs()
    frac = ((yd - ref).abs() / bound).max().item()
    if c["out_dtype"] == cabi.TF32 and int((y.contiguous().view(torch.int32) & 0x1FFF).abs().max()) != 0:
        return False, frac, "a CDS_TF32 output is not TF32-representable"
    return frac <= 1.0, frac, f"max |y - ref| / bound = {frac:.3g}"
