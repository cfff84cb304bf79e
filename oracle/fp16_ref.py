"""Per-layer reference of the 'fp16' mode (SE3TN_PREC_FP16), an additive extension of layer_ref.py: the fp16 storage format,
its encode / decode, the mode's weights and arithmetic, and the gate of every layer.  CPU only.

The mode (include/se3tn.h, DESIGN.md §2):
  * activations and the weights of layers 2-13 are IEEE fp16, 2 bytes per channel, laid out as 'bf16' (64 channels per
    128-byte chunk).  Encoding is cvt.rn.satfinite.f16x2.f32: round to nearest even, |x| > 65504 saturates to +-65504;
  * the stems read the bf16x3 stem input and run the bf16x3 arithmetic (stacked hi / lo weight rows), as in 'bf16', then
    store fp16;
  * every other layer runs wgmma ...k16.f32.f16.f16 on fp16 operands, one k16 MMA per 16 K elements, as 'bf16' does.

The gate (layer_ref.gate, both parts) with:
  * operands: the decoded stored input x^ (exact) and the weights as held, rne16(w) (stems: split2(w)) -- their products are
    exact in fp64;
  * accumulation: layer_ref's model and chain (stems: 'bf16x3'; the rest: 'bf16', whose MMA count per K it shares);
  * output: U_OUT_F16 = 2^-11 relative plus an absolute term of F16_SUB = 2^-25, half the spacing of fp16's subnormals
    (2^-24), which a relative bound cannot cover.  The reference saturates as the format does: where the fp64 output
    exceeds 65504 in magnitude it is +-65504, so a kernel that stores inf there fails.  The network's activations stay far
    below 65504 (DESIGN.md §2 lists the headroom).
"""
import numpy as np
import torch
import torch.nn.functional as F

import layer_ref as R

F16_MAX = 65504.0
U_OUT_F16 = 2.0 ** -11
F16_SUB = 2.0 ** -25
U_OUT = dict(R.U_OUT, fp16=U_OUT_F16)                 # layer_ref's table plus the new format


# ------------------------------------------------------------------------------------------- the format (bit-exact)
def f16_bits(x):
    """cvt.rn.satfinite.f16x2.f32: fp32 -> fp16 bits (uint16), round to nearest even, |x| > 65504 (inf included) saturates
    to +-65504, NaN stays NaN.  numpy's cast rounds the same way (subnormals included) but overflows to inf: clamp first."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    c = np.where(np.isnan(x), x, np.clip(x, -F16_MAX, F16_MAX)).astype(np.float32)
    return c.astype(np.float16).view(np.uint16)


def f16_value(bits):
    """fp16 bits -> float32 (exact)."""
    return np.ascontiguousarray(bits, dtype=np.uint16).view(np.float16).astype(np.float32)


def f16_rne(x):
    return f16_value(f16_bits(x))


# ------------------------------------------------------------------------------------------- buffers in the mode
def buf_format(buf):
    """Storage format of buffer `buf` in the 'fp16' mode: the stem inputs as in 'bf16', every conv output fp16."""
    if buf in ('X0A', 'X0B'):
        return R.stem_format('bf16')
    return 'fp16'


def image_bytes(buf, fmt=None):
    fmt = fmt or buf_format(buf)
    return R.floats_per_image(buf) * 2 if fmt == 'fp16' else R.image_bytes(buf, fmt)


def decode(raw, buf, fmt=None):
    """Raw bytes of ONE image of buffer `buf` -> layer_ref.Decoded, NCHW."""
    fmt = fmt or buf_format(buf)
    if fmt != 'fp16':
        return R.decode(raw, buf, fmt)
    _, H, W, C = R.BUFS[R.BUF_ID[buf]]
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if raw.size != image_bytes(buf, fmt):
        raise ValueError('%s: %d bytes, expected %d' % (buf, raw.size, image_bytes(buf, fmt)))
    return R.Decoded(np.ascontiguousarray(f16_value(raw.view(np.uint16)).reshape(H, W, C).transpose(2, 0, 1)))


def encode(value, buf, fmt=None):
    """NCHW float32 -> the raw bytes of one image, exactly as the device's Storage<SE3TN_PREC_FP16>::encode writes them."""
    fmt = fmt or buf_format(buf)
    if fmt != 'fp16':
        return R.encode(value, buf, fmt)
    _, H, W, C = R.BUFS[R.BUF_ID[buf]]
    x = np.asarray(value, dtype=np.float32).reshape(C, H, W).transpose(1, 2, 0)
    return np.ascontiguousarray(f16_bits(x)).view(np.uint8).reshape(-1)


def storage_addr(fmt, pix, C, c):
    """Storage<PREC>::addr: byte offset of channel c of pixel pix."""
    if fmt == 'fp16':
        return (pix * C + c) * 2
    return R.storage_addr(fmt, pix, C, c)


def trunk_ksplit(n):
    """run_network's split-K choice: 2 bytes per channel, as 'bf16' (convAB1's two 128-byte chunks: ksplit 2)."""
    return R.trunk_ksplit(n, 'bf16')


# ------------------------------------------------------------------------------------------- the arithmetic
def arith(li):
    """The arithmetic layer li runs in the mode: the stems read a bf16x3-format input."""
    return 'bf16x3' if R.LAYERS[li].kind == 'stem' else 'fp16'


def mode_weights(w_rows, li):
    """The weights as the mode holds them, in layer_ref.mode_weights' form [(rows, input part), ...]."""
    if arith(li) == 'bf16x3':
        return R.mode_weights(w_rows, li, 'bf16x3')
    return [(f16_rne(w_rows), 'x')]


def chain_units(li, ksplit=1):
    """c of the gate: the stems as bf16x3 (stacked halves), the rest one k16 MMA per 16 K elements, as 'bf16'."""
    return R.chain_units(li, 'bf16', ksplit)          # layer_ref.arith('bf16') already maps the stems to bf16x3


class Ref16(R.Ref):
    """layer_ref.Ref plus the fp16 output's absolute subnormal term abs_out."""
    def __init__(self, base, abs_out):
        super().__init__(base.y, base.S, base.Q, base.c, base.L, base.u_out, base.eps, base.extra_B, base.extra_Q)
        self.abs_out = abs_out

    def bound(self):
        return super().bound() + self.abs_out

    def scale(self):
        return super().scale() + self.abs_out


def layer_ref(li, x, w_rows, b, res=None, ksplit=1, out_fmt='fp16'):
    """Reference of layer li in the 'fp16' mode from its decoded stored input x and residual res (layer_ref.Decoded).
    out_fmt 'fp32': the last layer's fp32 pooled activation (H3 is never stored)."""
    if arith(li) == 'bf16x3':                         # the stems: exactly the 'bf16' mode's arithmetic and pool
        ref = R.layer_ref(li, 'bf16', x, w_rows, b, res=res, ksplit=ksplit, out_fmt='fp32')
    else:                                             # 'fp32' takes the held weights as given (their products are exact)
        ref = R.layer_ref(li, 'fp32', x, f16_rne(w_rows), b, res=res, out_fmt='fp32')
    ref.c = chain_units(li, ksplit)
    if out_fmt == 'fp32':
        return ref
    ref.u_out = U_OUT_F16
    ref.y = ref.y.clamp(-F16_MAX, F16_MAX)
    return Ref16(ref, torch.full_like(ref.y, F16_SUB))


def chained_ref(li_first, x, w1, b1, w2, b2, res2, ksplit=1):
    """layer_ref.chained_ref in the mode: two layers from the first one's input (convB2.conv1's output T2 is overwritten by
    convB3.conv1).  The first layer's output is rounded to fp16 as the device stores it; its worst-case error E1 (its bound
    plus the reference's own storage rounding) enters the second layer's bound through |w2| (gate 1) and w2^2 (gate 2)."""
    r1 = layer_ref(li_first, x, w1, b1, ksplit=ksplit)
    buf = R.LAYERS[li_first].out
    x2 = decode(encode(r1.y.float().numpy(), buf), buf)
    E1 = r1.bound() + r1.u_out * r1.y.abs() + F16_SUB
    li2 = li_first + 1
    r2 = layer_ref(li2, x2, w2, b2, res=res2, ksplit=ksplit)
    wt = R.oihw(f16_rne(w2), li2).abs()
    G = R.LAYERS[li2].groups
    r2.extra_B = F.conv2d(E1[None], wt, padding=1, groups=G)[0]
    r2.extra_Q = F.conv2d((E1 * E1)[None], wt * wt, padding=1, groups=G)[0].sqrt()
    return r1, r2
