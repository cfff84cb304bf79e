"""Per-layer reference of the 'fp8' mode (SE3TN_PREC_FP8), an additive extension of layer_ref.py: the e4m3 storage format,
its encode / decode, the mode's weights and scales, and the gate of each e4m3-written layer.  CPU only.

The mode (include/se3tn.h, DESIGN.md §3):
  * the stems and 64-channel layers run as in 'bf16' (bf16x3 stems, bf16 64-channel layers; layer_ref's 'bf16' references
    hold for them), except that the two layers that write CAT (convA2.conv2, convB3.conv2) encode it to e4m3 in their
    epilogue;
  * the six trunk layers read e4m3 activations and e4m3 weights: per e4m3 tensor one power-of-two activation scale
    (SCALE_NAMES; H1 and H2 one per head group of 512 channels), per weight row a power-of-two scale
    s_w = 2^ceil(log2(max|w_row| / 448));
  * trunk MMAs are wgmma ...k32.f32.e4m3.e4m3 on the CODES (4 per 128-byte chunk and tap); the epilogue forms
    acc * mul[co] + bias (+ residual code * its scale) with mul[co] = s_in * s_w[co], the activation, then the code
    e4m3(y / s_out) (cvt.rn.satfinite: round to nearest even, |x| > 448 -> 448).  The last layer keeps its fp32 pool.
Every scale is a power of two, so scaling is exact: the only roundings are the e4m3 encodes and the accumulation.

The gate (layer_ref.gate, both parts) with:
  * operands: the decoded stored input x^ = code * s_in (exact), the weights as held, w^ = code * s_w -- their products are
    exact in fp64;
  * accumulation: its own unit.  FP8 wgmma on Hopper is reported to keep fewer bits than fp32 (about 14) while it sums.
    The model: each k32 MMA truncates its sum at U_ACC_FP8 = 2^-13 of the running sum of absolute values (<= S).  So c =
    (K / 32) 2^11 units of 2^-24, + 1 (bias) + 1 (residual).  Not measured: an assumption the gate checks;
  * output: U_OUT_E4M3 = 2^-4 relative (3 mantissa bits, round to nearest) plus an absolute term of 2^-10 s_out (half the
    spacing of e4m3's subnormals, 2^-9 s_out).  Saturated elements (|y| > 448 s_out) fail the gate: the calibration's
    headroom keeps them out.
"""
import math
import numpy as np
import torch

import layer_ref as R

E4M3_MAX = 448.0
U_OUT_E4M3 = 2.0 ** -4
E4M3_SUB = 2.0 ** -10                                # x s_out: the absolute output term
U_ACC_FP8 = 2.0 ** -13                               # the accumulation model's unit per k32 MMA
HEADROOM = 2                                         # SE3TN_FP8_HEADROOM (include/se3tn.h)
U_OUT = dict(R.U_OUT, e4m3=U_OUT_E4M3)               # layer_ref's table plus the new format

SCALE_NAMES = ['CAT', 'F1', 'T4', 'F2', 'H1.trans', 'H1.rot', 'H2.trans', 'H2.rot']
E4M3_BUFS = ('CAT', 'F1', 'T4', 'F2', 'H1', 'H2')
TRUNK_IN = {8: 'CAT', 9: 'F1', 10: 'T4', 11: 'F2', 12: 'H1', 13: 'H2'}


# ------------------------------------------------------------------------------------------- the format (bit-exact)
def e4m3_bits(x):
    """cvt.rn.satfinite.e4m3x2.f32: fp32 -> e4m3 code bytes (uint8), round to nearest even, |x| > 448 (inf included)
    saturates to +-448, NaN -> NaN (0x7F / 0xFF).  torch's cast rounds the same way but does not saturate: clamp first."""
    x = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32))
    c = torch.where(torch.isnan(x), x, x.clamp(-E4M3_MAX, E4M3_MAX))
    return c.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def e4m3_value(bits):
    """e4m3 code bytes -> float32 (exact)."""
    b = torch.as_tensor(np.ascontiguousarray(bits, dtype=np.uint8))
    return b.view(torch.float8_e4m3fn).to(torch.float32).numpy()


def e4m3_rne(x):
    return e4m3_value(e4m3_bits(x))


def pow2_scale(amax):
    """2^ceil(log2(amax / 448)), 1 for amax == 0 -- exactly as the library forms it (frexp, no logarithm)."""
    amax = float(amax)
    if not amax > 0.0:
        return 1.0
    m, ex = math.frexp(amax)                          # amax = m 2^ex, m in [0.5, 1); 448 = 0.875 2^9
    return math.ldexp(1.0, ex - 9 + (1 if m > 0.875 else 0))


def calibrate(amax):
    """The scales se3tn_calibrate_fp8 sets from the 8 tensors' max|x|."""
    return np.array([pow2_scale(float(a) * HEADROOM) for a in amax], dtype=np.float32)


# ------------------------------------------------------------------------------------------- buffers in the mode
def buf_format(buf):
    """Storage format of buffer `buf` in the 'fp8' mode."""
    if buf in E4M3_BUFS:
        return 'e4m3'
    return R.buf_format(buf, 'bf16')


def image_bytes(buf, fmt=None):
    fmt = fmt or buf_format(buf)
    return R.floats_per_image(buf) if fmt == 'e4m3' else R.image_bytes(buf, fmt)


def channel_scales(buf, scales):
    """(C,) float64: the scale of each channel of e4m3 buffer `buf`."""
    s = np.asarray(scales, dtype=np.float64)
    _, _, _, C = R.BUFS[R.BUF_ID[buf]]
    if buf in ('H1', 'H2'):
        k = 4 if buf == 'H1' else 6
        return np.concatenate([np.full(512, s[k]), np.full(512, s[k + 1])])
    return np.full(C, s[SCALE_NAMES.index(buf)])


def decode(raw, buf, scales=None):
    """Raw bytes of ONE image -> layer_ref.Decoded (NCHW), the e4m3 buffers' values = code * scale."""
    fmt = buf_format(buf)
    if fmt != 'e4m3':
        return R.decode(raw, buf, fmt)
    _, H, W, C = R.BUFS[R.BUF_ID[buf]]
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if raw.size != H * W * C:
        raise ValueError('%s: %d bytes, expected %d' % (buf, raw.size, H * W * C))
    v = e4m3_value(raw).reshape(H, W, C).transpose(2, 0, 1).astype(np.float64)
    v = v * channel_scales(buf, scales)[:, None, None]
    return R.Decoded(np.ascontiguousarray(v.astype(np.float32)))


def encode(value, buf, scales):
    """NCHW float32 -> the e4m3 bytes of one image, as the device's epilogue writes them (codes of value / scale)."""
    _, H, W, C = R.BUFS[R.BUF_ID[buf]]
    x = np.asarray(value, dtype=np.float32).reshape(C, H, W) / channel_scales(buf, scales).astype(np.float32)[:, None, None]
    return np.ascontiguousarray(e4m3_bits(x.astype(np.float32)).transpose(1, 2, 0)).reshape(-1)


def trunk_ksplit(n):
    """run_network's split-K choice in this mode: convAB1's input CAT is one 128-byte chunk per pixel in e4m3, so the
    halving of layer_ref.trunk_ksplit ends at 1: no latency mode."""
    if n > 4:
        return 1
    ks = 4
    for L in R.LAYERS[R.FIRST_TRUNK:]:
        while (L.cin // 128) % ks:
            ks //= 2
    return ks


# ------------------------------------------------------------------------------------------- weights, references
def weight_codes(w_rows):
    """The trunk weights as the mode holds them: (codes float32 (rows, ktot) as values, s_w float64 (rows,))."""
    w = np.asarray(w_rows, dtype=np.float32)
    sw = np.array([pow2_scale(a) for a in np.abs(w).max(1)], dtype=np.float64)
    return e4m3_rne(w / sw.astype(np.float32)[:, None]), sw


def mode_weights(w_rows):
    """w^ = code * s_w (exact in float32: a power-of-two multiple of an e4m3 value)."""
    codes, sw = weight_codes(w_rows)
    return (codes.astype(np.float64) * sw[:, None]).astype(np.float32)


def out_scales(li, scales):
    """(rows,) float64 scale of layer li's e4m3 output, or None (the last layer pools in fp32)."""
    L = R.LAYERS[li]
    if li == 13:
        return None
    if L.out == 'CAT':
        return np.full(L.rows, float(scales[0]))
    return channel_scales(L.out, scales)


def chain_units(li):
    """c of the gate for trunk layer li: (K / 32) k32 MMAs at U_ACC_FP8 each, then + bias, + residual."""
    L = R.LAYERS[li]
    return (L.ktot // 32) * (U_ACC_FP8 / R.U24) + 1 + (1 if L.res else 0)


class Ref8(R.Ref):
    """layer_ref.Ref plus the e4m3 output's absolute subnormal term abs_out (per channel, 2^-10 s_out)."""
    def __init__(self, base, abs_out):
        super().__init__(base.y, base.S, base.Q, base.c, base.L, base.u_out, base.eps, base.extra_B, base.extra_Q)
        self.abs_out = abs_out

    def bound(self):
        return super().bound() + self.abs_out

    def scale(self):
        return super().scale() + self.abs_out


def _with_e4m3_out(ref, s_out):
    ref.u_out = U_OUT_E4M3
    return Ref8(ref, torch.from_numpy(E4M3_SUB * np.asarray(s_out, dtype=np.float64))[:, None, None].expand_as(ref.y).clone())


def layer_ref(li, x, w_rows, b, scales, res=None):
    """Reference of e4m3-written layer li (3, 7: the CAT writers; 8-13: the trunk) from its decoded stored input x and
    residual res (layer_ref.Decoded, values already scaled).  The last layer's output is its fp32 pooled activation."""
    L = R.LAYERS[li]
    if not L.trunk:                                   # bf16 arithmetic, e4m3 output
        ref = R.layer_ref(li, 'bf16', x, w_rows, b, res=res)
        return _with_e4m3_out(ref, out_scales(li, scales))
    ref = R.layer_ref(li, 'fp32', x, mode_weights(w_rows), b, res=res, out_fmt='fp32')   # fp32: w taken as given (exact)
    ref.c = chain_units(li)
    so = out_scales(li, scales)
    if so is None:
        return ref
    return _with_e4m3_out(ref, so)


# ------------------------------------------------------------------------------------------- a CPU stand-in of the device
def standin(li, x, w_rows, b, scales, res=None, mutate=None):
    """The mode's arithmetic of trunk layer li on the CPU: float32 conv of the CODES, then the epilogue -> the layer's output
    as the device would store and the harness decode it (NCHW float32; the last layer: its fp32 activation).  mutate injects
    one of the bugs the gate must catch: 'row_scale' (one scale for every weight row), 'other_group' (each head group's
    mul with the other group's input scale), 'drop_chunk' (the last 128-channel K chunk lost), 'no_residual',
    'unscaled_out' (codes of y, not y / s_out), 'other_res_group' (the residual's codes decoded with the other head group's
    scale)."""
    import torch.nn.functional as F
    L = R.LAYERS[li]
    codes, sw = weight_codes(w_rows)
    s_in = channel_scales(TRUNK_IN[li], scales)
    xc = np.asarray(x.value, dtype=np.float64) / s_in[:, None, None]          # the stored codes (exact)
    if mutate == 'drop_chunk':
        xc = xc.copy()
        per = L.cin
        for g in range(L.groups):
            xc[g * per + per - 128:(g + 1) * per] = 0.0
    xt = torch.from_numpy(xc.astype(np.float32))[None]
    wt = torch.from_numpy(codes.reshape(L.rows, 3, 3, L.cin).transpose(0, 3, 1, 2).copy())
    acc = F.conv2d(xt, wt, stride=L.stride, padding=1, groups=L.groups)[0].numpy()
    if mutate == 'row_scale':
        sw = np.full_like(sw, sw.max())
    grp_in = np.repeat(s_in[::L.cin][:L.groups], L.cout)                     # the input scale of each row's group
    if mutate == 'other_group' and L.groups > 1:
        grp_in = grp_in.reshape(2, -1)[::-1].reshape(-1)
    mul = (grp_in * sw).astype(np.float32)
    y = acc * mul[:, None, None] + np.asarray(b, np.float32)[:, None, None]
    if res is not None and mutate != 'no_residual':
        rv = np.asarray(res.value, np.float64)
        if mutate == 'other_res_group':
            cs = channel_scales(L.res, scales)
            rv = rv * (cs.reshape(2, -1)[::-1].reshape(-1) / cs)[:, None, None]
        y = y + rv.astype(np.float32)
    y = R.act_fp64(torch.from_numpy(y.astype(np.float64)), L.act).numpy().astype(np.float32)
    so = out_scales(li, scales)
    if so is None:
        return y
    if mutate == 'unscaled_out':
        return (e4m3_rne(y).astype(np.float64) * so[:, None, None]).astype(np.float32)
    return (e4m3_rne(y / so.astype(np.float32)[:, None, None]).astype(np.float64) * so[:, None, None]).astype(np.float32)
