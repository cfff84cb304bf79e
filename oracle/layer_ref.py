"""Per-layer reference of the conv stack: each of the 14 conv layers checked ALONE against an fp64 conv of its own stored
input, in the storage formats of csrc/storage.cuh and the arithmetic each precision mode runs.

CPU only (numpy + torch CPU functional ops); nothing here touches the package's kernels.  Used by tests/test_gpu_layers.py
(device buffers read through Engine.debug_buffer) and tests/test_layer_ref_cpu.py (the gate against a CPU stand-in of the
device arithmetic and against deliberately broken versions of it).

Storage formats (storage.cuh), per image, NHWC:
  tf32    4 bytes per channel, fp32 words rounded to tf32 (cvt.rna: ties away from zero)
  bf16x3  4 bytes per channel, per 32-channel (128-byte) chunk [32 x bf16 hi | 32 x bf16 lo], value hi + lo
  bf16    2 bytes per channel; the image stride is half the buffer's floats_per_image (run_network's out_feature offset)
  fp32    plain fp32 words (the FFMA mode)
  stem input X0A / X0B (182 x 184 x 4, 3-pixel zero halo, 16 bytes per pixel in every mode): tf32 words in tf32,
          [2 words hi | 2 words lo] (4 bf16 hi, then 4 bf16 lo) in BOTH bf16 modes, raw fp32 in fp32.

What the reference of one layer is.  The device's operands are the decoded stored input x^ (and residual r^) and the
weights as the mode holds them:
  tf32    rna(w);  x^ tf32                                     -> conv(w^, x^)
  bf16    rne(w);  x^ bf16                                     -> conv(w^, x^)
  bf16x3  (w_hi, w_lo) = split2(w); x^ = hi + lo             -> conv(w_hi, hi) + conv(w_hi, lo) + conv(w_lo, hi)
          conv_trunk_kernel forms exactly these three products (6 MMAs per 32-channel chunk and tap: AO/BO = hi.w_hi x2,
          lo.w_hi x2, hi.w_lo x2); conv_resident_kernel stacks [w_hi ; w_lo] along N, so one N = 128 MMA gives hi.w_hi and
          hi.w_lo and an N = 64 MMA adds lo.w_hi into the first half (the stems: [hi4|lo4] pixels against
          [w_hi|w_hi ; w_lo|0] rows -- the same three products).  lo.w_lo is never formed.  The bf16 mode's stems read a
          bf16x3-format input and run this arithmetic too (storage.cuh stem_input_prec).
  fp32    w exact; x^ fp32
Every product of these operands is exact in fp64, so z = conv + b + r^ is computed in float64, then the activation (SELU
or ReLU); the stems take max_pool2d(3, 2, 1) of the conv before the bias (the kernel pools, then adds the bias and applies
SELU, which commute with the max).  What remains between device and reference is fp32 accumulation, the activation's
expf and the rounding into the output's storage format.

The gate, per (layer, mode, case):
  1. elementwise, worst case:  |y_dev - y| <= L (c 2^-24 S + eps_act) + u_out (|y| + L (...)) + tiny
       S = conv(|w^|, |x^|) + |b| + |r^| in fp64 (for bf16x3 the absolute values of all three products);
       L = 1 for ReLU and max-pool, lambda*alpha = 1.7581 for SELU (the largest slope of SELU);
       u_out = output format's unit roundoff: 2^-11 tf32, 2^-8 bf16, 2^-16 bf16x3 (hi + lo holds 16 bits), 0 fp32;
       c = chain_units(): fp32 roundings along the longest accumulation chain of that kernel for that layer, counted
       from the code, in units of 2^-24 (round to nearest).
     Tensor cores do not sum a k-group with IEEE round to nearest.  The model used here: each MMA instruction adds its
     k-group of products into the accumulator exactly and then truncates the sum at 2^-23 of the group's largest term
     (accumulator included), i.e. at most 2 units of 2^-24 times the running sum of absolute values, which is <= S.
     Nobody has measured that model on this hardware: it is an assumption this gate checks.
  2. statistical: RMS over the layer's elements of (y_dev - y) / (L (c 2^-24 Q + eps_act) + u_out |y| + tiny) <= 1, with
     Q = sqrt(conv(w^2, x^2)) the root-sum-square scale of the products.  The worst-case S term is loose by ~sqrt(K) and
     alone cannot see e.g. one 32-channel chunk that lost its lo half; a partial sum of K products is of order Q, so the
     accumulation error of a correct kernel is at most c 2^-24 Q per element (less for unbiased rounding), and the output
     rounding at most u_out |y|: each part contributes at most 1 to every element's ratio, and their RMS stays below 1.
  NaN or Inf in a checked region fails both.
"""
import math
import numpy as np
import torch
import torch.nn.functional as F

U24 = 2.0 ** -24
SELU_ALPHA, SELU_SCALE = 1.6732632423543772, 1.0507009873554805
SELU_L = SELU_ALPHA * SELU_SCALE                     # 1.7581: SELU's largest slope (z -> -0)
TINY = 2.0 ** -120                                   # below every activation the net produces; absorbs subnormal flushing
U_OUT = {'tf32': 2.0 ** -11, 'bf16': 2.0 ** -8, 'bf16x3': 2.0 ** -16, 'fp32': 0.0}
RELU, SELU = 'relu', 'selu'

# Activation buffers behind Engine.debug_buffer(id, n): id -> (name, H, W, C); floats_per_image = H * W * C
BUFS = [('X0A', 182, 184, 4), ('X0B', 182, 184, 4), ('Y1A', 88, 88, 64), ('Y1B', 88, 88, 64), ('P1A', 44, 44, 64),
        ('P1B', 44, 44, 64), ('T1', 44, 44, 64), ('T2', 44, 44, 64), ('U', 44, 44, 64), ('CAT', 44, 44, 128),
        ('F1', 22, 22, 256), ('T4', 22, 22, 256), ('F2', 22, 22, 256), ('H1', 11, 11, 1024), ('H2', 11, 11, 1024),
        ('H3', 11, 11, 1024)]
BUF_ID = {b[0]: i for i, b in enumerate(BUFS)}


def floats_per_image(buf):
    _, H, W, C = BUFS[BUF_ID[buf]]
    return H * W * C


class Layer:
    def __init__(self, name, kind, inp, out, res, cin, cout, groups, coff, act, block_n):
        self.name, self.kind, self.inp, self.out, self.res = name, kind, inp, out, res
        self.cin, self.cout, self.groups, self.coff, self.act, self.block_n = cin, cout, groups, coff, act, block_n
        self.taps = 7 if kind == 'stem' else 9
        self.ktot = self.taps * cin                    # K per group (the stem: 7 filter rows x 8 pixels x 4 channels)
        self.rows = cout * groups
        self.stride = 1 if kind == 's1' else 2
        self.trunk = False
        self.L = SELU_L if act == SELU else 1.0


# The 14 layers of kLayers (se3tn.cu): kind, input, output (the stems' pooled output in the tensor-core modes), residual,
# cin / cout per group, groups, output channel offset, activation, output channels per work unit
LAYERS = [
    Layer('convA1', 'stem', 'X0A', 'P1A', None, 32, 64, 1, 0, SELU, 64),
    Layer('convB1', 'stem', 'X0B', 'P1B', None, 32, 64, 1, 0, SELU, 64),
    Layer('convA2.conv1', 's1', 'P1A', 'T1', None, 64, 64, 1, 0, RELU, 64),
    Layer('convA2.conv2', 's1', 'T1', 'CAT', 'P1A', 64, 64, 1, 0, RELU, 64),
    Layer('convB2.conv1', 's1', 'P1B', 'T2', None, 64, 64, 1, 0, RELU, 64),      # T2 is overwritten by convB3.conv1
    Layer('convB2.conv2', 's1', 'T2', 'U', 'P1B', 64, 64, 1, 0, RELU, 64),
    Layer('convB3.conv1', 's1', 'U', 'T2', None, 64, 64, 1, 0, RELU, 64),
    Layer('convB3.conv2', 's1', 'T2', 'CAT', 'U', 64, 64, 1, 64, RELU, 64),
    Layer('convAB1', 's2', 'CAT', 'F1', None, 128, 256, 1, 0, SELU, 128),
    Layer('convAB2.conv1', 's1', 'F1', 'T4', None, 256, 256, 1, 0, RELU, 128),
    Layer('convAB2.conv2', 's1', 'T4', 'F2', 'F1', 256, 256, 1, 0, RELU, 128),
    Layer('{trans,rot}_conv1', 's2', 'F2', 'H1', None, 256, 1024, 1, 0, SELU, 128),           # both heads' rows, one input
    Layer('{trans,rot}_conv2.conv1', 's1', 'H1', 'H2', None, 512, 512, 2, 0, RELU, 128),
    Layer('{trans,rot}_conv2.conv2', 's1', 'H2', 'H3', 'H1', 512, 512, 2, 0, RELU, 128),
]
FIRST_TRUNK = 8
for _li, _l in enumerate(LAYERS):
    _l.trunk = _li >= FIRST_TRUNK
FC_FLOATS = 6 * 512 + 6


def blob_offsets():
    """(w_off, b_off) per layer and fc_off in the fp32 blob, in the order prepare_weights walks it."""
    off, w_off, b_off = 0, [], []
    for L in LAYERS:
        w_off.append(off); off += L.rows * L.ktot
        b_off.append(off); off += L.rows
    return w_off, b_off, off


def layer_weights(blob, li):
    """-> (K-major rows float32 (rows, ktot), bias float32 (rows,)) of layer li, sliced from pack_state_dict's blob."""
    w_off, b_off, _ = blob_offsets()
    L = LAYERS[li]
    w = np.asarray(blob[w_off[li]:w_off[li] + L.rows * L.ktot], dtype=np.float32).reshape(L.rows, L.ktot)
    return w, np.asarray(blob[b_off[li]:b_off[li] + L.rows], dtype=np.float32)


def fc_weights(blob):
    _, _, fc = blob_offsets()
    return (np.asarray(blob[fc:fc + 6 * 512], dtype=np.float32).reshape(6, 512),
            np.asarray(blob[fc + 6 * 512:fc + FC_FLOATS], dtype=np.float32))


# ------------------------------------------------------------------------------------------- encoders (bit-exact)
def _f32(x):
    return np.ascontiguousarray(x, dtype=np.float32)


def tf32_rna(x):
    """cvt.rna.tf32.f32: keep 10 mantissa bits, round to nearest with ties away from zero (adding half an ulp to the
    magnitude bits carries into the exponent exactly like the hardware).  Non-finite values pass through."""
    x = _f32(x)
    u = x.view(np.uint32)
    r = ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    return np.where(np.isfinite(x), r, x).astype(np.float32)


def tf32_trunc(x):
    """tf32 by truncation (NOT what the device does: the CPU tests' mutation)."""
    return (_f32(x).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def bf16_bits(x):
    """__float2bfloat16_rn: fp32 -> bf16 bits, round to nearest even (NaN -> a quiet NaN)."""
    x = _f32(x)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), ((u >> 16) | 0x40).astype(np.uint16), r)


def bf16_value(bits):
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def bf16_rne(x):
    return bf16_value(bf16_bits(x))


def split2(x):
    """storage.cuh split2: hi = rne(x), lo = rne(x - hi) (x - hi is exact in fp32) -> (hi, lo) as float32 values."""
    x = _f32(x)
    hi = bf16_rne(x)
    return hi, bf16_rne(x - hi)


# ------------------------------------------------------------------------------------------- formats and decoders
def stem_format(prec):
    """Format of the stem input X0A / X0B in mode prec."""
    return {'tf32': 'tf32', 'fp32': 'fp32', 'bf16x3': 'stem_hilo', 'bf16': 'stem_hilo'}[prec]


def buf_format(buf, prec):
    if buf in ('X0A', 'X0B'):
        return stem_format(prec)
    return prec


def image_bytes(buf, fmt):
    """Bytes one image of buffer `buf` occupies in format fmt (the image stride of the buffer)."""
    return floats_per_image(buf) * (2 if fmt == 'bf16' else 4)


class Decoded:
    """A decoded activation: value (C, H, W) float32 as the device reads it; hi / lo (bf16x3-type formats) or None."""
    def __init__(self, value, hi=None, lo=None):
        self.value, self.hi, self.lo = value, hi, lo


def decode(raw, buf, fmt):
    """Raw bytes of ONE image of buffer `buf` (uint8, image_bytes long) -> Decoded, NCHW."""
    _, H, W, C = BUFS[BUF_ID[buf]]
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    if raw.size != image_bytes(buf, fmt):
        raise ValueError('%s: %d bytes, expected %d' % (buf, raw.size, image_bytes(buf, fmt)))
    t = lambda a: np.ascontiguousarray(a.reshape(H, W, C).transpose(2, 0, 1))
    if fmt in ('tf32', 'fp32'):
        return Decoded(t(raw.view(np.float32)))
    if fmt == 'bf16':
        return Decoded(t(bf16_value(raw.view(np.uint16))))
    if fmt == 'bf16x3':
        h = raw.view(np.uint16).reshape(H, W, C // 32, 2, 32)
        hi, lo = bf16_value(h[:, :, :, 0, :]), bf16_value(h[:, :, :, 1, :])
    elif fmt == 'stem_hilo':
        h = raw.view(np.uint16).reshape(H, W, 2, 4)
        hi, lo = bf16_value(h[:, :, 0, :]), bf16_value(h[:, :, 1, :])
    else:
        raise ValueError(fmt)
    hi, lo = t(hi), t(lo)
    return Decoded((hi + lo).astype(np.float32), hi, lo)       # exact: lo is at most half an ulp of hi


def encode(value, buf, fmt):
    """NCHW float32 -> the raw bytes of one image, exactly as the device's Storage<>::encode writes them."""
    _, H, W, C = BUFS[BUF_ID[buf]]
    x = _f32(value).reshape(C, H, W).transpose(1, 2, 0)
    if fmt == 'fp32':
        return np.ascontiguousarray(x).view(np.uint8).reshape(-1)
    if fmt == 'tf32':
        return np.ascontiguousarray(tf32_rna(x)).view(np.uint8).reshape(-1)
    if fmt == 'bf16':
        return np.ascontiguousarray(bf16_bits(x)).view(np.uint8).reshape(-1)
    hi, lo = split2(x)
    hb, lb = bf16_bits(hi), bf16_bits(lo)
    if fmt == 'bf16x3':
        out = np.stack([hb.reshape(H, W, C // 32, 32), lb.reshape(H, W, C // 32, 32)], axis=3)
    elif fmt == 'stem_hilo':
        out = np.stack([hb, lb], axis=2)
    else:
        raise ValueError(fmt)
    return np.ascontiguousarray(out).view(np.uint8).reshape(-1)


def storage_addr(fmt, pix, C, c):
    """Storage<PREC>::addr: byte offset of channel c of pixel pix (bf16x3: the hi half; lo is 64 bytes further)."""
    if fmt == 'bf16x3':
        return (pix * C + (c & ~31)) * 4 + (c & 31) * 2
    return (pix * C + c) * (2 if fmt == 'bf16' else 4)


# ------------------------------------------------------------------------------------------- the mode's arithmetic
def arith(li, prec):
    """The arithmetic layer li runs in mode prec: the stems of both bf16 modes read a bf16x3-format input."""
    if LAYERS[li].kind == 'stem' and prec == 'bf16':
        return 'bf16x3'
    return prec


def mode_weights(w_rows, li, prec):
    """The weights as mode prec holds them: a list of (weight rows, which input part they multiply) whose products sum to
    the layer's conv.  Input parts: 'x' (the decoded value) or 'hi' (the hi half of a bf16x3 input)."""
    a = arith(li, prec)
    if a == 'fp32':
        return [(_f32(w_rows), 'x')]
    if a == 'tf32':
        return [(tf32_rna(w_rows), 'x')]
    if a == 'bf16':
        return [(bf16_rne(w_rows), 'x')]
    hi, lo = split2(w_rows)
    return [(hi, 'x'), (lo, 'hi')]                   # hi.w_hi + lo.w_hi + hi.w_lo


def oihw(w_rows, li):
    """K-major rows -> (rows, cin, kh, kw) float64: 3x3 k = (r*3+s)*cin + c; stem k = r*32 + s*4 + c (s = 7 is zero)."""
    L = LAYERS[li]
    w = torch.from_numpy(np.asarray(w_rows, dtype=np.float64))
    if L.kind == 'stem':
        return w.reshape(L.rows, 7, 8, 4).permute(0, 3, 1, 2).contiguous()
    return w.reshape(L.rows, 3, 3, L.cin).permute(0, 3, 1, 2).contiguous()


def conv_terms(xd, w_rows, li, prec):
    """-> (z, S, Q2) float64 (1, rows, Ho, Wo): the conv of the mode's operands, the sum of its products' absolute values
    and the sum of their squares.  One grouped conv2d does all of it."""
    L = LAYERS[li]
    parts = mode_weights(w_rows, li, prec)
    x = torch.from_numpy(np.asarray(xd.value, dtype=np.float64))[None]
    if any(p == 'hi' for _, p in parts):
        if xd.hi is None:
            raise ValueError('bf16x3 arithmetic needs a hi / lo input')
        hi = torch.from_numpy(np.asarray(xd.hi, dtype=np.float64))[None]
        lo = torch.from_numpy(np.asarray(xd.lo, dtype=np.float64))[None]
        absx = hi.abs() + lo.abs()                   # |hi.w| + |lo.w|: the two products of w_hi are summed separately
        sqx = hi * hi + lo * lo
    else:
        hi = absx = sqx = None
    ins, ws = [], []
    for w, part in parts:
        wt = oihw(w, li)
        if part == 'x':
            ins += [x, x.abs() if absx is None else absx, x * x if sqx is None else sqx]
        else:
            ins += [hi, hi.abs(), hi * hi]
        ws += [wt, wt.abs(), wt * wt]
    # a grouped conv over the stacked inputs: block j of the output = conv(ins[j], ws[j])
    G = L.groups
    xs = torch.cat(ins, 1)
    wcat = torch.cat(ws, 0)
    if L.kind == 'stem':                             # the stored 182 x 184 padded input -> 88 x 89; column 88 is not an output
        out = F.conv2d(xs, wcat, stride=2, groups=len(ins))[:, :, :, :88]
    else:
        out = F.conv2d(xs, wcat, stride=L.stride, padding=1, groups=len(ins) * G)
    blocks = out.split(L.rows, 1)
    z = sum(blocks[3 * j] for j in range(len(parts)))
    S = sum(blocks[3 * j + 1] for j in range(len(parts)))
    Q2 = sum(blocks[3 * j + 2] for j in range(len(parts)))
    return z, S, Q2


def act_fp64(z, act):
    return torch.relu(z) if act == RELU else SELU_SCALE * torch.where(z > 0, z, SELU_ALPHA * torch.expm1(torch.clamp(z, max=0.0)))


def eps_act(y, act):
    """Absolute error of the device's activation in the z domain (the gate multiplies it by L).  SELU: selu_fast's
    __expf (ex2.approx: ~2^-22 relative, plus 2^-24 |z| from the z * log2(e) product, <= 2^-24 / e absolute for z < 0),
    the - 1 and the products by lambda / lambda alpha: <= 8 units of 2^-24 absolute plus 1 unit of |y|.  ReLU is exact."""
    if act == RELU:
        return torch.zeros_like(y)
    return U24 * (8.0 + y.abs())


def chain_units(li, prec, ksplit=1):
    """c of the gate: roundings (units of 2^-24) along the longest fp32 accumulation chain of the kernel that runs layer
    li in mode prec.  A tensor-core MMA instruction counts 2 (truncation at 2^-23, module docstring); an FFMA or fp32
    add counts 1.
      fp32 (conv_direct_kernel): one fmaf per K element, then + bias, + residual.
      tf32: one k8 MMA per 8 K elements (4 per 128-byte chunk and tap).  bf16: one k16 MMA per 16 K elements.
      bf16x3 trunk: 6 k16 MMAs per 32-channel chunk and tap into one accumulator = 3K/16.
      bf16x3 resident (stacked [w_hi ; w_lo]): columns 0-63 get hi.w_hi and lo.w_hi = 2K/16 MMAs, columns 64-127 hi.w_lo;
        the epilogue then adds the two halves (+1).  The stems likewise (28 MMAs over K = 224, then the halves, +1).
      trunk latency mode (ksplit > 1 pieces): each piece runs 1/ksplit of the K chunks, then the pieces are added in order
        (ksplit - 1 adds).
      Then + bias (+1) and + residual (+1).  The stems' max-pool is exact."""
    L = LAYERS[li]
    a = arith(li, prec)
    K = L.ktot
    if a == 'fp32':
        return K + 1 + (1 if L.res else 0)
    if a == 'tf32':
        n = K // 8
    elif a == 'bf16':
        n = K // 16
    elif L.trunk:
        n = 3 * K // 16
    else:
        n = 2 * K // 16
    units = 2 * n
    if L.trunk and ksplit > 1:
        units = 2 * (n // ksplit) + (ksplit - 1)
    if a == 'bf16x3' and not L.trunk:
        units += 1                                   # the stacked halves' sum
    return units + 1 + (1 if L.res else 0)


def trunk_ksplit(n, prec):
    """run_network's split-K choice: kSplitK = 4 pieces for n <= 4 images, halved while a trunk layer's 128-byte K
    chunk count is not divisible (2-byte storage: convAB1 has two)."""
    if prec == 'fp32' or n > 4:
        return 1
    ks = 4
    bpc = 2 if prec == 'bf16' else 4
    for L in LAYERS[FIRST_TRUNK:]:
        while (L.cin * bpc // 128) % ks:
            ks //= 2
    return ks


class Ref:
    """Reference of one layer: y (fp64 NCHW, no batch dim), the gate's per-element scales and constants."""
    def __init__(self, y, S, Q, c, L, u_out, eps, extra_B=None, extra_Q=None):
        self.y, self.S, self.Q, self.c, self.L, self.u_out, self.eps = y, S, Q, c, L, u_out, eps
        self.extra_B = extra_B if extra_B is not None else torch.zeros_like(y)
        self.extra_Q = extra_Q if extra_Q is not None else torch.zeros_like(y)

    def bound(self):
        """Per-element worst-case bound of gate 1."""
        B = self.L * (self.c * U24 * self.S + self.eps + self.extra_B)
        return B + self.u_out * (self.y.abs() + B) + TINY

    def scale(self):
        """Per-element denominator of gate 2."""
        return self.L * (self.c * U24 * self.Q + self.eps + self.extra_Q) + self.u_out * self.y.abs() + TINY


def layer_ref(li, prec, x, w_rows, b, res=None, ksplit=1, out_fmt=None, pool=None):
    """Reference of layer li in mode prec from its decoded input x (Decoded) and residual res (Decoded or None).
    pool: for the stems, True = the fused max-pool of the tensor-core modes (output 44 x 44), False = the fp32 mode's
    stored 88 x 88 conv.  Default: fused pool unless prec is fp32."""
    L = LAYERS[li]
    if pool is None:
        pool = prec != 'fp32'
    z, S, Q2 = conv_terms(x, w_rows, li, prec)
    bb = torch.from_numpy(np.asarray(b, dtype=np.float64))[None, :, None, None]
    if L.kind == 'stem' and pool:
        z = F.max_pool2d(z, 3, 2, 1)                 # -inf padding, like the kernel's staging tile
        S = F.max_pool2d(S, 3, 2, 1)
        Q2 = F.max_pool2d(Q2, 3, 2, 1)
    z = z + bb
    S = S + bb.abs()
    if res is not None:
        r = torch.from_numpy(np.asarray(res.value, dtype=np.float64))[None]
        z = z + r
        S = S + r.abs()
    y = act_fp64(z, L.act)
    out_fmt = out_fmt or prec
    return Ref(y[0], S[0], Q2[0].sqrt(), chain_units(li, prec, ksplit), L.L, U_OUT[out_fmt], eps_act(y[0], L.act))


def chained_ref(li_first, prec, x, w1, b1, w2, b2, res2, ksplit=1):
    """Two layers from the first one's input, for the one intermediate that is overwritten (convB2.conv1's output T2,
    reused by convB3.conv1): the first layer's output is rounded into the storage format as the device does, then fed to
    the second.  The first layer's worst-case error E1 (its gate-1 bound, plus the reference's own storage rounding
    u_out |y1|) enters the second layer's bound through the absolute weights: extra = conv(|w2|, E1), and in quadrature
    through the squared weights for gate 2.  In bf16x3 a perturbed input also moves its hi half, which multiplies w_lo: that
    adds |w_lo| (|dx| + 2^-8 (|x| + |dx|)) per product."""
    r1 = layer_ref(li_first, prec, x, w1, b1, ksplit=ksplit)
    y1 = r1.y.float().numpy()
    buf = LAYERS[li_first].out
    x2 = decode(encode(y1, buf, prec), buf, prec)
    E1 = r1.bound() + r1.u_out * r1.y.abs()
    li2 = li_first + 1
    r2 = layer_ref(li2, prec, x2, w2, b2, res=res2, ksplit=ksplit)
    L2 = LAYERS[li2]
    extra_B = torch.zeros_like(r2.y)
    extra_Q2 = torch.zeros_like(r2.y)
    for w, part in mode_weights(w2, li2, prec):
        wt = oihw(w, li2).abs()
        e = E1[None]
        if part == 'hi':
            e = e + 2.0 ** -8 * (torch.from_numpy(np.asarray(x2.value, dtype=np.float64)).abs()[None] + E1[None])
        extra_B = extra_B + F.conv2d(e, wt, padding=1, groups=L2.groups)[0]
        extra_Q2 = extra_Q2 + F.conv2d(e * e, wt * wt, padding=1, groups=L2.groups)[0]
    r2.extra_B, r2.extra_Q = extra_B, extra_Q2.sqrt()
    return r1, r2


class GateResult:
    def __init__(self, worst, rms, finite, count, where=None):
        self.worst, self.rms, self.finite, self.count, self.where = worst, rms, finite, count, where

    @property
    def ok(self):
        return self.finite and self.worst <= 1.0 and self.rms <= 1.0

    def __repr__(self):
        return 'worst %.3g rms %.3g%s' % (self.worst, self.rms, '' if self.finite else ' NON-FINITE')


def gate(y_dev, ref):
    """Both gates of one layer: y_dev (C, H, W) array / tensor as decoded from the device (or a stand-in)."""
    yd = torch.as_tensor(np.asarray(y_dev, dtype=np.float64)) if not torch.is_tensor(y_dev) else y_dev.double()
    if yd.shape != ref.y.shape:
        raise ValueError('shape %s vs reference %s' % (tuple(yd.shape), tuple(ref.y.shape)))
    finite = bool(torch.isfinite(yd).all())
    err = (yd - ref.y)
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, math.inf))
    r1 = err.abs() / ref.bound()
    r2 = err / ref.scale()
    worst = float(r1.max())
    rms = float(torch.sqrt((r2 * r2).mean())) if finite else math.inf
    where = tuple(int(i) for i in np.unravel_index(int(torch.argmax(r1)), tuple(r1.shape)))
    return GateResult(worst, rms, finite, r1.numel(), where)


# ------------------------------------------------------------------------------------------- the head
C_POOL_TC = 10     # head_pooled_kernel on pool_part: 4 rows per lane (3 adds), 2 shuffle adds, 8 slices pairwise (3), x 1/121 and its rounding (2)
C_POOL_FP32 = 34   # head_kernel on H3: ~31 pixels per thread group summed in sequence, 2 pairwise adds, x 1/121 and its rounding
C_FC = 13          # 4 products per thread (<= 4 roundings), 5 shuffle adds, 4 warps' partials + bias (4 adds)


def head_ref(h_relu, h_bound, fcw, fcb, c_pool):
    """tanh(W_fc . mean(h) + b_fc) for both heads (channels 0-511 -> trans with fc rows 0-2, 512-1023 -> rot with rows 3-5)
    from the last layer's activation h (1024, 11, 11) fp64 and its elementwise bound; -> (out (6,), bound (6,)).
    The bound propagates h's through the mean and |W_fc| (tanh' <= 1), plus the head's own fp32 roundings and tanhf's
    2-ulp error."""
    m = h_relu.reshape(1024, -1).mean(1)
    dm = h_bound.reshape(1024, -1).mean(1) + c_pool * U24 * h_relu.abs().reshape(1024, -1).mean(1)
    W = torch.from_numpy(np.asarray(fcw, dtype=np.float64))
    bf = torch.from_numpy(np.asarray(fcb, dtype=np.float64))
    pre = torch.empty(6, dtype=torch.float64)
    dpre = torch.empty(6, dtype=torch.float64)
    for h in range(2):
        mh, dmh = m[512 * h:512 * (h + 1)], dm[512 * h:512 * (h + 1)]
        Wh = W[3 * h:3 * h + 3]
        pre[3 * h:3 * h + 3] = Wh @ mh + bf[3 * h:3 * h + 3]
        dpre[3 * h:3 * h + 3] = Wh.abs() @ dmh + C_FC * U24 * (Wh.abs() @ mh.abs() + bf[3 * h:3 * h + 3].abs())
    out = torch.tanh(pre)
    return out, dpre + 2.0 ** -22 * out.abs() + TINY
