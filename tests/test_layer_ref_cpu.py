"""oracle/layer_ref.py on the CPU: its encoders / decoders against the device's storage formats, and its per-layer gate
against a stand-in of the device arithmetic (CPU float32 convs of the same emulated operands) -- it must accept that,
and reject each of a list of plausible kernel bugs applied to it.  tests/test_gpu_layers.py runs the same gate on the
device's buffers."""
import functools
import math
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_ref as R


# ------------------------------------------------------------------------------------------- encoders / decoders
def _f(bits):
    return np.array(bits, dtype=np.uint32).view(np.float32)


def test_tf32_rna_ties_away_and_round_trip():
    # a tie (exactly half of the 13 dropped bits) rounds AWAY from zero in both signs; below / above it to nearest
    one = 0x3F800000
    assert R.tf32_rna(_f([one | 0x1000]))[0] == _f([one + 0x2000])[0]
    assert R.tf32_rna(_f([one | 0x80000000 | 0x1000]))[0] == _f([(one + 0x2000) | 0x80000000])[0]
    assert R.tf32_rna(_f([one | 0x0FFF]))[0] == 1.0
    assert R.tf32_rna(_f([one | 0x3000]))[0] == _f([one + 0x4000])[0]          # a tie whose kept bits are odd: still away
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.normal(size=5000), rng.normal(size=1000) * 1e30, rng.normal(size=1000) * 1e-40,   # large, subnormal
                        -np.abs(rng.normal(size=1000))]).astype(np.float32)
    t = R.tf32_rna(x)
    assert np.array_equal(R.tf32_rna(t), t)                                      # idempotent: tf32 values are kept
    assert (t.view(np.uint32) & 0x1FFF).max() == 0
    fin = np.isfinite(t)
    # subnormals keep 10 bits of their fixed-point mantissa: half of 2^-136 absolute
    assert np.all(np.abs(t[fin].astype(np.float64) - x[fin]) <= 2.0 ** -11 * np.abs(x[fin]) + 2.0 ** -137)
    assert np.isinf(R.tf32_rna(np.array([np.finfo(np.float32).max], np.float32))[0])   # rounds up past the largest tf32


def test_bf16_rne_ties_to_even_and_split():
    one = 0x3F800000
    assert R.bf16_rne(_f([one | 0x8000]))[0] == 1.0                             # tie, even kept bits: down
    assert R.bf16_rne(_f([(one + 0x10000) | 0x8000]))[0] == _f([one + 0x20000])[0]   # tie, odd: up
    assert R.bf16_rne(_f([one | 0x80000000 | 0x8001]))[0] == -_f([one + 0x10000])[0]
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.normal(size=5000), rng.normal(size=500) * 3e37, rng.normal(size=500) * 1e-39,
                        -np.abs(rng.normal(size=500)), _f([one | 0x8000, (one + 0x10000) | 0x8000])]).astype(np.float32)
    b = R.bf16_rne(x)
    assert np.array_equal(R.bf16_rne(b), b)
    hi, lo = R.split2(x)
    assert np.array_equal(hi, b)
    fin = np.isfinite(hi + lo) & (np.abs(x) > 1e-30)
    rel = np.abs((hi.astype(np.float64) + lo) - x)[fin] / np.abs(x[fin])
    assert rel.max() <= 2.0 ** -16                                              # hi + lo holds x to 16 bits


@pytest.mark.parametrize('fmt', ['tf32', 'bf16x3', 'bf16', 'fp32'])
def test_encode_decode_round_trip(fmt):
    rng = np.random.default_rng(2)
    v = (rng.normal(size=(128, 44, 44)) * np.exp(rng.normal(size=(128, 44, 44)) * 4)).astype(np.float32)
    v[0, 0, :4] = [0.0, -0.0, 1e-41, -3e38]
    raw = R.encode(v, 'CAT', fmt)
    assert raw.size == R.image_bytes('CAT', fmt)
    d = R.decode(raw, 'CAT', fmt)
    expect = {'tf32': R.tf32_rna(v), 'bf16': R.bf16_rne(v), 'fp32': v}.get(fmt)
    if fmt == 'bf16x3':
        hi, lo = R.split2(v)
        expect = hi + lo
        assert np.array_equal(d.hi, hi) and np.array_equal(d.lo, lo)
    assert np.array_equal(d.value, expect)
    # stored values are kept by a second encode (in bf16x3 a tie may swap which half holds the last bit, so compare values)
    assert np.array_equal(R.decode(R.encode(d.value, 'CAT', fmt), 'CAT', fmt).value, d.value)


@pytest.mark.parametrize('fmt', ['tf32', 'bf16x3', 'bf16'])
def test_byte_layout_matches_storage_addr(fmt):
    """A value written at (pixel, channel) sits where Storage<PREC>::addr puts it (bf16x3: its lo half 64 bytes further)."""
    C, H, W = 128, 44, 44
    v = np.zeros((C, H, W), np.float32)
    cases = [(0, 0), (1, 31), (45, 32), (100, 63), (44 * 44 - 1, 127), (7, 96)]
    for k, (pix, c) in enumerate(cases):
        v[c, pix // W, pix % W] = 1.0 + 2.0 ** -12 * (k + 1) + (2.0 ** -20 if fmt == 'bf16x3' else 0.0)
    raw = R.encode(v, 'CAT', fmt)
    for pix, c in cases:
        a = R.storage_addr(fmt, pix, C, c)
        y = v[c, pix // W, pix % W]
        if fmt == 'tf32':
            assert raw[a:a + 4].view(np.float32)[0] == R.tf32_rna(np.float32(y)[None])[0]
        else:
            hi, lo = R.split2(np.float32(y)[None])
            assert raw[a:a + 2].view(np.uint16)[0] == R.bf16_bits(hi)[0]
            if fmt == 'bf16x3':
                assert raw[a + 64:a + 66].view(np.uint16)[0] == R.bf16_bits(lo)[0] and lo[0] != 0
    # the addresses written out for a few cases
    assert R.storage_addr('bf16x3', 1, 128, 33) == (128 + 32) * 4 + 2 and R.storage_addr('bf16', 1, 128, 33) == (128 + 33) * 2
    assert R.storage_addr('tf32', 2, 64, 5) == (128 + 5) * 4


def test_stem_input_format():
    """X0A / X0B: 16 bytes per pixel in every mode; both bf16 modes store [4 x bf16 hi | 4 x bf16 lo]."""
    rng = np.random.default_rng(3)
    v = np.zeros((4, 182, 184), np.float32)
    v[:, 3:179, 3:179] = rng.normal(size=(4, 176, 176)) * 30
    for prec in ('tf32', 'bf16x3', 'bf16', 'fp32'):
        fmt = R.buf_format('X0A', prec)
        raw = R.encode(v, 'X0A', fmt)
        assert raw.size == 182 * 184 * 16
        p = (5 * 184 + 7) * 16                                                  # pixel (5, 7)
        if fmt == 'stem_hilo':
            hi, lo = R.split2(v[:, 5, 7])
            assert np.array_equal(raw[p:p + 8].view(np.uint16), R.bf16_bits(hi))
            assert np.array_equal(raw[p + 8:p + 16].view(np.uint16), R.bf16_bits(lo))
        d = R.decode(raw, 'X0A', fmt)
        assert d.value.shape == (4, 182, 184) and np.abs(d.value - v).max() <= 2.0 ** -11 * np.abs(v).max()
    assert R.image_bytes('H1', 'bf16') * 2 == R.image_bytes('H1', 'bf16x3')    # bf16: half the image stride


def test_layer_table_matches_blob():
    w_off, b_off, fc = R.blob_offsets()
    assert fc + R.FC_FLOATS == 13528326                                         # SE3TN_WEIGHT_BLOB_FLOATS
    assert R.LAYERS[13].res == 'H1' and R.LAYERS[12].groups == 2 and R.LAYERS[8].stride == 2
    assert [L.out for L in R.LAYERS].count('T2') == 2                          # the one reused intermediate


# ------------------------------------------------------------------------------------------- the gate vs a stand-in
@functools.lru_cache(maxsize=None)
def _blob(seed):
    from importlib import import_module
    synth = import_module('iros20-6d-pose-tracking_b200.synth')
    weights = import_module('iros20-6d-pose-tracking_b200.weights')
    return weights.pack_state_dict(synth.make_state_dict(seed))


def _activation(buf, rng, selu=False):
    _, H, W, C = R.BUFS[R.BUF_ID[buf]]
    z = rng.normal(size=(C, H, W))
    if buf in ('X0A', 'X0B'):
        v = np.zeros((4, 182, 184))
        v[:, 3:179, 3:179] = z[:, 3:179, 3:179] * 3
        return v.astype(np.float32)
    y = np.where(z > 0, R.SELU_SCALE * z, R.SELU_L * np.expm1(np.minimum(z, 0))) if selu else np.maximum(z, 0)
    return y.astype(np.float32)


IN_SELU = {'X0A': False, 'P1A': True, 'T1': False, 'CAT': False, 'H1': True, 'H2': False, 'F2': False}


@functools.lru_cache(maxsize=None)
def _case(li, prec, seed):
    """Stored input / residual of layer li in mode prec (synthetic activations), and the layer's reference."""
    L = R.LAYERS[li]
    rng = np.random.default_rng(100 * li + seed)
    fin = R.buf_format(L.inp, prec)
    x = R.decode(R.encode(_activation(L.inp, rng, IN_SELU[L.inp]), L.inp, fin), L.inp, fin)
    res = None
    if L.res:
        res = R.decode(R.encode(_activation(L.res, rng, IN_SELU[L.res]), L.res, prec), L.res, prec)
    w, b = R.layer_weights(_blob(seed), li)
    return x, res, w, b, R.layer_ref(li, prec, x, w, b, res=res)


def stand_in(li, prec, x, w, b, res=None, mut=None, w_other=None):
    """The layer as the device computes it, on the CPU in float32: the mode's operands, fp32 sums, fp32 bias / residual /
    activation, output encoded into the storage format and decoded back.  `mut` applies one deliberate bug."""
    L = R.LAYERS[li]
    mut = mut or ''
    if mut == 'other_weights':
        w = w_other
    parts = R.mode_weights(w, li, prec)
    if mut == 'tf32_truncated':
        parts = [(R.tf32_trunc(w), 'x')]
    xv = torch.from_numpy(x.value.copy())[None]
    xh = torch.from_numpy(x.hi.copy())[None] if x.hi is not None else None
    if mut == 'lo_dropped':                                  # one 32-channel chunk read as hi only (bf16x3 -> bf16)
        xv[:, 32:64] = xh[:, 32:64]
    acc = 0
    for wr, part in parts:
        wt = R.oihw(wr, li).float()
        if mut == 'tap_shifted':                             # filter tap (0, 0) applied one pixel to the right
            wt = wt.clone(); wt[:, :, 0, 1] += wt[:, :, 0, 0]; wt[:, :, 0, 0] = 0
        inp = xv if part == 'x' else xh
        if L.kind == 'stem':
            acc = acc + F.conv2d(inp, wt, stride=2)[:, :, :, :88]
        else:
            acc = acc + F.conv2d(inp, wt, stride=L.stride, padding=1, groups=L.groups)
    bias = torch.from_numpy(b.copy())
    if mut == 'bias_block':                                 # output block 1's bias used for block 0
        n = L.block_n
        bias = bias.clone(); bias[:n] = bias[n:2 * n]
    if L.kind == 'stem' and prec != 'fp32':
        if mut == 'pool_window':                            # pooled row / column p from conv rows 2p .. 2p + 2 (window at 10t)
            acc = F.max_pool2d(F.pad(acc, (0, 1, 0, 1), value=-math.inf), 3, 2, 0)
        else:
            acc = F.max_pool2d(acc, 3, 2, 1)
    v = acc + bias[None, :, None, None]
    if res is not None and mut != 'res_omitted':
        v = v + torch.from_numpy(res.value.copy())[None] * (2 if mut == 'res_doubled' else 1)
    v = torch.relu(v) if L.act == R.RELU else F.selu(v)
    v = v[0].numpy().copy()
    if mut == 'rows_shifted':                               # tile (0, 0): tile row p written with row p + 1's value
        t = v[:, :11, :11].reshape(v.shape[0], 121).copy()
        t[:, :120] = t[:, 1:121]
        v[:, :11, :11] = t.reshape(-1, 11, 11)
    if mut == 'tile_unwritten':                             # tile (1, 1) keeps the 0xFF poison: NaN
        v[:, 11:22, 11:22] = np.nan
    buf = 'Y1A' if (L.kind == 'stem' and prec == 'fp32') else ('T1' if L.out == 'CAT' else L.out)   # CAT: a 64-channel half
    return R.decode(R.encode(v, buf, prec), buf, prec).value


ACCEPT = [(0, 'stem'), (3, 'resident 44x44x64 + residual'), (8, 'convAB1 stride 2'), (12, 'grouped 1024-channel')]


@pytest.mark.parametrize('seed', [0, 1])
@pytest.mark.parametrize('prec', ['bf16x3', 'tf32', 'bf16', 'fp32'])
@pytest.mark.parametrize('li', [a[0] for a in ACCEPT])
def test_gate_accepts_device_arithmetic(li, prec, seed):
    """Legitimate arithmetic passes both gates.  Where the output format rounds coarsely (tf32, bf16) one element's
    rounding error can reach u_out |y| itself, so gate 1's worst ratio may approach 1 there; elsewhere, and for gate 2
    everywhere, the stand-in must stay at or below half of the gate."""
    x, res, w, b, ref = _case(li, prec, seed)
    if li == 0 and prec == 'fp32':
        ref = R.layer_ref(0, prec, x, w, b, pool=False)
    g = R.gate(stand_in(li, prec, x, w, b, res), ref)
    print('%-24s %-6s seed %d: %r (c = %d)' % (R.LAYERS[li].name, prec, seed, g, ref.c))
    assert g.finite and g.rms <= 0.5, g
    assert g.worst <= (1.0 if prec in ('tf32', 'bf16') else 0.5), g


MUTATIONS = [
    # (mutation, layer, mode)
    ('tap_shifted', 3, 'bf16x3'), ('tap_shifted', 12, 'bf16'),
    ('lo_dropped', 3, 'bf16x3'), ('lo_dropped', 8, 'bf16x3'), ('lo_dropped', 12, 'bf16x3'),
    ('tf32_truncated', 3, 'tf32'), ('tf32_truncated', 8, 'tf32'), ('tf32_truncated', 12, 'tf32'),
    ('bias_block', 8, 'bf16x3'), ('bias_block', 12, 'bf16'),
    ('res_omitted', 3, 'bf16x3'), ('res_doubled', 3, 'bf16x3'), ('res_omitted', 3, 'bf16'),
    ('other_weights', 3, 'bf16x3'), ('other_weights', 12, 'tf32'),
    ('rows_shifted', 8, 'bf16x3'), ('rows_shifted', 12, 'bf16'),
    ('tile_unwritten', 8, 'bf16x3'),
    ('pool_window', 0, 'bf16x3'), ('pool_window', 0, 'tf32'),
]


@pytest.mark.parametrize('seed', [0, 1])
@pytest.mark.parametrize('mut,li,prec', MUTATIONS, ids=['%s-%s-%s' % (m, R.LAYERS[li].name, p) for m, li, p in MUTATIONS])
def test_gate_rejects_mutation(mut, li, prec, seed):
    x, res, w, b, ref = _case(li, prec, seed)
    w_other = R.layer_weights(_blob(1 - seed), li)[0] if mut == 'other_weights' else None
    g = R.gate(stand_in(li, prec, x, w, b, res, mut=mut, w_other=w_other), ref)
    over = max(g.worst, g.rms)
    print('mutation %-15s %-24s %-6s seed %d: %r -> %.3gx over the gate' % (mut, R.LAYERS[li].name, prec, seed, g, over))
    assert not g.ok, 'mutation %s on %s (%s) passes the gate: %r' % (mut, R.LAYERS[li].name, prec, g)


def test_chained_bound_accepts_stand_in():
    """convB2.conv1 -> convB2.conv2 through the overwritten T2: the stand-in's rounded intermediate feeds the second layer,
    and the chained bound (first layer's error pushed through |w2|) accepts the result."""
    blob = _blob(0)
    for prec in ('bf16x3', 'tf32', 'bf16'):
        rng = np.random.default_rng(7)
        x = R.decode(R.encode(_activation('P1A', rng, True), 'P1B', prec), 'P1B', prec)
        w1, b1 = R.layer_weights(blob, 4)
        w2, b2 = R.layer_weights(blob, 5)
        r1, r2 = R.chained_ref(4, prec, x, w1, b1, w2, b2, res2=x)
        t2 = stand_in(4, prec, x, w1, b1)
        t2d = R.decode(R.encode(t2, 'T2', prec), 'T2', prec)
        g1 = R.gate(t2, r1)
        g2 = R.gate(stand_in(5, prec, t2d, w2, b2, res=x), r2)
        print('chained %s: conv1 %r, conv2 %r' % (prec, g1, g2))
        assert g1.ok and g2.ok


def test_sample_images_sees_two_weight_sets():
    """The device tests' image sample (tests/layer_harness.py): with weight ids given it holds the first image's id and another
    one whenever the call has another; without a second id in the call it is the plain seeded sample."""
    from layer_harness import sample_images
    for seed in range(20):
        plain = sample_images(3, 12, seed)
        assert sample_images(3, 12, seed, [5] * 12) == plain and len(plain) == 4 and {3, 14} <= set(plain)
        for j in range(1, 11):                       # one image of another id, anywhere between the first and the last
            ids = [5] * 12
            ids[j] = 2
            got = sample_images(3, 12, seed, ids)
            assert 3 + j in got and {3, 14} <= set(got) and set(got) <= set(range(3, 15)), (seed, j, got)
            if 3 + j in plain:
                assert got == plain
