"""oracle/fp16_ref.py on the CPU: its fp16 encoder against numpy's float16 (every bit pattern, ties, subnormals and
saturation), the byte layout, and the 'fp16' gate against a CPU stand-in of the mode's arithmetic -- it must accept that,
and reject each of a list of plausible kernel bugs applied to it.  tests/test_gpu_fp16.py runs the same gate on the
device's buffers."""
import functools
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fp16_ref as H
import layer_ref as R


# ------------------------------------------------------------------------------------------- the format
def test_every_pattern_round_trips_as_numpy_float16():
    bits = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    v = H.f16_value(bits)
    assert np.array_equal(v, bits.view(np.float16).astype(np.float32), equal_nan=True)
    fin = np.isfinite(v)
    assert np.array_equal(H.f16_bits(v[fin]), bits[fin])                        # every finite value, +-0 and subnormals kept
    assert np.isnan(H.f16_value(H.f16_bits(np.array([np.nan], np.float32))))[0]
    assert H.f16_value(np.array([0x7BFF, 0x0400, 0x0001, 0x8000], np.uint16)).tolist() == [65504.0, 2.0 ** -14, 2.0 ** -24, 0.0]


def test_rounding_matches_numpy_float16():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.normal(size=20000), rng.normal(size=5000) * 3e4, rng.normal(size=5000) * 1e-6,
                        rng.normal(size=2000) * 1e-8]).astype(np.float32)
    x = x[np.abs(x) <= H.F16_MAX]
    assert np.array_equal(H.f16_bits(x), x.astype(np.float16).view(np.uint16))
    # ties: the midpoint of two neighbours goes to the even pattern, in both signs and among the subnormals
    pos = np.arange(0x0000, 0x7BFF, dtype=np.uint16)
    lo, hi = H.f16_value(pos), H.f16_value(pos + 1)
    mid = ((lo.astype(np.float64) + hi) / 2).astype(np.float32)                   # exact in fp32
    want = np.where(pos % 2 == 0, pos, pos + 1).astype(np.uint16)
    assert np.array_equal(H.f16_bits(mid), want)
    assert np.array_equal(H.f16_bits(-mid), want | 0x8000)


def test_saturation():
    big = np.array([65504.0, 65519.0, 65520.0, 70000.0, 1e30, np.inf], np.float32)
    assert (H.f16_bits(big) == 0x7BFF).all() and (H.f16_bits(-big) == 0xFBFF).all()
    with np.errstate(over='ignore'):
        assert np.isinf(big[2:].astype(np.float16)).all()                         # numpy alone would overflow to inf


def test_encode_decode_and_byte_layout():
    rng = np.random.default_rng(2)
    v = (rng.normal(size=(128, 44, 44)) * np.exp(rng.normal(size=(128, 44, 44)) * 3)).astype(np.float32)
    v[0, 0, :4] = [0.0, -0.0, 1e-8, -3e38]
    raw = H.encode(v, 'CAT')
    assert raw.size == H.image_bytes('CAT') == R.image_bytes('CAT', 'bf16')       # 2 bytes per channel: bf16's stride
    assert np.array_equal(H.decode(raw, 'CAT').value, H.f16_rne(v))
    for pix, c in [(0, 0), (1, 31), (45, 32), (100, 63), (44 * 44 - 1, 127), (7, 96)]:
        a = H.storage_addr('fp16', pix, 128, c)
        assert a == R.storage_addr('bf16', pix, 128, c)
        assert raw[a:a + 2].view(np.uint16)[0] == H.f16_bits(v[c, pix // 44, pix % 44][None])[0]
    assert H.buf_format('X0A') == 'stem_hilo' and H.trunk_ksplit(1) == R.trunk_ksplit(1, 'bf16') == 2


# ------------------------------------------------------------------------------------------- the gate vs a stand-in
@functools.lru_cache(maxsize=None)
def _blob(seed):
    from importlib import import_module
    synth = import_module('iros20-6d-pose-tracking_b200.synth')
    weights = import_module('iros20-6d-pose-tracking_b200.weights')
    return weights.pack_state_dict(synth.make_state_dict(seed))


def _activation(buf, rng, scale=1.0):
    _, Hh, W, C = R.BUFS[R.BUF_ID[buf]]
    z = rng.normal(size=(C, Hh, W))
    if buf in ('X0A', 'X0B'):
        v = np.zeros((4, 182, 184))
        v[:, 3:179, 3:179] = z[:, 3:179, 3:179] * 3
        return (v * scale).astype(np.float32)
    return (np.maximum(z, 0) * scale).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _case(li, seed, scale=1.0):
    """Stored input / residual of layer li in the mode (synthetic activations), and the layer's reference."""
    L = R.LAYERS[li]
    rng = np.random.default_rng(100 * li + seed)
    x = H.decode(H.encode(_activation(L.inp, rng, scale), L.inp), L.inp)
    res = H.decode(H.encode(_activation(L.res, rng, scale), L.res), L.res) if L.res else None
    w, b = R.layer_weights(_blob(seed), li)
    return x, res, w, b, H.layer_ref(li, x, w, b, res=res)


def stand_in(li, x, w, b, res=None, mut=None):
    """The layer as the device computes it, on the CPU in float32: the mode's operands, fp32 sums, fp32 bias / residual /
    activation, output encoded to fp16 and decoded back.  `mut` applies one deliberate bug: 'wrong_chunk' (the first
    64-channel K chunk read from the second), 'lost_tap' (filter tap (1, 1) dropped), 'bf16' (bf16 rounding of weights and
    output instead of fp16), 'no_saturation' (|x| > 65504 stored as inf), 'res_omitted'."""
    L = R.LAYERS[li]
    parts = H.mode_weights(w, li)
    if mut == 'bf16':
        parts = R.mode_weights(w, li, 'bf16')
    xv = torch.from_numpy(x.value.copy())[None]
    xh = torch.from_numpy(x.hi.copy())[None] if x.hi is not None else None
    if mut == 'wrong_chunk':
        xv[:, 0:64] = xv[:, 64:128]
    acc = 0
    for wr, part in parts:
        wt = R.oihw(wr, li).float()
        if mut == 'lost_tap':
            wt = wt.clone(); wt[:, :, 1, 1] = 0
        inp = xv if part == 'x' else xh
        if L.kind == 'stem':
            acc = acc + F.conv2d(inp, wt, stride=2)[:, :, :, :88]
        else:
            acc = acc + F.conv2d(inp, wt, stride=L.stride, padding=1, groups=L.groups)
    if L.kind == 'stem':
        acc = F.max_pool2d(acc, 3, 2, 1)
    v = acc + torch.from_numpy(b.copy())[None, :, None, None]
    if res is not None and mut != 'res_omitted':
        v = v + torch.from_numpy(res.value.copy())[None]
    v = (torch.relu(v) if L.act == R.RELU else F.selu(v))[0].numpy()
    if mut == 'bf16':
        return R.bf16_rne(v)
    if mut == 'no_saturation':
        with np.errstate(over='ignore'):
            return v.astype(np.float16).astype(np.float32)
    buf = 'T1' if L.out == 'CAT' else L.out                 # CAT: a 64-channel half
    return H.decode(H.encode(v, buf), buf).value


ACCEPT = [0, 1, 3, 6, 8, 10, 12]


@pytest.mark.parametrize('seed', [0, 1])
@pytest.mark.parametrize('li', ACCEPT)
def test_gate_accepts_fp16_arithmetic(li, seed):
    """The mode's arithmetic passes both gates.  One element's output rounding can reach u_out |y| itself, so gate 1's
    worst ratio may approach 1; gate 2 must stay at or below half of the gate."""
    x, res, w, b, ref = _case(li, seed)
    g = R.gate(stand_in(li, x, w, b, res), ref)
    print('%-24s seed %d: %r (c = %d)' % (R.LAYERS[li].name, seed, g, ref.c))
    assert g.ok and g.rms <= 0.5, g


MUTATIONS = [('wrong_chunk', 8), ('wrong_chunk', 12), ('lost_tap', 3), ('lost_tap', 10), ('bf16', 0), ('bf16', 3),
             ('bf16', 9), ('res_omitted', 3), ('res_omitted', 10)]


@pytest.mark.parametrize('mut,li', MUTATIONS, ids=['%s-%d' % m for m in MUTATIONS])
def test_gate_rejects_mutation(mut, li):
    x, res, w, b, ref = _case(li, 0)
    g = R.gate(stand_in(li, x, w, b, res, mut=mut), ref)
    assert not g.ok, '%s on %s passes the gate: %r' % (mut, R.LAYERS[li].name, g)


def test_saturation_passes_and_inf_fails():
    """Inputs scaled so convA2.conv2's output exceeds 65504: the saturating stand-in passes (the reference saturates as the
    format does), one that stores inf there fails."""
    x, res, w, b, ref = _case(3, 0, 3e4)
    assert float(ref.y.abs().max()) == H.F16_MAX
    g = R.gate(stand_in(3, x, w, b, res), ref)
    assert g.ok, g
    assert not R.gate(stand_in(3, x, w, b, res, mut='no_saturation'), ref).ok


def test_chained_bound_accepts_stand_in():
    """convB2.conv1 -> convB2.conv2 through the overwritten T2, in the mode."""
    blob = _blob(0)
    rng = np.random.default_rng(7)
    x = H.decode(H.encode(_activation('P1B', rng), 'P1B'), 'P1B')
    w1, b1 = R.layer_weights(blob, 4)
    w2, b2 = R.layer_weights(blob, 5)
    r1, r2 = H.chained_ref(4, x, w1, b1, w2, b2, res2=x)
    t2 = stand_in(4, x, w1, b1)
    g1 = R.gate(t2, r1)
    g2 = R.gate(stand_in(5, H.decode(H.encode(t2, 'T2'), 'T2'), w2, b2, res=x), r2)
    assert g1.ok and g2.ok, (g1, g2)


def test_layer_ref_results_unchanged():
    """The extension leaves layer_ref's own tables as they were."""
    assert R.U_OUT == {'tf32': 2.0 ** -11, 'bf16': 2.0 ** -8, 'bf16x3': 2.0 ** -16, 'fp32': 0.0}
    assert H.U_OUT['fp16'] == 2.0 ** -11 and H.chain_units(3) == R.chain_units(3, 'bf16')
