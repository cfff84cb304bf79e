"""oracle/fp8_ref.py on the CPU: its e4m3 encoder against every code of the format, round-to-nearest-even ties and
saturation, and the 'fp8' gate against a CPU stand-in of the mode's arithmetic -- it must accept that, and reject each of
a list of plausible kernel bugs applied to it.  tests/test_gpu_fp8.py runs the same gate on the device's buffers."""
import functools
import math
import numpy as np
import pytest

import fp8_ref as E
import layer_ref as R


# ------------------------------------------------------------------------------------------- the format
def _finite_codes():
    return [c for c in range(256) if c & 0x7F != 0x7F]             # 0x7F / 0xFF are e4m3's NaNs (no infinities)


def test_every_code_round_trips():
    codes = np.array(_finite_codes(), dtype=np.uint8)
    v = E.e4m3_value(codes)
    assert np.array_equal(E.e4m3_bits(v), codes)
    assert np.isnan(E.e4m3_value(np.array([0x7F, 0xFF], np.uint8))).all()
    # the known landmarks: largest normal, smallest normal, smallest subnormal, signed zero
    assert E.e4m3_value(np.array([0x7E, 0x08, 0x01, 0x80], np.uint8)).tolist() == [448.0, 2.0 ** -6, 2.0 ** -9, 0.0]
    assert E.e4m3_bits(np.array([-0.0], np.float32))[0] == 0x80


def test_ties_round_to_even_and_saturation():
    pos = np.array([c for c in _finite_codes() if c < 0x7E], dtype=np.uint8)     # each code and its upper neighbour
    lo, hi = E.e4m3_value(pos), E.e4m3_value(pos + 1)
    mid = ((lo.astype(np.float64) + hi) / 2).astype(np.float32)                  # exact in fp32
    want = np.where(pos % 2 == 0, pos, pos + 1).astype(np.uint8)                  # even mantissa wins
    assert np.array_equal(E.e4m3_bits(mid), want)
    assert np.array_equal(E.e4m3_bits(-mid), want | 0x80)
    # just off the midpoint: to the nearer code
    assert np.array_equal(E.e4m3_bits(np.nextafter(mid, np.float32(0))), pos)
    assert np.array_equal(E.e4m3_bits(np.nextafter(mid, np.float32(1e9))), (pos + 1).astype(np.uint8))
    big = np.array([448.0, 449.0, 464.0, 480.0, 1e30, np.inf], np.float32)
    assert (E.e4m3_bits(big) == 0x7E).all() and (E.e4m3_bits(-big) == 0xFE).all()
    assert np.isnan(E.e4m3_value(E.e4m3_bits(np.array([np.nan], np.float32))))[0]


def test_pow2_scale():
    assert E.pow2_scale(448.0) == 1.0 and E.pow2_scale(449.0) == 2.0 and E.pow2_scale(224.0) == 0.5
    assert E.pow2_scale(0.0) == 1.0
    rng = np.random.default_rng(0)
    for a in np.exp(rng.normal(size=500) * 8):
        s = E.pow2_scale(a)
        assert a / s <= 448.0 < 2 * a / s and math.frexp(s)[0] == 0.5


def test_encode_decode_with_scales():
    rng = np.random.default_rng(3)
    v = (np.maximum(rng.normal(size=(1024, 11, 11)), 0) * 5).astype(np.float32)
    v[512:] *= 16
    s = np.ones(8, np.float32)
    s[4], s[5] = E.pow2_scale(v[:512].max()), E.pow2_scale(v[512:].max())
    raw = E.encode(v, 'H1', s)
    assert raw.size == E.image_bytes('H1')
    d = E.decode(raw, 'H1', s).value
    sc = E.channel_scales('H1', s)[:, None, None]
    assert np.array_equal(d, (E.e4m3_rne(v / sc.astype(np.float32)) * sc).astype(np.float32))
    assert np.all(np.abs(d - v) <= 2.0 ** -4 * np.abs(v) + 2.0 ** -10 * sc)


# ------------------------------------------------------------------------------------------- the gate vs a stand-in
@functools.lru_cache(maxsize=None)
def _blob(seed):
    from importlib import import_module
    synth = import_module('iros20-6d-pose-tracking_b200.synth')
    weights = import_module('iros20-6d-pose-tracking_b200.weights')
    return weights.pack_state_dict(synth.make_state_dict(seed))


def _activation(buf, rng):
    _, H, W, C = R.BUFS[R.BUF_ID[buf]]
    y = np.maximum(rng.normal(size=(C, H, W)), 0) * 2
    if C == 1024:
        y[512:] *= 8                                               # the head groups' scales differ
    return y.astype(np.float32)


@functools.lru_cache(maxsize=None)
def _case(li, seed):
    """Stored e4m3 input / residual of trunk layer li with calibrated scales, and the layer's reference."""
    L = R.LAYERS[li]
    rng = np.random.default_rng(10 * li + seed)
    scales = np.ones(8, np.float32)
    vals = {}
    for buf in {L.inp, L.res} - {None}:
        vals[buf] = _activation(buf, rng)
        if buf in ('H1', 'H2'):
            k = 4 if buf == 'H1' else 6
            scales[k] = E.pow2_scale(vals[buf][:512].max() * E.HEADROOM)
            scales[k + 1] = E.pow2_scale(vals[buf][512:].max() * E.HEADROOM)
        else:
            scales[E.SCALE_NAMES.index(buf)] = E.pow2_scale(vals[buf].max() * E.HEADROOM)
    dec = {b: E.decode(E.encode(v, b, scales), b, scales) for b, v in vals.items()}
    w, b = R.layer_weights(_blob(seed), li)
    x, res = dec[L.inp], dec.get(L.res)
    y = E.layer_ref(li, x, w, b, scales, res=res).y.numpy()       # the output scale from the output's own range
    if li != 13:
        if L.out in ('H1', 'H2'):
            k = 4 if L.out == 'H1' else 6
            scales[k], scales[k + 1] = E.pow2_scale(np.abs(y[:512]).max() * 2), E.pow2_scale(np.abs(y[512:]).max() * 2)
        else:
            scales[E.SCALE_NAMES.index(L.out)] = E.pow2_scale(np.abs(y).max() * 2)
    return x, res, w, b, scales, E.layer_ref(li, x, w, b, scales, res=res)


ACCEPT = [8, 9, 10, 11, 12, 13]


@pytest.mark.parametrize('seed', [0, 1])
@pytest.mark.parametrize('li', ACCEPT)
def test_gate_accepts_fp8_arithmetic(li, seed):
    x, res, w, b, scales, ref = _case(li, seed)
    g = R.gate(E.standin(li, x, w, b, scales, res=res), ref)
    assert g.ok, g
    assert g.rms <= 0.5, g


MUTATIONS = [('row_scale', 9), ('other_group', 12), ('drop_chunk', 10), ('no_residual', 10), ('unscaled_out', 12),
             ('unscaled_out', 9), ('no_residual', 13), ('other_res_group', 13), ('row_scale', 13)]


@pytest.mark.parametrize('mut,li', MUTATIONS, ids=['%s-%d' % m for m in MUTATIONS])
def test_gate_rejects_mutation(mut, li):
    x, res, w, b, scales, ref = _case(li, 0)
    if mut == 'unscaled_out':
        so = E.out_scales(li, scales)
        assert not np.all(so == 1.0)                               # otherwise this bug changes nothing
    if mut == 'other_res_group':
        assert scales[4] != scales[5]
    g = R.gate(E.standin(li, x, w, b, scales, res=res, mutate=mut), ref)
    assert not g.ok, '%s passed the gate: %r' % (mut, g)


def test_cat_writers_reference():
    """convA2.conv2 / convB3.conv2: bf16 arithmetic, e4m3 output with CAT's scale -- a bf16 stand-in encoded to e4m3 passes."""
    import torch
    import torch.nn.functional as F
    li = 3
    rng = np.random.default_rng(5)
    x = R.decode(R.encode(np.maximum(rng.normal(size=(64, 44, 44)), 0).astype(np.float32), 'T1', 'bf16'), 'T1', 'bf16')
    res = R.decode(R.encode(np.maximum(rng.normal(size=(64, 44, 44)), 0).astype(np.float32), 'P1A', 'bf16'), 'P1A', 'bf16')
    w, b = R.layer_weights(_blob(0), li)
    scales = np.ones(8, np.float32)
    y0 = R.layer_ref(li, 'bf16', x, w, b, res=res).y.numpy()
    scales[0] = E.pow2_scale(np.abs(y0).max() * 2)
    ref = E.layer_ref(li, x, w, b, scales, res=res)
    wt = R.oihw(R.bf16_rne(w), li).float()
    v = F.conv2d(torch.from_numpy(x.value)[None], wt, padding=1) + torch.from_numpy(b)[None, :, None, None]
    v = torch.relu(v + torch.from_numpy(res.value)[None])[0].numpy()
    dev = (E.e4m3_rne(v / scales[0]) * scales[0]).astype(np.float32)
    g = R.gate(dev, ref)
    assert g.ok, g
    assert scales[0] != 1.0                                        # otherwise the unscaled output below changes nothing
    assert not R.gate((E.e4m3_rne(v) * scales[0]).astype(np.float32), ref).ok
