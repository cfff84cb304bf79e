"""Device side of the per-layer check (oracle/layer_ref.py is the fp64 side, with oracle/fp16_ref.py and oracle/fp8_ref.py
for those two modes' formats and layers), shared by the test files that run it, in all six precision modes.

Before each call every conv output buffer (P1A ... H2; also Y1A / Y1B and H3 in the fp32 mode) is filled with 0xFF bytes,
a NaN in every storage format, through the debug_buffer view into the Engine's own workspace.  After the call each checked
element must have been overwritten (NaN fails the gate) and every image outside [first, first + n) must still hold the
poison byte for byte.  The stem inputs X0A / X0B are never poisoned: their halo is the conv padding.

Each case checks the 14 layers plus the head on a sample of its images (all of them up to 4; else first, last and two
picked with a seed); `-s` prints a per-layer table of the worst ratio of each gate (gate 1 elementwise worst case, gate 2
RMS; both pass at <= 1).  In 'fp8' an image is checked with the activation scales of its own weight set.
"""
import numpy as np
import torch
import torch.nn.functional as F

import fp16_ref as H
import fp8_ref as E
import layer_ref as R

CONV_OUT = ['P1A', 'P1B', 'T1', 'T2', 'U', 'CAT', 'F1', 'T4', 'F2', 'H1', 'H2']
FP32_OUT = ['Y1A', 'Y1B', 'H3']


def buffer_bytes(eng, buf):
    """The whole debug_buffer allocation of `buf` (max_batch images at 4 bytes per channel) as a uint8 view."""
    return eng.debug_buffer(R.BUF_ID[buf], eng.max_batch).view(torch.uint8).reshape(-1)


def _out_bufs(prec):
    return CONV_OUT + (FP32_OUT if prec == 'fp32' else [])


def image_bytes(buf, prec):
    """Bytes one image of buffer `buf` occupies in mode prec: the buffer's image stride."""
    if prec == 'fp16':
        return H.image_bytes(buf)
    if prec == 'fp8':
        return E.image_bytes(buf)
    return R.image_bytes(buf, R.buf_format(buf, prec))


def decode(raw, buf, prec, scales=None):
    """One image's bytes of buffer `buf` in mode prec -> layer_ref.Decoded; scales: the image's set's fp8 scales."""
    if prec == 'fp16':
        return H.decode(raw, buf)
    if prec == 'fp8':
        return E.decode(raw, buf, scales)
    return R.decode(raw, buf, R.buf_format(buf, prec))


def trunk_ksplit(n, prec):
    """run_network's split-K choice for n images in mode prec."""
    if prec == 'fp16':
        return H.trunk_ksplit(n)
    if prec == 'fp8':
        return E.trunk_ksplit(n)
    return R.trunk_ksplit(n, prec)


def poison(eng, prec):
    for buf in _out_bufs(prec):
        buffer_bytes(eng, buf).fill_(0xFF)


def check_poison_outside(eng, prec, first, n):
    """Images outside [first, first + n) -- and, in the 2-byte bf16 mode, the allocation's unused second half -- still hold
    the poison, byte for byte."""
    bad = []
    for buf in _out_bufs(prec):
        nb = image_bytes(buf, prec)
        u = buffer_bytes(eng, buf)
        for part in (u[:first * nb], u[(first + n) * nb:]):
            if part.numel() and not bool((part == 0xFF).all()):
                bad.append(buf)
    assert not bad, 'written outside images [%d, %d): %s' % (first, first + n, bad)


def sample_images(first, n, seed, wids=None):
    """The images of [first, first + n) to check: all of them up to 4, else first, last and two picked with `seed`.
    wids (the weight id of each image): when the call uses more than one id and the sample does not, one of the two picks is
    replaced by an image of another id than the first image's, so that the sample always sees two weight sets."""
    if n <= 4:
        return list(range(first, first + n))
    rng = np.random.default_rng(seed)
    mid = [int(i) for i in rng.choice(np.arange(first + 1, first + n - 1), size=2, replace=False)]
    if wids is not None:
        w = np.asarray(wids)
        other = np.flatnonzero(w != w[0])
        if other.size and (w[np.array(mid) - first] == w[0]).all() and w[-1] == w[0]:
            mid[0] = first + int(rng.choice(other))
    return sorted({first, first + n - 1, *mid})


def _head_row(out, bound, six):
    d = torch.as_tensor(np.asarray(six, dtype=np.float64))
    finite = bool(torch.isfinite(d).all())
    return ('head (trans, rot)', R.GateResult(float(((d - out).abs() / bound).max()) if finite else np.inf, 0.0, finite, 6))


def check_image(raw, prec, blob, ksplit, six, scales=None):
    """All 14 layers and the head of one image ('fp8': the layers fp8_ref checks).  raw(buf) -> that image's bytes of
    buffer buf; blob: the image's fp32 weight blob; six: the (6,) trans ++ rot the call returned for it; scales: its set's
    fp8 scales.  -> [(layer name, GateResult)]."""
    D = {}

    def dec(buf):
        if buf not in D:
            D[buf] = decode(raw(buf), buf, prec, scales)
        return D[buf]

    if prec == 'fp8':
        return _check_image_fp8(dec, blob, scales, six)
    if prec == 'fp16':
        layer_ref = lambda li, x, w, b, **kw: H.layer_ref(li, x, w, b, **kw)
        chained_ref = lambda li, x, *wb, **kw: H.chained_ref(li, x, *wb, **kw)
    else:
        layer_ref = lambda li, x, w, b, **kw: R.layer_ref(li, prec, x, w, b, **kw)
        chained_ref = lambda li, x, *wb, **kw: R.chained_ref(li, prec, x, *wb, **kw)
    W = lambda li: R.layer_weights(blob, li)
    rows = []

    def one(li, out_value, res=None, **kw):
        L = R.LAYERS[li]
        w, b = W(li)
        ref = layer_ref(li, dec(L.inp), w, b, res=dec(res) if res else None, ksplit=ksplit, **kw)
        rows.append((L.name, R.gate(out_value, ref)))
        return ref

    cat = dec('CAT').value                          # convA2.conv2 writes channels 0-63, convB3.conv2 64-127
    # stems: the tensor-core modes store the fused max-pool, the fp32 mode the conv (Y1) and then a separate max-pool
    for li, y1, p1 in ((0, 'Y1A', 'P1A'), (1, 'Y1B', 'P1B')):
        if prec == 'fp32':
            one(li, dec(y1).value, pool=False)
            pooled = F.max_pool2d(torch.from_numpy(dec(y1).value)[None], 3, 2, 1)[0].numpy()
            same = np.array_equal(pooled, dec(p1).value, equal_nan=False)
            rows.append(('maxpool %s -> %s (bit-exact)' % (y1, p1), R.GateResult(0.0 if same else np.inf, 0.0, same, pooled.size)))
        else:
            one(li, dec(p1).value)
    one(2, dec('T1').value)
    one(3, cat[:64], res='P1A')
    # convB2.conv1's output T2 is overwritten by convB3.conv1: check convB2.conv2 through both layers from P1B
    w4, b4 = W(4); w5, b5 = W(5)
    _, r5 = chained_ref(4, dec('P1B'), w4, b4, w5, b5, res2=dec('P1B'), ksplit=ksplit)
    rows.append((R.LAYERS[4].name + ' + conv2', R.gate(dec('U').value, r5)))
    one(6, dec('T2').value)
    one(7, cat[64:], res='U')
    one(8, dec('F1').value)
    one(9, dec('T4').value)
    one(10, dec('F2').value, res='F1')
    one(11, dec('H1').value)
    one(12, dec('H2').value)
    fcw, fcb = R.fc_weights(blob)
    if prec == 'fp32':
        one(13, dec('H3').value, res='H1')
        h3 = torch.from_numpy(dec('H3').value).double()
        out, bound = R.head_ref(h3, torch.zeros_like(h3), fcw, fcb, R.C_POOL_FP32)
    else:
        # H3 is never stored: the average pool is fused into the last conv's epilogue.  Check that layer through the head.
        w, b = W(13)
        ref = layer_ref(13, dec('H2'), w, b, res=dec('H1'), ksplit=ksplit, out_fmt='fp32')
        out, bound = R.head_ref(ref.y, ref.bound(), fcw, fcb, R.C_POOL_TC)
    rows.append(_head_row(out, bound, six))
    return rows


def _check_image_fp8(dec, blob, scales, six):
    """The e4m3-written layers (the CAT writers and the six trunk layers) and the head of one image, plus the bf16 layers
    that feed them."""
    rows = []
    cat = dec('CAT').value
    for li in (0, 1, 2, 6):                         # the bf16 mode's layers, as they are
        L = R.LAYERS[li]
        w, b = R.layer_weights(blob, li)
        out = dec({0: 'P1A', 1: 'P1B'}.get(li, L.out)).value
        rows.append((L.name + ' (bf16)', R.gate(out, R.layer_ref(li, 'bf16', dec(L.inp), w, b))))
    for li, part, res in ((3, cat[:64], 'P1A'), (7, cat[64:], 'U')):
        w, b = R.layer_weights(blob, li)
        rows.append((R.LAYERS[li].name + ' -> CAT e4m3', R.gate(part, E.layer_ref(li, dec(R.LAYERS[li].inp), w, b, scales, res=dec(res)))))
    for li in range(8, 13):
        L = R.LAYERS[li]
        w, b = R.layer_weights(blob, li)
        ref = E.layer_ref(li, dec(L.inp), w, b, scales, res=dec(L.res) if L.res else None)
        rows.append((L.name, R.gate(dec(L.out).value, ref)))
    w, b = R.layer_weights(blob, 13)                # H3 is never stored: the last layer through the head
    ref = E.layer_ref(13, dec('H2'), w, b, scales, res=dec('H1'))
    fcw, fcb = R.fc_weights(blob)
    out, bound = R.head_ref(ref.y, ref.bound(), fcw, fcb, R.C_POOL_TC)
    rows.append(_head_row(out, bound, six))
    return rows


def report(label, per_image):
    """Per-layer table of the worst ratio of each gate over the sampled images; asserts every row passed."""
    names = [n for n, _ in per_image[0][1]]
    print('\n%s  (images %s)' % (label, [i for i, _ in per_image]))
    print('  %-34s %10s %10s' % ('layer', 'gate 1', 'gate 2'))
    failed = []
    for k, name in enumerate(names):
        gs = [rows[k][1] for _, rows in per_image]
        worst, rms = max(g.worst for g in gs), max(g.rms for g in gs)
        print('  %-34s %10.3g %10.3g%s' % (name, worst, rms, '' if all(g.ok for g in gs) else '   FAIL'))
        failed += ['%s image %d: %r at %s' % (name, i, rows[k][1], rows[k][1].where) for i, rows in per_image if not rows[k][1].ok]
    assert not failed, '\n'.join(failed)


def run_case(eng, prec, first, n, call, wids, blobs, label, seed=0):
    """Poison, run `call` (-> trans (n,3), rot (n,3), feature or None), check the untouched images, then every layer of
    the sampled ones.  wids: weight-set id per image of the call; blobs[id]: that set's fp32 weight blob.  'fp8': each image
    is decoded with eng.fp8_scales of its own set."""
    poison(eng, prec)
    trans, rot, feat = call()
    torch.cuda.synchronize()
    check_poison_outside(eng, prec, first, n)
    scales = {int(w): eng.fp8_scales(int(w)) if prec == 'fp8' else None for w in wids}
    six = torch.cat((trans, rot), 1).cpu().numpy()
    ks = trunk_ksplit(n, prec)
    if feat is not None:                           # the feature output is the F2 buffer through launch_nhwc_to_nchw, bit for bit
        nb = image_bytes('F2', prec)
        f2 = buffer_bytes(eng, 'F2')[first * nb:(first + n) * nb].cpu().numpy()
        fc = feat.cpu().numpy()
        for j in range(n):
            s = scales[int(wids[j])]
            assert np.array_equal(decode(f2[j * nb:(j + 1) * nb], 'F2', prec, s).value, fc[j]), 'feature %d != decoded F2' % j
    per_image = []
    for i in sample_images(first, n, seed, wids):
        cache = {}

        def raw(buf, i=i):
            nb = image_bytes(buf, prec)
            if buf not in cache:
                cache[buf] = buffer_bytes(eng, buf)[i * nb:(i + 1) * nb].cpu().numpy()
            return cache[buf]

        w = int(wids[i - first])
        per_image.append((i, check_image(raw, prec, blobs[w], ks, six[i - first], scales[w])))
    report('%s, %s, n = %d%s (ksplit %d)' % (label, prec, n, ', first = %d' % first if first else '', ks), per_image)


def track_inputs(synth, n, seed):
    """A raw-regime frame, n poses and their input A views: (rgb, depth, poses, rgbA, depthA) numpy arrays."""
    rgb, depth = synth.raw_frame(seed)
    poses = synth.raw_poses(n, seed=seed)
    rgbA, depthA = synth.rendered_views(n, poses, seed=seed)
    return rgb, depth, poses, rgbA, depthA


def distinct_fp8_scales(eng, calibrated):
    """Give every weight id of `calibrated` ({id < 256: its calibrated fp8 scales}) its own scale vector: the elementwise
    maximum of the calibrated ones, doubled on e4m3 tensor k where bit k of the id is set.  Calibration rounds each scale
    to a power of two, so sets of similar weights may share scales, and a kernel that read another image's set's scales
    would then pass.  The maximum keeps every set's headroom and a larger scale only coarsens the quantisation; the
    references read the engine's scales.  -> {id: the scales set}"""
    base = np.max(np.stack([np.asarray(s, np.float32) for s in calibrated.values()]), axis=0)
    out = {}
    for w in calibrated:
        out[w] = (base * 2.0 ** ((w >> np.arange(len(E.SCALE_NAMES))) & 1)).astype(np.float32)
        eng.set_fp8_scales(out[w], w)
    return out
