"""Every conv layer checked ALONE on the H100: the layer's stored input (Engine.debug_buffer) decoded exactly, the same
operation run in fp64 on the CPU (oracle/layer_ref.py), and the layer's stored output compared element by element against
a bound derived from the mode's arithmetic -- in every precision mode and at the batch shapes the kernels split on.

Before each call every conv output buffer (P1A ... H2; also Y1A / Y1B and H3 in the fp32 mode) is filled with 0xFF bytes,
a NaN in every storage format, through the debug_buffer view into the Engine's own workspace.  After the call each checked
element must have been overwritten (NaN fails the gate) and every image outside [first, first + n) must still hold the
poison byte for byte.  The stem inputs X0A / X0B are never poisoned: their halo is the conv padding.

Each case checks the 14 layers plus the head on a sample of its images (first, last and two picked with a seed); `-s`
prints a per-layer table of the worst ratio of each gate (gate 1 elementwise worst case, gate 2 RMS; both pass at <= 1).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_ref as R

pytestmark = pytest.mark.gpu

TN, RN = 0.03, 5 * np.pi / 180
CONV_OUT = ['P1A', 'P1B', 'T1', 'T2', 'U', 'CAT', 'F1', 'T4', 'F2', 'H1', 'H2']
FP32_OUT = ['Y1A', 'Y1B', 'H3']


def _make_engine(pkg, synth, max_batch):
    e = pkg.Engine(max_batch=max_batch)
    e.load_state_dict(synth.make_state_dict(0), 0)
    e.load_state_dict(synth.make_state_dict(1), 1)
    mean, std = synth.default_mean_std()
    e.set_stats(mean, std, 0)
    e.set_stats(mean + 1.5, std * 1.25, 1)
    return e


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = _make_engine(pkg, synth, 64)
    yield e
    e.close()


@pytest.fixture(scope='module')
def blobs(pkg, synth):
    from importlib import import_module
    pack = import_module(pkg.__name__ + '.weights').pack_state_dict
    return {0: pack(synth.make_state_dict(0)), 1: pack(synth.make_state_dict(1))}


def _bytes(eng, buf):
    """The whole debug_buffer allocation of `buf` (max_batch images at 4 bytes per channel) as a uint8 view."""
    return eng.debug_buffer(R.BUF_ID[buf], eng.max_batch).view(torch.uint8).reshape(-1)


def _out_bufs(prec):
    return CONV_OUT + (FP32_OUT if prec == 'fp32' else [])


def poison(eng, prec):
    for buf in _out_bufs(prec):
        _bytes(eng, buf).fill_(0xFF)


def check_poison_outside(eng, prec, first, n):
    """Images outside [first, first + n) -- and, in the 2-byte bf16 mode, the allocation's unused second half -- still hold
    the poison, byte for byte."""
    bad = []
    for buf in _out_bufs(prec):
        nb = R.image_bytes(buf, R.buf_format(buf, prec))
        u = _bytes(eng, buf)
        for part in (u[:first * nb], u[(first + n) * nb:]):
            if part.numel() and not bool((part == 0xFF).all()):
                bad.append(buf)
    assert not bad, 'written outside images [%d, %d): %s' % (first, first + n, bad)


def sample_images(first, n, seed):
    if n <= 4:
        return list(range(first, first + n))
    rng = np.random.default_rng(seed)
    mid = rng.choice(np.arange(first + 1, first + n - 1), size=2, replace=False)
    return sorted({first, first + n - 1, *(int(i) for i in mid)})


def check_image(raw, prec, blob, ksplit, six):
    """All 14 layers and the head of one image.  raw(buf) -> that image's bytes of buffer buf; blob: the image's fp32
    weight blob; six: the (6,) trans ++ rot the call returned for it.  -> [(layer name, GateResult)]."""
    D = {}

    def dec(buf):
        if buf not in D:
            D[buf] = R.decode(raw(buf), buf, R.buf_format(buf, prec))
        return D[buf]

    W = lambda li: R.layer_weights(blob, li)
    rows = []

    def one(li, out_value, res=None, **kw):
        L = R.LAYERS[li]
        w, b = W(li)
        ref = R.layer_ref(li, prec, dec(L.inp), w, b, res=dec(res) if res else None, ksplit=ksplit, **kw)
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
    _, r5 = R.chained_ref(4, prec, dec('P1B'), w4, b4, w5, b5, res2=dec('P1B'), ksplit=ksplit)
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
        ref = R.layer_ref(13, prec, dec('H2'), w, b, res=dec('H1'), ksplit=ksplit, out_fmt='fp32')
        out, bound = R.head_ref(ref.y, ref.bound(), fcw, fcb, R.C_POOL_TC)
    d = torch.as_tensor(np.asarray(six, dtype=np.float64))
    finite = bool(torch.isfinite(d).all())
    rows.append(('head (trans, rot)', R.GateResult(float(((d - out).abs() / bound).max()) if finite else np.inf, 0.0, finite, 6)))
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
    the sampled ones.  wids: weight-set id per image of the call."""
    poison(eng, prec)
    trans, rot, feat = call()
    torch.cuda.synchronize()
    check_poison_outside(eng, prec, first, n)
    six = torch.cat((trans, rot), 1).cpu().numpy()
    ks = R.trunk_ksplit(n, prec)
    if feat is not None:                           # the feature output is the F2 buffer through launch_nhwc_to_nchw, bit for bit
        nb = R.image_bytes('F2', prec)
        f2 = _bytes(eng, 'F2')[first * nb:(first + n) * nb].cpu().numpy()
        fc = feat.cpu().numpy()
        for j in range(n):
            assert np.array_equal(R.decode(f2[j * nb:(j + 1) * nb], 'F2', prec).value, fc[j]), 'feature %d != decoded F2' % j
    per_image = []
    for i in sample_images(first, n, seed):
        cache = {}

        def raw(buf, i=i):
            nb = R.image_bytes(buf, R.buf_format(buf, prec))
            if buf not in cache:
                cache[buf] = _bytes(eng, buf)[i * nb:(i + 1) * nb].cpu().numpy()
            return cache[buf]

        per_image.append((i, check_image(raw, prec, blobs[int(wids[i - first])], ks, six[i - first])))
    report('%s, %s, n = %d%s (ksplit %d)' % (label, prec, n, ', first = %d' % first if first else '', ks), per_image)


# ------------------------------------------------------------------------------------------- Engine.forward
FORWARD = [(p, n) for n in (1, 3, 4, 5, 13, 64) for p in ('bf16x3', 'tf32', 'bf16')] + [('fp32', 1), ('fp32', 3)]


@pytest.mark.parametrize('prec,n', FORWARD, ids=['%s-n%d' % c for c in FORWARD])
def test_forward_layers(synth, eng, blobs, prec, n):
    """Tensor-regime pairs.  n <= 4: the trunk's split-K latency mode (ksplit 4, 2 in bf16); 5, 13: throughput mode with
    ragged unit counts per CTA (a ping-pong warpgroup idles on the last unit); 64: the full batch.  fp32: the FFMA path,
    where Y1A / Y1B and H3 are stored and checked directly."""
    A, B = synth.tensor_pairs(n, seed=40 + n)
    Ad, Bd = A.to(eng.device), B.to(eng.device)
    run_case(eng, prec, 0, n, lambda: eng.forward(Ad, Bd, weight_id=0, precision=prec, want_feature=True),
             [0] * n, blobs, 'forward', seed=n)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_forward_many_waves(pkg, synth, blobs, prec):
    """250 images on a 256-image engine: many waves of work units; images 250-255 stay poisoned."""
    e = _make_engine(pkg, synth, 256)
    try:
        A, B = synth.tensor_pairs(250, seed=7)
        Ad, Bd = A.to(e.device), B.to(e.device)
        run_case(e, prec, 0, 250, lambda: e.forward(Ad, Bd, weight_id=0, precision=prec), [0] * 250, blobs, 'forward (max_batch 256)')
    finally:
        e.close()


@pytest.mark.parametrize('prec', ['bf16x3', 'tf32'])
def test_forward_preprocessed_offset(synth, eng, blobs, prec):
    """normalize() fills 8 images, forward_preprocessed(3, first=5) runs images 5-7: img_first in both conv kernels and the
    head's pool_part + first.  Images 0-4 (and 8 on) stay poisoned."""
    rng = np.random.default_rng(11)
    poses = synth.raw_poses(8, seed=11)
    rgbA, depthA = synth.rendered_views(8, poses, seed=11)
    rgbB, depthB = synth.rendered_views(8, poses, seed=12)
    rgbB = np.where(rgbB == 0, rng.integers(0, 256, size=rgbB.shape), rgbB).astype(np.uint8)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    def call():                                    # normalize writes only X0A / X0B, so the poison of images 0-4 stays
        eng.normalize(t(rgbA), t(depthA), t(rgbB), t(depthB), t(poses), precision=prec, want_tensors=False)
        return eng.forward_preprocessed(3, weight_id=0, first=5, precision=prec)

    run_case(eng, prec, 5, 3, call, [0] * 3, blobs, 'forward_preprocessed')


# ------------------------------------------------------------------------------------------- track_batch
def _track_inputs(synth, n, seed):
    rgb, depth = synth.raw_frame(seed)
    poses = synth.raw_poses(n, seed=seed)
    rgbA, depthA = synth.rendered_views(n, poses, seed=seed)
    return rgb, depth, poses, rgbA, depthA


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_track_batch_per_image_weights(synth, eng, blobs, prec):
    """A raw-regime frame (normalised magnitudes up to ~40), 37 tracks with weight ids alternating 0 / 1: per-image weight
    maps and biases (gbmaps / gbias) in the resident and trunk kernels; the reference uses each image's own set.  In bf16x3
    a second call with new poses replays the step's CUDA graph and must write the same buffers correctly."""
    n = 37
    rgb, depth, poses, rgbA, depthA = _track_inputs(synth, n, 5)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    wid = np.arange(n, dtype=np.int32) % 2
    wdev, P, ow = t(wid), t(poses), t(np.full(n, 200.0))
    fr, fd, A_, dA = t(rgb), t(depth), t(rgbA), t(depthA)
    out_p = torch.empty_like(P)
    out_t = torch.empty(n, 3, dtype=torch.float32, device=dev); out_r = torch.empty_like(out_t)

    def call():
        eng.track_batch(fr, fd, synth.CAMERA_K, P, ow, A_, dA, TN, RN, weight_ids_host=wid, weight_ids_dev=wdev,
                        precision=prec, out_poses=out_p, out_trans=out_t, out_rot=out_r)
        return out_t, out_r, None

    run_case(eng, prec, 0, n, call, wid, blobs, 'track_batch, ids 0/1', seed=1)
    if prec == 'bf16x3':
        P.copy_(t(synth.raw_poses(n, seed=6)))     # same addresses: the second call replays the captured graph
        run_case(eng, prec, 0, n, call, wid, blobs, 'track_batch graph replay, new poses', seed=2)
        assert eng.last_step_was_graph()


def test_track_batch_fp32_runs(synth, eng, blobs):
    """fp32: one FFMA forward per run of equal ids ([0, 0], [1, 1, 1], [0]): the direct path at nonzero `first`."""
    n = 6
    rgb, depth, poses, rgbA, depthA = _track_inputs(synth, n, 8)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    wid = np.array([0, 0, 1, 1, 1, 0], dtype=np.int32)

    def call():
        _, tr, ro = eng.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA),
                                    TN, RN, weight_ids_host=wid, precision='fp32')
        return tr, ro, None

    run_case(eng, 'fp32', 0, n, call, wid, blobs, 'track_batch, ids [0,0,1,1,1,0]', seed=3)
