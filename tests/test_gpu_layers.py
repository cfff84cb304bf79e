"""Every conv layer checked ALONE on the H100: the layer's stored input (Engine.debug_buffer) decoded exactly, the same
operation run in fp64 on the CPU (oracle/layer_ref.py), and the layer's stored output compared element by element against
a bound derived from the mode's arithmetic -- in every precision mode and at the batch shapes the kernels split on.

Poisoning, the images checked and the per-layer tables `-s` prints: tests/layer_harness.py.
"""
import numpy as np
import pytest
import torch

from layer_harness import run_case, track_inputs

pytestmark = pytest.mark.gpu

TN, RN = 0.03, 5 * np.pi / 180


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
@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_track_batch_per_image_weights(synth, eng, blobs, prec):
    """A raw-regime frame (normalised magnitudes up to ~40), 37 tracks with weight ids alternating 0 / 1: per-image weight
    maps and biases (gbmaps / gbias) in the resident and trunk kernels; the reference uses each image's own set.  In bf16x3
    a second call with new poses replays the step's CUDA graph and must write the same buffers correctly."""
    n = 37
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 5)
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
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 8)
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    wid = np.array([0, 0, 1, 1, 1, 0], dtype=np.int32)

    def call():
        _, tr, ro = eng.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA),
                                    TN, RN, weight_ids_host=wid, precision='fp32')
        return tr, ro, None

    run_case(eng, 'fp32', 0, n, call, wid, blobs, 'track_batch, ids [0,0,1,1,1,0]', seed=3)
