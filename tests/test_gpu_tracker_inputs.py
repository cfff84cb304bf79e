"""Tracker.on_track_batch takes its inputs as numpy arrays, pageable or pinned CPU tensors, CUDA tensors or any mix of them.
Every mix gives the poses of the all-CUDA call bit for bit, with input A passed in or drawn inside the step, in bf16x3 and in
fp8 (where every call calibrates its weight sets on its own inputs).  Host inputs are staged through two fixed slots, so the
step of a mixed call sees at most two sets of device pointers, and a pageable input may be overwritten once the call returns."""
import importlib
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
N = 3
WIDTHS = np.array([200.0, 180.0, 150.0])
IDS = np.array([0, 1, 0], dtype=np.int32)
# (frame kind, poses kind); input A, when passed, is of the frame's kind.  The first is the reference.
KINDS = (('cuda', 'cuda'), ('numpy', 'numpy'), ('cpu', 'cpu'), ('pinned', 'pinned'), ('cuda', 'numpy'), ('cuda', 'cpu'),
         ('numpy', 'cuda'))
MIXED = KINDS[2:]                                      # device route with host inputs
VARIANTS = ((None, None), ('numpy', 'tensor'), ('tensor', 'numpy'))    # (object widths, weight ids)


@pytest.fixture(scope='module')
def setup(pkg, synth, tmp_path_factory):
    """A Tracker with the CUDA rasteriser and two weight sets with their meshes, and one synthetic frame of N tracks."""
    mio = importlib.import_module(pkg.__name__ + '.mesh_io')
    path = str(tmp_path_factory.mktemp('mesh') / 'model.ply')
    mio.save_ply_mesh(path, synth.mesh(2, seed=4))
    K = synth.CAMERA_K
    info = {'resolution': 176, 'object_width': 200.0, 'boundingbox': 10,
            'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2], 'centerY': K[1, 2], 'height': 480, 'width': 640}}
    mean, std = synth.default_mean_std()
    sds = [synth.make_state_dict(w) for w in (0, 1)]
    trk = pkg.Tracker(info, mean, std, {'state_dict': sds[0]}, model_path=path, max_batch=8)
    eng = trk.engine
    eng.load_state_dict(sds[1], 1)
    eng.set_stats(mean + 1.5, std * 1.25, 1)
    eng.set_mesh(synth.mesh(1, seed=1), 1)
    rgb, depth = synth.raw_frame(31)
    poses = synth.raw_poses(N, seed=31)
    poses[0, :3, 3] = (0.32, -0.2, 0.5)                           # the first window hangs over the frame's edge
    rgbA, depthA = synth.rendered_views(N, poses, seed=31)
    try:
        yield trk, sds, dict(rgb=rgb, depth=depth, poses=poses, rgbA=rgbA, depthA=depthA)
    finally:
        eng.close()
        importlib.import_module(pkg.__name__ + '.Utils').set_engine(None)   # the Tracker made this engine Utils' own


def _as(a, kind, dev):
    if kind == 'numpy':
        return np.array(a)
    t = torch.from_numpy(np.array(a))
    return t.to(dev) if kind == 'cuda' else t.pin_memory() if kind == 'pinned' else t


def _inputs(trk, d, kinds, drawn, widths, ids):
    """on_track_batch's arguments: the frame, input A and poses of `kinds`; widths and ids None, numpy or a CPU tensor (the
    reference passes CUDA tensors)."""
    dev = trk.engine.device
    fk, pk = kinds

    def extra(v, kind):
        if kind is None:
            return None
        return _as(v, 'cuda' if kinds == KINDS[0] else 'cpu' if kind == 'tensor' else 'numpy', dev)
    A = (None, None) if drawn else (_as(d['rgbA'], fk, dev), _as(d['depthA'], fk, dev))
    return ((_as(d['poses'], pk, dev), _as(d['rgb'], fk, dev), _as(d['depth'], fk, dev)) + A,
            dict(object_width=extra(WIDTHS, widths), weight_ids=extra(IDS, ids)))


@pytest.mark.parametrize('precision', ['bf16x3', 'fp8'])
@pytest.mark.parametrize('drawn', [False, True])
def test_every_input_kind_gives_the_all_cuda_poses(setup, precision, drawn):
    trk, sds, d = setup
    eng = trk.engine
    trk.precision = precision
    try:
        for widths, ids in VARIANTS:
            sets = (0, 1) if ids is not None else (0,)
            want = scales = None
            for kinds in KINDS:
                if precision == 'fp8':                        # a reload drops the scales: this call calibrates on its own inputs
                    for w in sets:
                        eng.load_state_dict(sds[w], w)
                args, kw = _inputs(trk, d, kinds, drawn, widths, ids)
                got = trk.on_track_batch(*args, **kw)
                if kinds[1] == 'numpy':
                    assert isinstance(got, np.ndarray) and got.dtype == np.float64 and got.shape == (N, 4, 4)
                else:
                    assert torch.is_tensor(got) and got.is_cuda and got.dtype == torch.float64
                    got = got.cpu().numpy()
                case = (kinds, widths, ids)
                if want is None:
                    want = got
                    assert np.isfinite(want).all()
                    if precision == 'fp8':
                        scales = [eng.fp8_scales(w) for w in sets]
                        assert all(s is not None for s in scales)
                assert np.array_equal(got, want), case
                if precision == 'fp8':
                    assert all(np.array_equal(eng.fp8_scales(w), s) for w, s in zip(sets, scales)), case
    finally:
        trk.precision = 'bf16x3'


@pytest.mark.parametrize('drawn', [False, True])
def test_mixed_calls_step_on_two_pointer_sets(pkg, setup, monkeypatch, drawn):
    """Six calls with the same inputs reach the step with at most two sets of input pointers (one per staging slot), while the
    caller keeps every result and allocates between calls: the step's CUDA graph is found again instead of captured anew."""
    trk, _, d = setup
    seen = []

    def record(fn):
        def wrap(self, *a, **k):
            seen.append(tuple(x.data_ptr() for x in (*a, k.get('weight_ids_dev')) if torch.is_tensor(x)))
            return fn(self, *a, **k)
        return wrap
    for name in ('track_batch', 'track_render'):
        monkeypatch.setattr(pkg.Engine, name, record(getattr(pkg.Engine, name)))
    keep = []
    for kinds in MIXED:
        for widths, ids in VARIANTS:
            args, kw = _inputs(trk, d, kinds, drawn, widths, ids)
            seen.clear()
            for _ in range(6):
                keep.append((trk.on_track_batch(*args, **kw), torch.empty(64, device=trk.engine.device)))
            assert len(seen) == 6 and len(set(seen)) <= 2, (kinds, widths, ids, len(set(seen)))
    torch.cuda.synchronize()


def test_pageable_inputs_can_be_overwritten_at_once(setup):
    """A numpy array or a pageable CPU tensor has been read when the call returns: overwriting it then, while the device is
    still busy with earlier work, does not change the result."""
    trk, _, d = setup
    dev = trk.engine.device
    P = torch.from_numpy(d['poses']).to(dev)
    names = ('rgb', 'depth', 'rgbA', 'depthA')
    want = trk.on_track_batch(P, *(_as(d[k], 'cuda', dev) for k in names), object_width=_as(WIDTHS, 'cuda', dev)).cpu().numpy()
    outs = []
    for k in range(6):
        torch.cuda._sleep(20_000_000)                          # the copies of this call queue behind device work
        ins = [_as(d[x], 'numpy' if k % 2 == 0 else 'cpu', dev) for x in names] + [np.array(WIDTHS)]
        outs.append(trk.on_track_batch(P, *ins[:4], object_width=ins[4]))
        for a in ins:
            a[...] = 7
    torch.cuda.synchronize()
    for k, out in enumerate(outs):
        assert np.array_equal(out.cpu().numpy(), want), k
