"""Weight-set switches inside the resident conv launches' per-CTA tile ranges, in every tensor-core precision.

64 tracks of one frame, track i on weight set (i // 3) % 2: the set changes every 3 images, so inside the contiguous tile range of
many CTAs (stems: 81 tiles per image, ~39 per CTA; 64-channel layers: 16 per image, ~8 per CTA), and the changes land on tiles
of either consumer warpgroup of the ping-pong schedule.  Each track's network output must equal, bit for bit, that of the same
64 tracks run with one weight set for all of them (the single-set launches, where no weights are reloaded).

In fp8 the two sets also get different activation scales (layer_harness.distinct_fp8_scales): the writers of CAT take the
scale of every tile's own set, so a set switch between two tiles of one CTA must switch the scale too."""
import numpy as np
import pytest
import torch

from layer_harness import distinct_fp8_scales

pytestmark = pytest.mark.gpu

TN, RN = 0.03, 5 * np.pi / 180
N = 64


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=N)
    mean, std = synth.default_mean_std()
    for wid in (0, 1):
        e.load_state_dict(synth.make_state_dict(wid), wid)
        e.set_stats(mean, std, wid)
    yield e
    e.close()


@pytest.mark.parametrize('prec', ['bf16x3', 'tf32', 'bf16', 'fp16', 'fp8'])
def test_weight_switch_inside_cta_ranges(synth, eng, prec):
    dev = eng.device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    rgb, depth = synth.raw_frame(3)
    poses = synth.raw_poses(N, seed=3)
    rgbA, depthA = synth.rendered_views(N, poses, seed=3)
    fr, fd, P, ow, A_, dA = t(rgb), t(depth), t(poses), t(np.full(N, 200.0)), t(rgbA), t(depthA)

    def run(wid):
        out_t = torch.empty(N, 3, dtype=torch.float32, device=dev); out_r = torch.empty_like(out_t)
        eng.track_batch(fr, fd, synth.CAMERA_K, P, ow, A_, dA, TN, RN, weight_ids_host=wid, precision=prec,
                        out_trans=out_t, out_rot=out_r)
        torch.cuda.synchronize()
        return torch.cat([out_t, out_r], 1).cpu().numpy()

    mixed_ids = (np.arange(N, dtype=np.int32) // 3) % 2
    if prec == 'fp8':
        eng.calibrate_fp8_tracks(fr, fd, synth.CAMERA_K, P, ow, A_, dA, weight_ids=mixed_ids)
        distinct_fp8_scales(eng, {w: eng.fp8_scales(w) for w in (0, 1)})
        assert not np.array_equal(eng.fp8_scales(0), eng.fp8_scales(1))
    mixed = run(mixed_ids)
    single = {w: run(np.full(N, w, dtype=np.int32)) for w in (0, 1)}
    assert not np.array_equal(single[0], single[1])      # the two sets give different outputs: a wrong set would show
    want = np.where(mixed_ids[:, None] == 0, single[0], single[1])
    bad = np.nonzero((mixed.view(np.uint32) != want.view(np.uint32)).any(1))[0]
    assert bad.size == 0, 'tracks %s differ from their one-set run' % bad.tolist()
