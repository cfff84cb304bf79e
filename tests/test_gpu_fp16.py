"""The 'fp16' mode on the H100: every conv layer checked ALONE against an fp64 conv of its own stored input
(oracle/fp16_ref.py), the latency mode's independence of n and of the other tracks' sets, the end-to-end 6-vector against
the fp32 reference, saturation, and the refusal of a weight set outside fp16's range.

The per-layer check (poisoning, image sampling, the tables `-s` prints) is tests/layer_harness.py's in the fp16 formats:
2 bytes per channel, so an image stride half of the 4-byte modes'.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import fp16_ref as H
import layer_ref as R
import se3_oracle as O
from layer_harness import CONV_OUT, buffer_bytes, check_poison_outside, poison, run_case, track_inputs

pytestmark = pytest.mark.gpu

TN, RN = 0.03, 5 * np.pi / 180
RTOL, ATOL = 1e-3, 1e-4                               # the fp32 gate, as tf32 meets it


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


def _t(eng):
    return lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


# ------------------------------------------------------------------------------------------- layers
@pytest.mark.parametrize('n', [1, 3, 4, 5, 13, 64])
def test_fp16_forward_layers(synth, eng, blobs, n):
    """Tensor-regime pairs.  n <= 4: the trunk's split-K latency mode (ksplit 2, as bf16); 5, 13: ragged unit counts per
    CTA; 64: the full batch."""
    A, B = synth.tensor_pairs(n, seed=40 + n)
    Ad, Bd = A.to(eng.device), B.to(eng.device)
    run_case(eng, 'fp16', 0, n, lambda: eng.forward(Ad, Bd, weight_id=0, precision='fp16', want_feature=True), [0] * n, blobs, 'forward', seed=n)


def test_fp16_forward_many_waves(pkg, synth, blobs):
    """250 images on a 256-image engine; images 250-255 stay poisoned."""
    e = _make_engine(pkg, synth, 256)
    try:
        A, B = synth.tensor_pairs(250, seed=7)
        Ad, Bd = A.to(e.device), B.to(e.device)
        run_case(e, 'fp16', 0, 250, lambda: e.forward(Ad, Bd, weight_id=0, precision='fp16'), [0] * 250, blobs, 'forward (max_batch 256)')
    finally:
        e.close()


def test_fp16_forward_preprocessed_offset(synth, eng, blobs):
    """normalize() fills 8 images, forward_preprocessed(3, first=5) runs images 5-7; images 0-4 and 8 on stay poisoned."""
    rng = np.random.default_rng(11)
    poses = synth.raw_poses(8, seed=11)
    rgbA, depthA = synth.rendered_views(8, poses, seed=11)
    rgbB, depthB = synth.rendered_views(8, poses, seed=12)
    rgbB = np.where(rgbB == 0, rng.integers(0, 256, size=rgbB.shape), rgbB).astype(np.uint8)
    t = _t(eng)

    def call():
        eng.normalize(t(rgbA), t(depthA), t(rgbB), t(depthB), t(poses), precision='fp16', want_tensors=False)
        return eng.forward_preprocessed(3, weight_id=0, first=5, precision='fp16')

    run_case(eng, 'fp16', 5, 3, call, [0] * 3, blobs, 'forward_preprocessed')


def test_fp16_track_batch_per_image_weights(synth, eng, blobs):
    """A raw-regime frame, 37 tracks with weight ids 0 / 1 in one step; a second call with new poses replays its graph."""
    n = 37
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 5)
    t = _t(eng)
    wid = np.arange(n, dtype=np.int32) % 2
    wdev, P, ow = t(wid), t(poses), t(np.full(n, 200.0))
    fr, fd, A_, dA = t(rgb), t(depth), t(rgbA), t(depthA)
    out_p = torch.empty_like(P)
    out_t = torch.empty(n, 3, dtype=torch.float32, device=eng.device); out_r = torch.empty_like(out_t)

    def call():
        eng.track_batch(fr, fd, synth.CAMERA_K, P, ow, A_, dA, TN, RN, weight_ids_host=wid, weight_ids_dev=wdev,
                        precision='fp16', out_poses=out_p, out_trans=out_t, out_rot=out_r)
        return out_t, out_r, None

    run_case(eng, 'fp16', 0, n, call, wid, blobs, 'track_batch, ids 0/1', seed=1)
    P.copy_(t(synth.raw_poses(n, seed=6)))            # same addresses: the second call replays the captured graph
    run_case(eng, 'fp16', 0, n, call, wid, blobs, 'track_batch graph replay, new poses', seed=2)
    assert eng.last_step_was_graph()


def test_fp16_latency_mode_independent_of_n_and_other_sets(synth, eng):
    """n <= 4 (split-K): a track's pose is the same bits alone, among 4 tracks, and whatever sets the other tracks use."""
    n = 4
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 8)
    t = _t(eng)
    args = lambda s: (t(rgb), t(depth), synth.CAMERA_K, t(poses[s]), t(np.full(len(poses[s]), 200.0)), t(rgbA[s]), t(depthA[s]), TN, RN)
    mixed = np.array([0, 1, 1, 0], np.int32)
    out_m, _, _ = eng.track_batch(*args(slice(0, n)), weight_ids_host=mixed, weight_ids_dev=t(mixed), precision='fp16')
    for w in (0, 1):
        out_w, _, _ = eng.track_batch(*args(slice(0, n)), weight_ids_host=np.full(n, w, np.int32), precision='fp16')
        for i in np.flatnonzero(mixed == w):
            one, _, _ = eng.track_batch(*args(slice(i, i + 1)), weight_ids_host=np.array([w], np.int32), precision='fp16')
            assert torch.equal(one[0], out_m[i]) and torch.equal(one[0], out_w[i]), 'track %d' % i


# ------------------------------------------------------------------------------------------- end to end
def test_fp16_config1_against_reference(synth, golden_dir, eng):
    """BASELINE config 1 (the shipped pair, batch 1) against the reference's own forward (golden), at the fp32 gate."""
    import cv2
    g = np.load(os.path.join(golden_dir, 'golden_model.npz'))
    rgbA = cv2.imread(os.path.join(golden_dir, 'c1_rgbA.png'))[..., ::-1].copy()
    rgbB = cv2.imread(os.path.join(golden_dir, 'c1_rgbB.png'))[..., ::-1].copy()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)[None]).to(eng.device)
    tA, tB = eng.normalize(t(rgbA), t(synth.depth_from_rgb(rgbA)), t(rgbB), t(synth.depth_from_rgb(rgbB)), t(synth.config1_pose()),
                           precision='fp16')
    tr, ro, _ = eng.forward(tA, tB, weight_id=0, precision='fp16')
    ref = np.concatenate([g['c1_trans'], g['c1_rot']], 1)
    out = torch.cat((tr, ro), 1).double().cpu().numpy()
    err = np.abs(out - ref)
    print('\nconfig 1, fp16: max |err| %.4g, max err/tol %.3f' % (err.max(), (err / (ATOL + RTOL * np.abs(ref))).max()))
    assert np.isfinite(out).all() and (err <= ATOL + RTOL * np.abs(ref)).all()


@pytest.mark.parametrize('n', [1, 2, 3, 7, 64])
def test_fp16_tensor_regime_against_reference(synth, eng, n):
    sd = synth.make_state_dict(0)
    A, B = synth.tensor_pairs(n, seed=10 + n)
    ref = O.forward(sd, A, B)
    ref6 = torch.cat((ref['trans'], ref['rot']), 1).double()
    tr, ro, _ = eng.forward(A.to(eng.device), B.to(eng.device), precision='fp16')
    out = torch.cat((tr, ro), 1).double().cpu()
    err = (out - ref6).abs() / (ATOL + RTOL * ref6.abs())
    print('\ntensor regime n = %d, fp16: max err/tol %.3f' % (n, err.max().item()))
    assert torch.isfinite(out).all() and (err <= 1).all()


# The 6-vector's worst |error| against the fp32 reference in a CPU emulation of this exact arithmetic (scripts/precision_raw.py
# --fp16: bf16x3 stems, fp16 operands and activations, fp32 sums) on the raw-regime case below.  The gates are 2x these, the way
# the bf16 mode's gate was set.  (Weight seed 1 exceeds the fp32 gate there, as tf32 does: 3.6x in the emulation.)
EMU_WORST = {'raw set 0': 1.553e-4, 'raw set 1': 9.653e-4}


def test_fp16_raw_regime_batch64_against_reference(synth, eng):
    """The parity tests' raw-regime frame, 64 tracks, weight seeds 0 / 1 on 32 each in one step."""
    n = 64
    rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 11)
    t = _t(eng)
    wid = np.repeat(np.array([0, 1], dtype=np.int32), n // 2)
    _, tr, ro = eng.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA), TN, RN,
                                weight_ids_host=wid, weight_ids_dev=t(wid), precision='fp16')
    out = torch.cat((tr, ro), 1).double().cpu().numpy()
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    sds = {0: synth.make_state_dict(0), 1: synth.make_state_dict(1)}
    ref = np.stack([np.concatenate([d['trans'], d['rot']]) for _, d in
                    (O.on_track(sds[int(wid[i])], poses[i], rgb, depth, rgbA[i], depthA[i], synth.CAMERA_K, 200.0,
                                *stats[int(wid[i])], return_all=True) for i in range(n))])
    assert np.isfinite(out).all()
    for w in (0, 1):
        err = float(np.abs(out[wid == w] - ref[wid == w]).max())
        e = EMU_WORST['raw set %d' % w]
        print('\nraw regime n = 64, set %d, fp16: max |err| %.4g (emulation %.4g, gate %.4g)' % (w, err, e, 2 * e))
        assert err <= 2 * e


def test_fp16_eval_pairs_loss_against_reference_loop(pkg, synth, tmp_path):
    """se3tn_eval_pairs in fp16 against Problem.validate's loop on the CPU (oracle forward, nn.MSELoss): the 6-vectors at the
    fp32 gate, and the loss within what those 6-vectors' deviation allows."""
    import glob
    from test_gpu_validate import MEAN_ROUNDING, TN as VTN, RN as VRN, _load_batch, loss_bound, oracle_validate, write_folder
    e = _make_engine(pkg, synth, 8)
    try:
        e.set_mesh(synth.mesh(), 0)
        write_folder(e, synth, str(tmp_path), 8, seed=1)
        files = sorted(glob.glob(str(tmp_path / '*rgbA.png')))
        mean, std = synth.default_mean_std()
        tl_ref, rl_ref, pred_ref, lab = oracle_validate(synth.make_state_dict(0), files, mean, std, 8)
        rgbA, depthA, rgbB, depthB, A, B, _ = _load_batch(e, files)
        tr, ro, sums, _, _ = e.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, VTN, VRN, precision='fp16', want_terms=True)
        six = np.concatenate((tr.cpu().numpy(), ro.cpu().numpy()), 1).astype(np.float64)
        assert (np.abs(six - pred_ref) <= ATOL + RTOL * np.abs(pred_ref)).all()
        loss = sums.cpu().numpy().astype(np.float64) / (len(files) * 3)
        ref = np.array([tl_ref, rl_ref])
        moved = loss_bound(pred_ref, lab, 8, np.abs(six - pred_ref))
        print('\neval_pairs fp16 loss: trans %.6g (ref %.6g), rot %.6g (ref %.6g); relative difference %.2e, %.2e'
              % (loss[0], ref[0], loss[1], ref[1], *(np.abs(loss - ref) / ref)))
        assert (np.abs(loss - ref) <= moved + MEAN_ROUNDING * ref).all()
    finally:
        e.close()


# ------------------------------------------------------------------------------------------- saturation and range
def test_fp16_stem_saturates(synth, eng, blobs):
    """Inputs scaled so the stems' fp64 outputs exceed 65504: the stored pooled outputs hold +-65504 there (the reference
    saturates), no stored activation is inf or NaN, and the 6-vector is finite."""
    n = 2
    A, B = synth.tensor_pairs(n, seed=31)
    poison(eng, 'fp16')
    tr, ro, _ = eng.forward(A.to(eng.device) * 3e4, B.to(eng.device) * 3e4, weight_id=0, precision='fp16')
    torch.cuda.synchronize()
    assert bool(torch.isfinite(tr).all()) and bool(torch.isfinite(ro).all())
    for buf in CONV_OUT:
        u = buffer_bytes(eng, buf)[:n * H.image_bytes(buf)].view(torch.int16)
        assert not bool(((u & 0x7C00) == 0x7C00).any()), 'inf or NaN stored in ' + buf
    saturated = 0
    for li, inp, out in ((0, 'X0A', 'P1A'), (1, 'X0B', 'P1B')):
        w, b = R.layer_weights(blobs[0], li)
        for j in range(n):
            x = H.decode(buffer_bytes(eng, inp)[j * H.image_bytes(inp):(j + 1) * H.image_bytes(inp)].cpu().numpy(), inp)
            y = H.decode(buffer_bytes(eng, out)[j * H.image_bytes(out):(j + 1) * H.image_bytes(out)].cpu().numpy(), out).value
            ref = H.layer_ref(li, x, w, b)
            g = R.gate(y, ref)
            assert g.ok, '%s image %d: %r' % (R.LAYERS[li].name, j, g)
            saturated += int((np.abs(y) == H.F16_MAX).sum())
    assert saturated > 0


def test_fp16_refuses_weights_outside_its_range(pkg, synth):
    """A set with one conv weight of 1e5 loads; an fp16 step on it fails with SE3TN_ERR_STATE naming the id and launches
    nothing, while bf16x3 on the same set and fp16 on the other sets run."""
    L = pkg._lib
    from importlib import import_module
    pack = import_module(pkg.__name__ + '.weights').pack_state_dict
    e = _make_engine(pkg, synth, 8)
    try:
        blob = np.ascontiguousarray(pack(synth.make_state_dict(0)), dtype=np.float32)
        w_off, _, _ = R.blob_offsets()
        blob[w_off[9] + 1234] = 1e5                    # convAB2.conv1
        L.check(e.lib.se3tn_load_weights(e._ctx, 2, blob.ctypes.data_as(ctypes.c_void_p), blob.size), e._ctx)
        mean, std = synth.default_mean_std()
        e.set_stats(mean, std, 2)
        n = 3
        A, B = synth.tensor_pairs(n, seed=9)
        Ad, Bd = A.to(e.device), B.to(e.device)
        poison(e, 'fp16')
        torch.cuda.synchronize()
        with pytest.raises(L.Se3tnError) as ex:
            e.forward(Ad, Bd, weight_id=2, precision='fp16')
        assert ex.value.code == L.ERR_STATE and 'weight set 2' in str(ex.value)
        rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, 4)
        t = _t(e)
        wid = np.array([0, 2, 1], np.int32)
        with pytest.raises(L.Se3tnError) as ex:
            e.track_batch(t(rgb), t(depth), synth.CAMERA_K, t(poses), t(np.full(n, 200.0)), t(rgbA), t(depthA), TN, RN,
                          weight_ids_host=wid, weight_ids_dev=t(wid), precision='fp16')
        assert ex.value.code == L.ERR_STATE and 'weight set 2' in str(ex.value)
        torch.cuda.synchronize()
        check_poison_outside(e, 'fp16', 0, 0)          # nothing was launched
        tr, ro, _ = e.forward(Ad, Bd, weight_id=2, precision='bf16x3')
        assert bool(torch.isfinite(tr).all()) and bool(torch.isfinite(ro).all())
        tr, ro, _ = e.forward(Ad, Bd, weight_id=1, precision='fp16')
        assert bool(torch.isfinite(tr).all())
        # reloading the set with weights in range lifts the refusal
        e.load_state_dict(synth.make_state_dict(0), 2)
        e.forward(Ad, Bd, weight_id=2, precision='fp16')
    finally:
        e.close()
