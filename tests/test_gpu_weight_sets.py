"""Steps whose tracks use different weight sets, loaded as the one-pass drivers load them: one set per class under weight id =
class id (1..21 here), none at 0.  The device tables the mixed launches index (per-set weight maps, bias and fc pointers,
statistics) then have max_id + 1 rows, with empty rows below the first id.

  * every layer of mixed steps against fp64 (tests/layer_harness.py), in the trunk's split-K latency mode (n <= 4: every
    unit's K loop cut into kSplitK pieces, 2 in bf16 and fp16, by different CTAs; fp8 does not split) and in its throughput
    mode, in bf16x3, tf32, bf16, fp16 and fp8.  In fp8 every id has scales of its own (layer_harness.distinct_fp8_scales),
    so a launch that read another image's set's scale block would fail the gate;
  * bit identities on every track: within latency mode a track's results do not depend on n or on the sets of the other
    tracks, so each track of a mixed step equals that track run alone on the single-set path; a mixed throughput step equals
    the single-set launches of the same tracks; eval_pairs likewise, pair by pair;
  * K0 with sparse ids: each track normalised with its own id's statistics, bit for bit, in fp32 and in fp64;
  * reloads: a set added after steps were captured (the tables grow), a set replaced under its id, new statistics and, in
    fp8, new scales all reach the next step, and leave every other track as it was;
  * the state rules of fp16 (a set outside its range) and fp8 (a set without scales) with sparse ids.
"""
import ctypes
import importlib
import numpy as np
import pytest
import torch

import layer_ref as R
import se3_oracle as O
from layer_harness import (check_poison_outside, decode, distinct_fp8_scales, image_bytes, poison, run_case,
                           track_inputs)

pytestmark = pytest.mark.gpu

TN, RN = 0.03, 5 * np.pi / 180
IDS = tuple(range(1, 22))
PRECS = ('bf16x3', 'tf32', 'bf16', 'fp16', 'fp8')
# latency mode: repeated and unsorted ids, the repeat not adjacent
LATENCY = {2: [17, 3], 3: [5, 21, 1], 4: [9, 2, 14, 9]}
SHUFFLED = [int(i) for i in np.random.default_rng(21).permutation(IDS)]
# throughput mode: ragged unit counts (n = 5), every set once in a shuffled order (21), ids drawn with repeats (64)
THROUGHPUT = [(p, ids) for ids in ([20, 4, 4, 13, 1], SHUFFLED, [int(i) for i in np.random.default_rng(64).choice(IDS, 64)])
              for p in PRECS]


def stats(synth, wid, dtype=np.float32):
    """Statistics of weight id `wid`: distinct for every id, in the given dtype."""
    mean, std = synth.default_mean_std()
    return mean.astype(dtype) + dtype(0.05 * wid), std.astype(dtype) * dtype(1 + 0.01 * wid)


def load(e, synth, wid, seed=None, dtype=np.float32):
    e.load_state_dict(synth.make_state_dict(wid if seed is None else seed), wid)
    e.set_stats(*stats(synth, wid, dtype), wid)


class Blobs(dict):
    """weight id -> the fp32 blob of synth.make_state_dict(seed), packed when first asked for (a blob is 54 MB)."""

    def __init__(self, pkg, synth, seeds=None):
        super().__init__()
        self.pack = importlib.import_module(pkg.__name__ + '.weights').pack_state_dict
        self.synth, self.seeds = synth, seeds or {}

    def __missing__(self, wid):
        blob = self[wid] = self.pack(self.synth.make_state_dict(self.seeds.get(wid, wid)))
        return blob


def assert_distinct_fp8_scales(e, ids, prec):
    """fp8: the premise of a mixed step's checks, that no two of its ids share scales."""
    if prec != 'fp8':
        return
    u = sorted(set(int(w) for w in ids))
    assert len({e.fp8_scales(w).tobytes() for w in u}) == len(u), 'ids %s share fp8 scales' % u


@pytest.fixture(scope='module')
def eng(pkg, synth):
    """Sets 1..21, each calibrated for fp8 on its own tracks of one frame, then given scales of its own."""
    e = pkg.Engine(max_batch=64)
    for w in IDS:
        load(e, synth, w)
    distinct_fp8_scales(e, Tracks(e, synth, 2 * len(IDS), seed=2).calibrate(e, list(IDS) * 2))
    assert_distinct_fp8_scales(e, IDS, 'fp8')
    yield e
    e.close()


@pytest.fixture(scope='module')
def blobs(pkg, synth):
    return Blobs(pkg, synth)


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


class Tracks:
    """n tracks of one raw-regime frame (layer_harness.track_inputs) on the device.  run(e, ids, prec, j0) is one track_batch
    of tracks j0 .. j0 + len(ids) - 1 with those weight ids on engine e -> numpy (trans, rot, updated poses)."""

    def __init__(self, e, synth, n, seed):
        rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, seed)
        self.K = synth.CAMERA_K
        self.frame, self.poses = (_dev(e, rgb), _dev(e, depth)), _dev(e, poses)
        self.width, self.A = _dev(e, np.full(n, 200.0)), (_dev(e, rgbA), _dev(e, depthA))

    def call(self, e, ids, prec, j0=0, **outs):
        wh = np.asarray(ids, dtype=np.int32)
        s = slice(j0, j0 + len(wh))
        p, t, r = e.track_batch(*self.frame, self.K, self.poses[s], self.width[s], self.A[0][s], self.A[1][s], TN, RN,
                                weight_ids_host=wh, weight_ids_dev=outs.pop('wid_dev', None), precision=prec, **outs)
        return t, r, p

    def run(self, e, ids, prec, j0=0):
        return [x.cpu().numpy() for x in self.call(e, ids, prec, j0)]

    def calibrate(self, e, ids):
        """calibrate_fp8_tracks on tracks 0 .. len(ids) - 1 with those ids -> {id it calibrated: its scales}, in the order
        it returned them."""
        m = len(ids)
        done = e.calibrate_fp8_tracks(*self.frame, self.K, self.poses[:m], self.width[:m], self.A[0][:m], self.A[1][:m],
                                      weight_ids=np.asarray(ids, np.int32))
        return {w: e.fp8_scales(w) for w in done}


def assert_tracks_alone(e, tracks, ids, prec, got, label):
    """got (trans, rot, poses) of a latency-mode step with `ids`: each track equals, bit for bit, that track run alone (n = 1)
    on e with its own id, the single-set path."""
    bad = []
    for j, w in enumerate(ids):
        alone = tracks.run(e, [w], prec, j0=j)
        bad += ['track %d (id %d) %s' % (j, w, name) for name, a, b in zip(('trans', 'rot', 'pose'), got, alone) if not same_bits(a[j:j + 1], b)]
    assert not bad, '%s: differ from the track run alone: %s' % (label, bad)


# ------------------------------------------------------------------------------------------- every layer against fp64
@pytest.mark.parametrize('prec,n', [(p, n) for n in LATENCY for p in PRECS], ids=['%s-n%d' % (p, n) for n in LATENCY for p in PRECS])
def test_latency_mixed_layers(synth, eng, blobs, prec, n):
    """n <= 4 tracks on different sets: the trunk's B producer takes every unit's weights from its image's set while the unit's
    K pieces run on different CTAs, and the pieces' sums are added before the epilogue adds that set's bias.  All images."""
    ids, tracks = LATENCY[n], Tracks(eng, synth, n, seed=20 + n)
    assert_distinct_fp8_scales(eng, ids, prec)
    run_case(eng, prec, 0, n, lambda: (*tracks.call(eng, ids, prec)[:2], None), ids, blobs, 'track_batch, ids %s' % ids)


@pytest.mark.parametrize('prec,ids', THROUGHPUT, ids=['%s-n%d' % (p, len(ids)) for p, ids in THROUGHPUT])
def test_throughput_mixed_layers(synth, eng, blobs, prec, ids):
    """n > 4 tracks on sparse sets; the sampled images always include two weight ids."""
    n = len(ids)
    tracks = Tracks(eng, synth, n, seed=30 + n)
    assert_distinct_fp8_scales(eng, ids, prec)
    label = 'track_batch, ids %s' % ids if n <= 5 else 'track_batch, %d distinct ids' % len(set(ids))
    run_case(eng, prec, 0, n, lambda: (*tracks.call(eng, ids, prec)[:2], None), ids, blobs, label, seed=n)


# ------------------------------------------------------------------------------------------- bit identities on every track
@pytest.mark.parametrize('prec', PRECS)
def test_latency_tracks_equal_their_single_set_runs(synth, eng, prec):
    for n, ids in LATENCY.items():
        assert_distinct_fp8_scales(eng, ids, prec)
        tracks = Tracks(eng, synth, n, seed=20 + n)
        assert_tracks_alone(eng, tracks, ids, prec, tracks.run(eng, ids, prec), 'n = %d, ids %s' % (n, ids))


@pytest.mark.parametrize('prec', PRECS)
def test_throughput_step_equals_single_set_launches(synth, eng, prec):
    """64 tracks on ids drawn from 1..21 against the same 64 tracks run with one set for all of them, once per id used."""
    ids = np.asarray(THROUGHPUT[-1][1], dtype=np.int32)
    tracks = Tracks(eng, synth, 64, seed=3)
    assert_distinct_fp8_scales(eng, ids, prec)
    mixed = tracks.run(eng, ids, prec)
    bad = []
    for w in np.unique(ids):
        single = tracks.run(eng, np.full(64, w, np.int32), prec)
        sel = ids == w
        bad += ['id %d %s' % (w, name) for name, a, b in zip(('trans', 'rot', 'pose'), mixed, single) if not same_bits(a[sel], b[sel])]
    assert not bad, bad


def test_eval_pairs_equal_single_set_pairs(synth, eng):
    """Validation steps with ids [17, 3, 9]: each pair's 6-vector and squared-error terms equal that pair's single-set step."""
    ids, n = np.array([17, 3, 9], np.int32), 3
    A = synth.raw_poses(n, seed=9)
    B = A.copy()
    B[:, :3, 3] += (0.004, -0.003, 0.006)
    rgbA, depthA = synth.rendered_views(n, A, seed=9)
    rgbB, depthB = synth.rendered_views(n, B, seed=10)
    args = [_dev(eng, x) for x in (rgbA, depthA, rgbB, depthB, A, B)]
    for prec in PRECS:
        assert_distinct_fp8_scales(eng, ids, prec)
        tr, ro, _, sq, _ = eng.eval_pairs(*args, TN, RN, weight_ids_host=ids, precision=prec, want_terms=True)
        got = [x.cpu().numpy() for x in (tr, ro, sq)]
        for j, w in enumerate(ids):
            t1, r1, _, q1, _ = eng.eval_pairs(*(x[j:j + 1] for x in args), TN, RN, weight_ids_host=[w], precision=prec, want_terms=True)
            for name, a, b in zip(('trans', 'rot', 'terms'), got, (t1, r1, q1)):
                assert same_bits(a[j:j + 1], b.cpu().numpy()), (prec, j, int(w), name)


# ------------------------------------------------------------------------------------------- K0 with sparse ids
def assert_k0(tA, tB, synth, rgb, depth, poses, rgbA, depthA, ids, dtype):
    """The (n,4,176,176) tensors of K0 equal, bit for bit, processData with each track's own statistics."""
    for i, w in enumerate(ids):
        bb = O.compute_bbox(poses[i], synth.CAMERA_K, 200.0, scale=(1000, 1000, 1000))
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        (dA_, dB_), _ = O.process_data(rgbA[i], depthA[i], poses[i], rB, dB, np.eye(4), *stats(synth, w, dtype))
        assert same_bits(tA[i], dA_) and same_bits(tB[i], dB_), 'track %d (id %d)' % (i, w)


@pytest.mark.parametrize('dtype', [np.float32, np.float64], ids=['fp32', 'fp64'])
def test_preprocess_sparse_ids(pkg, synth, dtype):
    """Weights and statistics only at ids 4, 13 and 20: the statistics table has 21 rows, 18 of them empty."""
    e = pkg.Engine(max_batch=4)
    try:
        for w in (4, 13, 20):
            load(e, synth, w, dtype=dtype)
        ids = np.array([20, 4, 13, 4], np.int32)
        rgb, depth, poses, rgbA, depthA = track_inputs(synth, 4, seed=12)
        tA, tB, _, _ = e.preprocess(_dev(e, rgb), _dev(e, depth), synth.CAMERA_K, _dev(e, poses), _dev(e, np.full(4, 200.0)),
                                    _dev(e, rgbA), _dev(e, depthA), weight_ids=_dev(e, ids), want_tensors=True)
        assert_k0(tA.cpu().numpy(), tB.cpu().numpy(), synth, rgb, depth, poses, rgbA, depthA, ids, dtype)
    finally:
        e.close()


def test_mixed_statistics_dtypes_refuse_the_step(pkg, synth):
    lib = importlib.import_module(pkg.__name__ + '._lib')
    e = pkg.Engine(max_batch=2)
    try:
        load(e, synth, 4, dtype=np.float32)
        load(e, synth, 13, dtype=np.float64)
        tracks = Tracks(e, synth, 2, seed=13)
        with pytest.raises(lib.Se3tnError) as err:
            tracks.call(e, [4, 13], 'bf16x3')
        assert err.value.code == lib.ERR_STATE and 'dtype' in str(err.value)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------- state rules with sparse ids
def test_fp16_refuses_a_set_outside_its_range_among_sparse_ids(pkg, synth, blobs):
    """Sets at 4, 13 and 20, set 13 with one conv weight of 1e5: an fp16 step on ids [4, 13, 20] is refused with
    SE3TN_ERR_STATE naming 13 and writes nothing; the same step runs in bf16x3."""
    lib = importlib.import_module(pkg.__name__ + '._lib')
    e = pkg.Engine(max_batch=3)
    try:
        for w in (4, 20):
            load(e, synth, w)
        blob = np.array(blobs[13], dtype=np.float32)
        w_off, _, _ = R.blob_offsets()
        blob[w_off[9] + 1234] = 1e5                    # convAB2.conv1
        lib.check(e.lib.se3tn_load_weights(e._ctx, 13, blob.ctypes.data_as(ctypes.c_void_p), blob.size), e._ctx)
        e.set_stats(*stats(synth, 13), 13)
        ids = [4, 13, 20]
        tracks = Tracks(e, synth, 3, seed=16)
        poison(e, 'fp16')
        with pytest.raises(lib.Se3tnError) as err:
            tracks.call(e, ids, 'fp16')
        torch.cuda.synchronize()
        assert err.value.code == lib.ERR_STATE and 'weight set 13 ' in str(err.value)
        check_poison_outside(e, 'fp16', 0, 0)
        t, r, _ = tracks.run(e, ids, 'bf16x3')
        assert np.isfinite(t).all() and np.isfinite(r).all()
    finally:
        e.close()


def test_calibrate_fp8_tracks_sparse_ids(pkg, synth):
    """calibrate_fp8_tracks on tracks with ids [20, 4, 13, 4, 20, 13]: it calibrates 4, 13 and 20, in that order, and each
    set's scales are, bit for bit, those of calibrate_fp8 on exactly that set's pairs."""
    e = pkg.Engine(max_batch=6)
    try:
        for w in (4, 13, 20):
            load(e, synth, w)
        ids = np.array([20, 4, 13, 4, 20, 13], np.int32)
        tracks = Tracks(e, synth, len(ids), seed=17)
        got = tracks.calibrate(e, ids)
        assert list(got) == [4, 13, 20]
        A, B, _, _ = e.preprocess(*tracks.frame, tracks.K, tracks.poses, tracks.width, *tracks.A, weight_ids=_dev(e, ids),
                                  want_tensors=True)
        for w in (4, 13, 20):
            idx = torch.from_numpy(np.flatnonzero(ids == w)).to(e.device)
            assert same_bits(e.calibrate_fp8(A[idx], B[idx], weight_id=w), got[w]), 'id %d' % w
    finally:
        e.close()


# ------------------------------------------------------------------------------------------- reloads
def reload_steps(pkg, synth, prec):
    """One engine with sets at 3, 9, 17 and 21 (tables of 22 rows) and steps captured as CUDA graphs; the step's ids, outputs
    and inputs stay at the same addresses throughout, as the drivers keep them.
      1. id 30 is loaded (the tables grow to 31 rows): a step with ids [30, 3, 17] equals its tracks run alone and passes the
         per-layer gate against id 30's weights;
      2. id 9 is replaced by another seed: its tracks equal a fresh engine holding that seed at id 9, the others are unchanged;
      3. id 9's statistics change: K0 of its tracks in the next step uses the new values.
    fp8: every set has scales of its own.  A set without scales -- id 30 once loaded, id 9 once replaced (a reload drops
    them) -- refuses the step with SE3TN_ERR_STATE naming it, and nothing is written; once it has scales the step runs as
    above.  New statistics keep the set's scales."""
    lib = importlib.import_module(pkg.__name__ + '._lib')
    n = 4
    fp8 = prec == 'fp8'
    e = pkg.Engine(max_batch=n)
    fresh = None
    try:
        for w in (3, 9, 17, 21):
            load(e, synth, w)
        tracks = Tracks(e, synth, n, seed=14)
        if fp8:
            calibrated = tracks.calibrate(e, [3, 9, 17, 21])
            scales = distinct_fp8_scales(e, calibrated)
        wid_dev = torch.empty(n, dtype=torch.int32, device=e.device)
        outs = dict(out_poses=torch.empty(n, 4, 4, dtype=torch.float64, device=e.device),
                    out_trans=torch.empty(n, 3, device=e.device), out_rot=torch.empty(n, 3, device=e.device))

        def step(ids):
            m = len(ids)
            wid_dev[:m].copy_(torch.tensor(ids, dtype=torch.int32))
            t, r, _ = tracks.call(e, ids, prec, wid_dev=wid_dev[:m], **{k: v[:m] for k, v in outs.items()})
            return t, r, None

        def results(m):
            return [outs[k][:m].cpu().numpy() for k in ('out_trans', 'out_rot', 'out_poses')]

        def refused(ids, wid):
            poison(e, prec)
            with pytest.raises(lib.Se3tnError) as err:
                step(ids)
            torch.cuda.synchronize()
            assert err.value.code == lib.ERR_STATE and 'weight set %d ' % wid in str(err.value), str(err.value)
            check_poison_outside(e, prec, 0, 0)

        for _ in range(2):
            step([21, 3, 17])
        assert e.last_step_was_graph()
        # 1. a set added after steps were captured
        load(e, synth, 30)
        ids = [30, 3, 17]
        if fp8:
            refused(ids, 30)
            calibrated.update(tracks.calibrate(e, ids))
            scales = distinct_fp8_scales(e, calibrated)
            assert_distinct_fp8_scales(e, ids, prec)
        run_case(e, prec, 0, 3, lambda: step(ids), ids, Blobs(pkg, synth), 'track_batch after loading id 30, ids %s' % ids)
        assert_tracks_alone(e, tracks, ids, prec, results(3), 'after loading id 30')
        # 2. a set replaced under its id
        ids = [9, 3, 9, 17]
        for _ in range(2):
            step(ids)
        assert e.last_step_was_graph()
        before = results(n)
        e.load_state_dict(synth.make_state_dict(109), 9)
        if fp8:
            assert e.fp8_scales(9) is None
            refused(ids, 9)
            e.set_fp8_scales(scales[9], 9)
        step(ids)
        after = results(n)
        fresh = pkg.Engine(max_batch=n)
        load(fresh, synth, 9, seed=109)
        if fp8:
            fresh.set_fp8_scales(scales[9], 9)
        for j, w in enumerate(ids):
            want = before if w != 9 else tracks.run(fresh, [9], prec, j0=j)
            lo = 0 if w == 9 else j                      # a track run alone has one row
            for name, a, b in zip(('trans', 'rot', 'pose'), after, want):
                assert same_bits(a[j:j + 1], b[lo:lo + 1]), 'track %d (id %d) %s after id 9 was replaced' % (j, w, name)
        assert not same_bits(after[0][0], before[0][0])                  # the new weights changed the result
        # 3. new statistics for id 9 (in the step's stem buffers, whose format stores each value as bf16 hi + lo)
        e.set_stats(*stats(synth, 109), 9)
        if fp8:
            assert same_bits(e.fp8_scales(9), scales[9])
        step(ids)
        torch.cuda.synchronize()
        rgb, depth, poses, rgbA, depthA = track_inputs(synth, n, seed=14)
        k0 = []
        for buf in ('X0A', 'X0B'):
            nb = image_bytes(buf, prec)
            raw = e.debug_buffer(R.BUF_ID[buf], n).view(torch.uint8).reshape(-1)[:n * nb].cpu().numpy()
            k0.append(np.stack([decode(raw[i * nb:(i + 1) * nb], buf, prec).value[:, 3:179, 3:179] for i in range(n)]))
        want = [np.empty_like(k) for k in k0]
        for i, w in enumerate(ids):
            bb = O.compute_bbox(poses[i], synth.CAMERA_K, 200.0, scale=(1000, 1000, 1000))
            rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
            (dA_, dB_), _ = O.process_data(rgbA[i], depthA[i], poses[i], rB, dB, np.eye(4), *stats(synth, 109 if w == 9 else w))
            for k, d in zip(want, (dA_, dB_)):
                hi, lo = R.split2(d)
                k[i] = hi + lo
        for i, w in enumerate(ids):
            assert same_bits(k0[0][i], want[0][i]) and same_bits(k0[1][i], want[1][i]), 'K0 of track %d (id %d) after new statistics' % (i, w)
    finally:
        e.close()
        if fresh is not None:
            fresh.close()


def test_added_replaced_and_restated_sets_reach_the_next_step(pkg, synth):
    reload_steps(pkg, synth, 'bf16x3')


@pytest.mark.parametrize('prec', ['fp16', 'fp8'])
def test_reloads_reach_the_next_step_in_fp16_and_fp8(pkg, synth, prec):
    reload_steps(pkg, synth, prec)


def test_fp8_new_scales_of_one_set_reach_a_captured_step(pkg, synth, eng):
    """A captured fp8 step on all 21 sets, new scales for one of them: the step replays its graph (a set's scales sit at
    fixed device addresses), only that id's tracks change, and every track equals the same step on a fresh engine holding
    the same sets and scales.  The old scales give the old bits back."""
    ids = np.asarray(SHUFFLED, dtype=np.int32)
    n, w = len(ids), 5
    tracks = Tracks(eng, synth, n, seed=15)
    wid_dev = _dev(eng, ids)
    outs = dict(out_poses=torch.empty(n, 4, 4, dtype=torch.float64, device=eng.device),
                out_trans=torch.empty(n, 3, device=eng.device), out_rot=torch.empty(n, 3, device=eng.device))

    def step():
        tracks.call(eng, ids, 'fp8', wid_dev=wid_dev, **outs)
        return [outs[k].cpu().numpy() for k in ('out_trans', 'out_rot', 'out_poses')]

    step()
    old = step()
    assert eng.last_step_was_graph()
    s = eng.fp8_scales(w)
    fresh = None
    try:
        eng.set_fp8_scales(s * 2, w)
        new = step()
        assert eng.last_step_was_graph()
        sel = ids == w
        assert not same_bits(new[0][sel], old[0][sel]), 'new scales of id %d did not change its tracks' % w
        bad = [name for name, a, b in zip(('trans', 'rot', 'pose'), new, old) if not same_bits(a[~sel], b[~sel])]
        assert not bad, 'new scales of id %d changed the other tracks: %s' % (w, bad)
        fresh = pkg.Engine(max_batch=n)
        for v in IDS:
            load(fresh, synth, v)
            fresh.set_fp8_scales(eng.fp8_scales(v), v)
        want = tracks.run(fresh, ids, 'fp8')
        bad = [name for name, a, b in zip(('trans', 'rot', 'pose'), new, want) if not same_bits(a, b)]
        assert not bad, 'differs from a fresh engine: %s' % bad
    finally:
        eng.set_fp8_scales(s, w)
        if fresh is not None:
            fresh.close()
    back = step()
    assert eng.last_step_was_graph()
    assert all(same_bits(a, b) for a, b in zip(back, old)), 'the old scales did not give the old bits back'
