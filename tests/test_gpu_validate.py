"""GPU: checkpoint validation (se3tn_eval_pairs, se3tn_pair_loss, TrackDataset.__getitem__, Problem.validate) against the CPU
oracle on pair folders written in the reference's on-disk format: <i>rgbA.png, rgbB.png, depthA.png, depthB.png, [segB.png],
meta.npz (A_in_cam, B_in_cam).  rgbB / depthB are crops of synthetic frames at A's pose, input A is drawn by the CUDA rasteriser,
and A_in_cam is B_in_cam moved by a restatement of the reference's random_gaussian_magnitude (Utils.py:372-390)."""
import os
import cv2
import numpy as np
import pytest
import torch
from PIL import Image
import se3_oracle as O

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
TN, RN = 0.02, 15 * np.pi / 180                       # reference dataset_info.yml: max_translation, max_rotation
GATES = {'bf16x3': (1e-3, 1e-4), 'tf32': (1e-3, 1e-4), 'fp32': (1e-4, 2e-6), 'bf16': (1e-2, 5e-3)}   # DESIGN §2, test_gpu_parity.py
# The validation loss against the reference loop on the CPU.  fp32: rtol 1e-5.  Every mode: the loss may move only as far as
# its own 6-vectors moved (each gated above): |(p' - l)^2 - (p - l)^2| <= 2 |p - l| |p' - p| + (p' - p)^2 per element, plus
# the rounding of the two float32 means (2e-6 relative).  No pipeline error fits under that bound: a wrong label, term or
# batch split moves the loss far beyond what the 6-vector deviation explains.
LOSS_RTOL = {'fp32': 1e-5}
MEAN_ROUNDING = 2e-6


def random_gaussian_magnitude(rng, max_T, max_R):
    """Utils.py:372-390: a random direction times a truncated-normal magnitude, for the translation (m) and the rotation (deg)."""
    def direction():
        v = rng.normal(size=3)
        return v / np.linalg.norm(v)
    while True:
        mT = rng.normal(0, max_T)
        if abs(mT) <= max_T:
            break
    T = direction() * mT
    while True:
        mR = rng.normal(0, max_R)
        if abs(mR) <= max_R:
            break
    pose = np.eye(4)
    pose[:3, :3] = cv2.Rodrigues(direction() * mR / 180.0 * np.pi)[0]
    pose[:3, 3] = T
    return pose


def write_folder(eng, synth, d, n, seed, size=176, seg=True):
    """n pairs in d; returns the arrays as written (A_in_cam, B_in_cam)."""
    os.makedirs(d, exist_ok=True)
    rng = np.random.default_rng(seed)
    K = synth.CAMERA_K
    rgb, depth = synth.raw_frame(seed)
    B = synth.raw_poses(n, seed=seed)
    A = np.stack([random_gaussian_magnitude(rng, TN, 15.0) for _ in range(n)])
    A[:, :3, :3] = A[:, :3, :3] @ B[:, :3, :3]
    A[:, :3, 3] += B[:, :3, 3]
    dev = eng.device
    views = [eng.render(K, torch.from_numpy(A[i:i + eng.max_batch].copy()).to(dev),
                        torch.full((min(n - i, eng.max_batch),), 200.0, dtype=torch.float64, device=dev)) for i in range(0, n, eng.max_batch)]
    rgbA = torch.cat([v[0] for v in views]).cpu().numpy(); depthA = torch.cat([v[1] for v in views]).cpu().numpy()
    for i in range(n):
        bb = O.compute_bbox(A[i], K, 200.0, scale=(1000, 1000, 1000))
        rB, dB = O.crop_bbox(rgb, depth, bb, (size, size))
        rA, dA = rgbA[i], depthA[i]
        if size != 176:
            rA = cv2.resize(rA, (size, size), interpolation=cv2.INTER_NEAREST)
            dA = cv2.resize(dA, (size, size), interpolation=cv2.INTER_NEAREST)
        stem = os.path.join(d, '%05d' % i)
        Image.fromarray(rA).save(stem + 'rgbA.png'); Image.fromarray(rB).save(stem + 'rgbB.png')
        cv2.imwrite(stem + 'depthA.png', dA); cv2.imwrite(stem + 'depthB.png', dB)
        if seg:
            m = (dB > 100).astype(np.uint8)
            m[size // 2, size // 2] = 1
            cv2.imwrite(stem + 'segB.png', m)
        np.savez(stem + 'meta.npz', A_in_cam=A[i], B_in_cam=B[i])
    return A, B


def reference_item(path, res=176):
    """TrackDataset.__getitem__'s file reading (datasets.py:70-104) restated with PIL / cv2 as the reference does it."""
    rgbB = np.array(Image.open(path.replace('rgbA', 'rgbB')))
    depthB = cv2.imread(path.replace('rgbA', 'depthB'), cv2.IMREAD_UNCHANGED)
    maskB = cv2.imread(path.replace('rgbA', 'segB'), cv2.IMREAD_UNCHANGED)
    meta = np.load(path.replace('rgbA.png', 'meta.npz'))
    rgbA = np.array(Image.open(path))
    depthA = cv2.imread(path.replace('rgbA', 'depthA'), cv2.IMREAD_UNCHANGED)
    if rgbB.shape[0] != res:
        rgbA, rgbB = (cv2.resize(x, (res, res), interpolation=cv2.INTER_NEAREST) for x in (rgbA, rgbB))
        depthA, depthB = (cv2.resize(x, (res, res), interpolation=cv2.INTER_NEAREST) for x in (depthA, depthB))
        if maskB is not None:
            maskB = cv2.resize(maskB, (res, res), interpolation=cv2.INTER_NEAREST)
    if maskB is None:
        maskB = (depthB > 100).astype(np.uint8)
    return rgbA, depthA, rgbB, depthB, maskB, meta['A_in_cam'], meta['B_in_cam']


def oracle_validate(sd, files, mean, std, batch_size):
    """Problem.validate (problems.py:106-132) on the CPU: the reference model (oracle forward), oracle processData, nn.MSELoss,
    DataLoader(batch_size, shuffle=False, drop_last=False).  -> (trans, rot, per-pair 6-vectors, per-pair labels)."""
    tl_all, rl_all, preds, labels = [], [], [], []
    for b0 in range(0, len(files), batch_size):
        As, Bs, tls, rls = [], [], [], []
        for f in files[b0:b0 + batch_size]:
            rgbA, depthA, rgbB, depthB, maskB, A, B = reference_item(f)
            assert np.sum(maskB) > 0
            (dA, dB), (tl, rl) = O.process_data(rgbA, depthA, A, rgbB, depthB, B, mean, std, TN, RN)
            As.append(dA); Bs.append(dB); tls.append(tl); rls.append(rl)
        out = O.forward(sd, torch.from_numpy(np.stack(As)), torch.from_numpy(np.stack(Bs)))
        tt, rt = torch.from_numpy(np.stack(tls)), torch.from_numpy(np.stack(rls))
        tl_all.append(torch.nn.MSELoss()(out['trans'].float(), tt.float()).item())
        rl_all.append(torch.nn.MSELoss()(out['rot'].float(), rt.float()).item())
        preds.append(torch.cat((out['trans'], out['rot']), 1).numpy()); labels.append(np.concatenate((tls, rls), 1))
    return np.array(tl_all).mean(), np.array(rl_all).mean(), np.concatenate(preds), np.concatenate(labels)


def loss_bound(pred_ref, labels, batch_size, tol):
    """How far a batch-mean MSE may move when every prediction moves by at most `tol` (per element, or a scalar):
    mean over batches of mean(2 |p - l| tol + tol^2), per head."""
    d = np.abs(pred_ref - labels.astype(np.float32))
    e = 2 * d * tol + tol * tol
    per_batch = [(e[b:b + batch_size, :3].mean(), e[b:b + batch_size, 3:].mean()) for b in range(0, len(e), batch_size)]
    return np.mean(per_batch, axis=0)


@pytest.fixture(scope='module')
def setup(pkg, synth, tmp_path_factory):
    eng = pkg.Engine(max_batch=8)
    sd0, sd1 = synth.make_state_dict(0), synth.make_state_dict(1)
    eng.load_state_dict(sd0, 0); eng.load_state_dict(sd1, 1)
    mean, std = synth.default_mean_std()
    eng.set_stats(mean, std, 0); eng.set_stats(mean + 1.5, std * 1.25, 1)
    eng.set_mesh(synth.mesh(), 0)
    root = tmp_path_factory.mktemp('val')
    dirs = {'seg': str(root / 'seg'), 'noseg': str(root / 'noseg'), 'small': str(root / 'small')}
    write_folder(eng, synth, dirs['seg'], 21, seed=1, seg=True)
    write_folder(eng, synth, dirs['noseg'], 5, seed=2, seg=False)
    write_folder(eng, synth, dirs['small'], 4, seed=3, size=128, seg=True)
    yield dict(eng=eng, sd=(sd0, sd1), mean=mean, std=std, dirs=dirs)
    eng.close()


def _load_batch(eng, files):
    items = [reference_item(f) for f in files]
    dev = eng.device
    st = lambda k, dt: torch.from_numpy(np.ascontiguousarray(np.stack([it[k] for it in items]).astype(dt))).to(dev)
    return (st(0, np.uint8), st(1, np.uint16), st(2, np.uint8), st(3, np.uint16), st(5, np.float64), st(6, np.float64), items)


def test_eval_pairs_labels_terms_and_six_vectors(pkg, setup):
    eng, sd, mean, std = setup['eng'], setup['sd'][0], setup['mean'], setup['std']
    files = sorted(__import__('glob').glob(setup['dirs']['seg'] + '/*rgbA.png'))[:8]
    rgbA, depthA, rgbB, depthB, A, B, items = _load_batch(eng, files)
    tl_ref, rl_ref = eng.so3_log(A, B, TN, RN)
    for prec, (rt, at) in GATES.items():
        tr, ro, sums, sq, lab = eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, precision=prec, want_terms=True, want_labels=True)
        torch.cuda.synchronize()
        lab = lab.cpu().numpy()
        assert np.array_equal(lab, torch.cat((tl_ref, rl_ref), 1).cpu().numpy())      # the same device function as se3tn_so3_log
        six = np.concatenate((tr.cpu().numpy(), ro.cpu().numpy()), 1)
        expect = np.square(six - lab.astype(np.float32))                               # numpy float32: (pred - float(label))^2
        assert expect.dtype == np.float32 and np.array_equal(sq.cpu().numpy(), expect)
        # the sums are se3tn_pair_loss's on the same predictions and labels, bit for bit
        s2 = eng.pair_loss(tr, ro, torch.from_numpy(lab[:, :3].copy()).to(eng.device), torch.from_numpy(lab[:, 3:].copy()).to(eng.device))
        assert torch.equal(sums, s2)
        np.testing.assert_allclose(sums.cpu().numpy(), [expect[:, :3].sum(dtype=np.float64), expect[:, 3:].sum(dtype=np.float64)], rtol=1e-6)
        # against the oracle: labels (cv2.Rodrigues' SVD vs the polar iteration: the so3_log tolerance), 6-vectors within the gates
        pd = [O.process_data(it[0], it[1], it[5], it[2], it[3], it[6], mean, std, TN, RN) for it in items]
        oracle_labels = np.stack([np.concatenate(p[1]) for p in pd])
        assert np.array_equal(lab[:, :3], oracle_labels[:, :3]) and np.abs(lab[:, 3:] - oracle_labels[:, 3:]).max() < 1e-9
        out = O.forward(sd, torch.from_numpy(np.stack([p[0][0] for p in pd])), torch.from_numpy(np.stack([p[0][1] for p in pd])))
        ref6 = torch.cat((out['trans'], out['rot']), 1).numpy()
        assert (np.abs(six - ref6) <= at + rt * np.abs(ref6)).all(), prec


def test_eval_pairs_graph_replay_launches_and_mixed_sets(pkg, setup):
    eng = setup['eng']
    files = sorted(__import__('glob').glob(setup['dirs']['seg'] + '/*rgbA.png'))[:8]
    rgbA, depthA, rgbB, depthB, A, B, _ = _load_batch(eng, files)
    outs = [torch.empty(8, 3, device=eng.device), torch.empty(8, 3, device=eng.device), torch.empty(2, device=eng.device)]
    kw = dict(precision='bf16x3', out_trans=outs[0], out_rot=outs[1], out_sums=outs[2])
    eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, **kw)
    first = [o.clone() for o in outs]
    eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, **kw)
    torch.cuda.synchronize()
    assert eng.last_step_was_graph() and eng.last_launch_count() == 12        # normalize + 8 resident + trunk + head + reduction
    assert all(torch.equal(a, b) for a, b in zip(first, outs))
    eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, precision='fp32')
    assert not eng.last_step_was_graph() and eng.last_launch_count() == 1 + 17 + 1
    # two weight sets interleaved in one step: each pair as if its set ran alone
    ids = np.array([0, 1] * 4, dtype=np.int32)
    for prec in ('bf16x3', 'fp32'):
        tr, ro, sums, sq, _ = eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, weight_ids_host=ids, precision=prec, want_terms=True)
        if prec == 'fp32':
            assert eng.last_launch_count() == 1 + 8 * 17 + 1                     # one FFMA forward per run of equal ids
        for w in (0, 1):                                 # the same 8 pairs, all with set w
            t1, r1, _, q1, _ = eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, weight_ids_host=np.full(8, w, np.int32),
                                              precision=prec, want_terms=True)
            sel = ids == w
            assert torch.equal(tr[sel], t1[sel]) and torch.equal(ro[sel], r1[sel]) and torch.equal(sq[sel], q1[sel]), (prec, w)


def test_eval_pairs_errors(pkg, setup, synth):
    eng = setup['eng']
    L = __import__('importlib').import_module(PKG + '._lib')
    files = sorted(__import__('glob').glob(setup['dirs']['seg'] + '/*rgbA.png'))[:2]
    rgbA, depthA, rgbB, depthB, A, B, _ = _load_batch(eng, files)
    with pytest.raises(L.Se3tnError) as e:
        eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, weight_ids_host=np.array([0, 5], np.int32))
    assert e.value.code == L.ERR_STATE and 'weight set 5' in str(e.value)
    eng.load_state_dict(synth.make_state_dict(2), 7)                         # weights without statistics
    with pytest.raises(L.Se3tnError) as e:
        eng.eval_pairs(rgbA, depthA, rgbB, depthB, A, B, TN, RN, weight_ids_host=np.array([7, 0], np.int32))
    assert e.value.code == L.ERR_STATE and '7' in str(e.value) and 'mean/std' in str(e.value)
    idx = torch.zeros(9, dtype=torch.long, device=eng.device)
    big = lambda t: (t.view(torch.int16)[idx].view(torch.uint16) if t.dtype == torch.uint16 else t[idx]).contiguous()
    with pytest.raises(L.Se3tnError) as e:
        eng.eval_pairs(big(rgbA), big(depthA), big(rgbB), big(depthB), big(A), big(B), TN, RN)
    assert e.value.code == L.ERR_INVALID


def _dataset(pkg, setup, key, eng):
    D = __import__('importlib').import_module(PKG + '.datasets')
    return D.TrackDataset(setup['dirs'][key], 'val', setup['mean'], setup['std'], dataset_info={
        'resolution': 176, 'camera': {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109}},
        trans_normalizer=TN, rot_normalizer=RN, engine=eng, precision='fp32')


def test_getitem_and_resize_branch(pkg, setup):
    eng = setup['eng']
    D = __import__('importlib').import_module(PKG + '.datasets')
    for key in ('seg', 'noseg', 'small'):
        ds = _dataset(pkg, setup, key, eng)
        for i in range(min(3, len(ds))):
            data, (tl, rl), A, B, rgbA, rgbB, maskA, maskB = ds[i]
            rA, dA, rB, dB, mB, A_r, B_r = reference_item(ds.rgbA_files[i])
            assert np.array_equal(rgbA, rA) and np.array_equal(rgbB, rB) and np.array_equal(maskB, mB), (key, i)
            assert np.array_equal(A, A_r) and np.array_equal(B, B_r) and maskA.shape == (176, 176)
            (oA, oB), (otl, orl) = O.process_data(rA, dA, A_r, rB, dB, B_r, setup['mean'], setup['std'], TN, RN)
            assert np.array_equal(data[0].numpy(), oA) and np.array_equal(data[1].numpy(), oB)
            assert np.array_equal(tl, otl) and np.abs(rl - orl).max() < 1e-9
    # the device resize is cv2.resize(INTER_NEAREST) bit for bit, down and up
    rng = np.random.default_rng(5)
    for (h, w), s in (((128, 128), 176), ((200, 150), 176), ((176, 176), 100), ((37, 251), 176)):
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8); dep = rng.integers(0, 65536, (h, w)).astype(np.uint16)
        r, d = D.resize_nearest(eng, rgb, dep, s)
        assert np.array_equal(r.cpu().numpy(), cv2.resize(rgb, (s, s), interpolation=cv2.INTER_NEAREST))
        assert np.array_equal(d.cpu().numpy(), cv2.resize(dep, (s, s), interpolation=cv2.INTER_NEAREST))


def test_getitem_in_a_worker_is_refused(pkg, setup, monkeypatch):
    ds = _dataset(pkg, setup, 'seg', setup['eng'])
    monkeypatch.setattr(torch.utils.data, 'get_worker_info', lambda: object())   # what a DataLoader worker process sees
    with pytest.raises(RuntimeError, match='Problem.validate'):
        ds[0]


def test_problem_validate_vs_reference_loop(pkg, setup, synth):
    P = __import__('importlib').import_module(PKG + '.problems')
    Se3TrackNet = pkg.Se3TrackNet
    root = os.path.dirname(setup['dirs']['seg'])
    allf = os.path.join(root, 'all')
    os.makedirs(allf, exist_ok=True)
    for key in ('seg', 'noseg', 'small'):                # 30 pairs from the three folders, both naming patterns
        for f in os.listdir(setup['dirs'][key]):
            dst = os.path.join(allf, key + f)
            if not os.path.exists(dst):
                os.symlink(os.path.join(setup['dirs'][key], f), dst)
    ds = _dataset(pkg, setup, 'seg', setup['eng'])
    ds.root = allf
    ds.rgbA_files = sorted(__import__('glob').glob(allf + '/*rgbA.png'))
    assert len(ds) == 30
    sd = setup['sd'][0]
    for bs in (12, 200):                                 # 12: partial last batch, batches of 2 steps (max_batch 8)
        loader = torch.utils.data.DataLoader(ds, batch_size=bs, shuffle=False, drop_last=False)
        t_ref, r_ref, pred_ref, lab = oracle_validate(sd, ds.rgbA_files, setup['mean'], setup['std'], bs)
        model = Se3TrackNet(engine=setup['eng'], weight_id=0)
        model.load_state_dict(sd)
        prob = P.Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}})
        for prec, (rt, at) in GATES.items():
            r = prob.validation_losses(prec, keep_predictions=True)
            six = r['predictions']
            assert (np.abs(six - pred_ref) <= at + rt * np.abs(pred_ref)).all(), prec
            gate = loss_bound(pred_ref, lab, bs, at + rt * np.abs(pred_ref))
            moved = loss_bound(pred_ref, lab, bs, np.abs(six.astype(np.float64) - pred_ref))
            for got, ref, g, m in ((r['trans'], t_ref, gate[0], moved[0]), (r['rot'], r_ref, gate[1], moved[1])):
                print('validate %-6s batch %3d: %.9g vs reference %.9g (rel %.2e; bound from its 6-vector deviation %.2e, from the gate %.2e)'
                      % (prec, bs, got, ref, abs(got - ref) / ref, m, g))
                assert abs(got - ref) <= m + MEAN_ROUNDING * abs(ref) and abs(got - ref) <= g, (prec, bs, got, ref, m, g)
                if prec in LOSS_RTOL:
                    assert abs(got - ref) <= LOSS_RTOL[prec] * abs(ref), (prec, bs, got, ref)
            assert prob.validate(0, precision=prec) == pytest.approx(r['trans'] + r['rot'], rel=0, abs=0)
        # Se3TrackNet.loss agrees with the step's sums bit for bit
        tr = torch.from_numpy(pred_ref[:8, :3].copy()); ro = torch.from_numpy(pred_ref[:8, 3:].copy())
        out = model.loss((tr, ro), [torch.from_numpy(lab[:8, :3].copy()), torch.from_numpy(lab[:8, 3:].copy())])
        ref_t = torch.nn.MSELoss()(tr.float(), torch.from_numpy(lab[:8, :3]).float()).item()
        assert out['trans'].is_cuda and abs(out['trans'].item() - ref_t) <= 1e-6 * ref_t


# ------------------------------------------------------------------ the tracking steps with the loss in the head kernel
GOLDEN_TRACK = 'golden_track_steps.npz'


def track_step_digests(pkg, synth):
    """sha256 of the poses, and the launch count, of track_batch and track_render steps: n = 4 (split-K latency mode) and 37,
    all four modes, one weight set and two interleaved, each step launched twice (capture, then graph replay)."""
    import hashlib
    eng = pkg.Engine(max_batch=64)
    mean, std = synth.default_mean_std()
    for w in (0, 1):
        eng.load_state_dict(synth.make_state_dict(w), w)
        eng.set_mesh(synth.mesh(seed=w), w)
    eng.set_stats(mean, std, 0); eng.set_stats(mean + 1.5, std * 1.25, 1)
    dev = eng.device
    rgb, depth = synth.raw_frame(0)
    fr, fd = torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev)
    out = {}
    for n in (4, 37):
        poses = synth.raw_poses(n, seed=n)
        rgbA, depthA = synth.rendered_views(n, poses, seed=n)
        P = torch.from_numpy(poses).to(dev); ow = torch.full((n,), 200.0, dtype=torch.float64, device=dev)
        rA, dA = torch.from_numpy(rgbA).to(dev), torch.from_numpy(depthA).to(dev)
        for prec in ('bf16x3', 'tf32', 'bf16', 'fp32'):
            for ids in (None, np.arange(n, dtype=np.int32) % 2):
                for call in range(2):
                    tag = '%d_%s_%s_%d' % (n, prec, 'mixed' if ids is not None else 'one', call)
                    p, _, _ = eng.track_batch(fr, fd, synth.CAMERA_K, P, ow, rA, dA, 0.03, 5 * np.pi / 180, weight_ids_host=ids, precision=prec)
                    out['batch_' + tag] = (hashlib.sha256(p.cpu().numpy().tobytes()).hexdigest(), eng.last_launch_count())
                    p, _, _ = eng.track_render(fr, fd, synth.CAMERA_K, P, ow, 0.03, 5 * np.pi / 180, weight_ids_host=ids, precision=prec)
                    out['render_' + tag] = (hashlib.sha256(p.cpu().numpy().tobytes()).hexdigest(), eng.last_launch_count())
    eng.close()
    return out


def write_track_digests(pkg, synth, path):
    d = track_step_digests(pkg, synth)
    np.savez(path, **{k: np.array(v[0]) for k, v in d.items()}, **{k + '_launches': np.array(v[1]) for k, v in d.items()})


def test_tracking_steps_unchanged_by_the_loss_head(pkg, synth, golden_dir):
    """The head kernel also forms the loss terms now; with them off, track_batch and track_render give the poses and launch
    counts of the commit before that change (6d7f128), which recorded the fixture with write_track_digests."""
    g = np.load(os.path.join(golden_dir, GOLDEN_TRACK))
    got = track_step_digests(pkg, synth)
    assert sorted(got) == sorted(k for k in g.files if not k.endswith('_launches'))
    for k, (digest, launches) in got.items():
        assert digest == str(g[k]) and launches == int(g[k + '_launches']), k
