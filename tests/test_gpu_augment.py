"""GPU: validation under the reference's train-time augmentations (se3tn_eval_pairs_augmented, se3tn_augment_draws,
se3tn_augment_crops, TrackDataset(augmentations=...), problems --augment).  The device's augmented crops are compared bit for bit
with oracle/augment_ref.py applied to the draws the device reports; the step's outputs with plain se3tn_eval_pairs on those
crops; the draws' distributions with the reference's."""
import importlib
import os

import cv2
import numpy as np
import pytest
import torch
import yaml
from scipy import stats

import augment_ref as R

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
TN, RN = 0.02, 15 * np.pi / 180
MODES = ('fp32', 'bf16x3', 'tf32', 'bf16', 'fp16', 'fp8')
REF_CONFIG = {'data_augmentation': {'hsv_noise': [15, 15, 15], 'bright_mag': [0.5, 1.5], 'gaussian_noise': {'rgb': 2, 'depth': 5},
                                    'gaussian_blur_kernel': 6, 'depth_missing_percent': 0.4}}     # the reference's config.yml


def A():
    return importlib.import_module(PKG + '.data_augmentation')


def chain(seed=0):
    return A().chain_config(A().from_config(REF_CONFIG), seed)


def make_pairs(n, seed):
    """Random crops: rgb over the full range (the noise wraps at 0 and 255), depth with pixels on both sides of 100 mm, a
    segB disc of ones somewhere in the crop, and poses near each other."""
    rng = np.random.default_rng(seed)
    rgb = rng.integers(0, 256, (n, 176, 176, 3), dtype=np.uint8)
    depth = rng.integers(0, 2500, (n, 176, 176)).astype(np.uint16)
    depth[:, :8] = rng.integers(95, 106, (n, 8, 176))
    yy, xx = np.mgrid[:176, :176]
    seg = np.zeros((n, 176, 176), np.uint8)
    for i in range(n):
        cy, cx, r = rng.integers(20, 156), rng.integers(20, 156), rng.integers(10, 60)
        seg[i] = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
    B = np.tile(np.eye(4), (n, 1, 1))
    B[:, :3, 3] = [0.0, 0.0, 0.8] + rng.normal(0, 0.05, (n, 3))
    Ap = B.copy()
    Ap[:, :3, 3] += rng.normal(0, 0.01, (n, 3))
    Ap[:, :3, :3] = np.stack([cv2.Rodrigues(rng.normal(0, 0.05, 3))[0] for _ in range(n)]) @ B[:, :3, :3]
    rgbA = rng.integers(0, 256, (n, 176, 176, 3), dtype=np.uint8)
    depthA = rng.integers(0, 2500, (n, 176, 176)).astype(np.uint16)
    return dict(rgbA=rgbA, depthA=depthA, rgbB=rgb, depthB=depth, segB=seg, A=Ap, B=B)


def take(t, sel):
    """t[sel] as a contiguous tensor (uint16 rows through an int16 view)"""
    return (t.view(torch.int16)[sel].view(torch.uint16) if t.dtype == torch.uint16 else t[sel]).contiguous()


def same(a, b):
    a, b = (x.view(torch.int16) if x.dtype == torch.uint16 else x for x in (a, b))
    return torch.equal(a, b)


def dev(p, eng):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(eng.device) for k, v in p.items()}


@pytest.fixture(scope='module')
def eng(pkg, synth):
    e = pkg.Engine(max_batch=200)
    e.load_state_dict(synth.make_state_dict(0), 0)
    mean, std = synth.default_mean_std()
    e.set_stats(mean, std, 0)
    yield e
    e.close()


def check_against_oracle(eng, cfg, p, idx, with_seg):
    d = dev(p, eng)
    seg = d['segB'] if with_seg else None
    params, nr, nd = eng.augment_draws(cfg, d['depthB'], idx, segB=seg, want_noise=True)
    r, dp = eng.augment_crops(cfg, d['rgbB'], d['depthB'], idx, segB=seg)
    params, nr, nd, r, dp = (t.cpu().numpy() for t in (params, nr, nd, r, dp))
    for i in range(len(idx)):
        mask = p['segB'][i] if with_seg else (p['depthB'][i] > 100).astype(np.uint8)
        er, ed, _ = R.augment(p['rgbB'][i], p['depthB'][i], mask, params[i], nr[i], nd[i])
        assert np.array_equal(r[i], er), (i, params[i], int((r[i] != er).any(-1).sum()))
        assert np.array_equal(dp[i], ed), (i, params[i], int((dp[i] != ed).sum()))
        if params[i, R.COVER_BRANCH]:
            check_cover(cfg, int(idx[i]), mask, params[i])
    return params


def check_cover(cfg, pair, mask, p):
    """The reference's corner loop over the corners the device drew (replayed on the host) picks the device's corner and
    quadrant after as many corners; when no corner of the cap passes, the device reports quadrant -1 after all of them."""
    used = int(p[R.COVER_CORNERS])
    assert p[R.COVER_VALID] == mask.sum(dtype=np.int64) and 0 < used <= 64
    found = R.cover_search(mask, R.cover_corners(cfg.seed, pair, used))
    if p[R.COVER_QUADRANT] < 0:
        assert used == 64 and found is None
    else:
        assert found == (int(p[R.COVER_U]), int(p[R.COVER_V]), int(p[R.COVER_QUADRANT]), used)


@pytest.mark.parametrize('n', [1, 5, 200])
@pytest.mark.parametrize('with_seg', [True, False])
def test_crops_match_oracle(eng, n, with_seg):
    p = make_pairs(n, seed=n + 10 * with_seg)
    idx = torch.arange(1000, 1000 + n, dtype=torch.int64, device=eng.device)
    params = check_against_oracle(eng, chain(seed=5), p, idx, with_seg)
    if n == 200:                                         # every branch is taken and skipped somewhere in the batch
        for k in (R.HSV_BRANCH, R.NOISE_RGB_BRANCH, R.NOISE_DEPTH_BRANCH, R.BLUR_RGB_BRANCH, R.BLUR_DEPTH_BRANCH, R.COVER_BRANCH):
            assert 0 < params[:, k].sum() < n, k
        assert set(params[params[:, R.BLUR_RGB_BRANCH] > 0, R.BLUR_RGB_K]) == {3.0, 5.0, 7.0}


@pytest.mark.parametrize('stage', ['hsv', 'bright', 'noise', 'blur', 'cover'])
def test_each_stage_alone(eng, stage):
    E = type(eng)
    kw = dict(hsv=dict(h=15, s=15, v=15, prob=1.0), bright=dict(lo=0.5, hi=1.5), noise=dict(rgb=2, depth=5, prob=1.0),
              blur=dict(max_kernel=6, prob=1.0), cover=dict(prob=1.0))
    cfg = E.augment_config(seed=9, **{stage: kw[stage]})
    p = make_pairs(5, seed=3)
    params = check_against_oracle(eng, cfg, p, torch.arange(5, dtype=torch.int64, device=eng.device), True)
    assert params[:, [R.HSV_ON, R.BRIGHT_ON, R.NOISE_RGB_BRANCH, R.BLUR_RGB_BRANCH, R.COVER_BRANCH][
        ['hsv', 'bright', 'noise', 'blur', 'cover'].index(stage)]].all()


def cover_masks(n):
    """Discs of 1 with a ring of 2 (the ring's 2s add 0.8 of the disc to num_valid), the last four all 255."""
    yy, xx = np.mgrid[:176, :176]
    m = np.zeros((n, 176, 176), np.uint8)
    for i in range(n):
        d2 = (yy - 80 - i % 17) ** 2 + (xx - 95 + i % 13) ** 2
        m[i] = (d2 < 60 ** 2) + ((d2 >= 60 ** 2) & (d2 < 71 ** 2)) * 2
    m[-4:] = 255
    return m


def test_cover_retries_across_corners_and_the_cap(eng):
    """maskB with 2s (num_valid counts them, the keep test does not): whole corners fail and the next one is drawn; an all-255
    maskB keeps no cover at all, so the device stops at the cap and leaves the pair uncovered."""
    n = 100
    p = make_pairs(n, seed=8)
    p['segB'][:] = cover_masks(n)
    p['segB'][-4:] = 255
    cfg = type(eng).augment_config(seed=3, cover=dict(prob=1.0))
    params = check_against_oracle(eng, cfg, p, torch.arange(500, 500 + n, dtype=torch.int64, device=eng.device), True)
    assert (params[:-4, R.COVER_CORNERS] > 1).sum() >= 3 and (params[:-4, R.COVER_QUADRANT] >= 0).all()
    assert (params[-4:, R.COVER_QUADRANT] == -1).all() and (params[-4:, R.COVER_CORNERS] == 64).all()


def test_step_equals_plain_eval_on_its_crops(eng):
    n = 8
    p = make_pairs(n, seed=21)
    d = dev(p, eng)
    idx = torch.arange(40, 40 + n, dtype=torch.int64, device=eng.device)
    cfg = chain(seed=2)
    eng.calibrate_fp8_pairs(d['rgbA'], d['depthA'], d['rgbB'], d['depthB'], d['A'])
    for m in MODES:
        out_r = torch.empty_like(d['rgbB']); out_d = torch.empty_like(d['depthB'])
        got = eng.eval_pairs(d['rgbA'], d['depthA'], d['rgbB'], d['depthB'], d['A'], d['B'], TN, RN, precision=m, want_terms=True,
                             want_labels=True, augment=cfg, segB=d['segB'], pair_index=idx, out_rgbB=out_r, out_depthB=out_d)
        got = [t.clone() for t in got]
        r, dp = eng.augment_crops(cfg, d['rgbB'], d['depthB'], idx, segB=d['segB'])
        assert same(r, out_r) and same(dp, out_d), m
        plain = eng.eval_pairs(d['rgbA'], d['depthA'], out_r, out_d, d['A'], d['B'], TN, RN, precision=m, want_terms=True, want_labels=True)
        for a, b in zip(got, plain):
            assert same(a, b), m
        assert not same(out_r, d['rgbB'])


def test_invariance_seeds_and_graph_replay(pkg, eng):
    n = 8
    p = make_pairs(n, seed=33)
    d = dev(p, eng)
    cfg = chain(seed=4)
    idx = torch.arange(100, 100 + n, dtype=torch.int64, device=eng.device)
    r8, d8 = eng.augment_crops(cfg, d['rgbB'], d['depthB'], idx, segB=d['segB'])
    sel = torch.tensor([6, 1, 3, 0], device=eng.device)            # another batch size and order
    r4, d4 = eng.augment_crops(cfg, take(d['rgbB'], sel), take(d['depthB'], sel), take(idx, sel), segB=take(d['segB'], sel))
    assert same(r4, take(r8, sel)) and same(d4, take(d8, sel))
    other = pkg.Engine(max_batch=16)                               # another max_batch
    r16, _ = other.augment_crops(cfg, d['rgbB'], d['depthB'], idx, segB=d['segB'])
    assert same(r16, r8)
    other.close()
    rs, _ = eng.augment_crops(chain(seed=5), d['rgbB'], d['depthB'], idx, segB=d['segB'])
    assert not same(rs, r8)
    # fp32 loss terms of a pair do not depend on its batch either
    t8 = eng.eval_pairs(d['rgbA'], d['depthA'], d['rgbB'], d['depthB'], d['A'], d['B'], TN, RN, precision='fp32', want_terms=True,
                        augment=cfg, segB=d['segB'], pair_index=idx)[3].clone()
    sel6 = torch.tensor([7, 2, 5, 0, 4, 1], device=eng.device)
    pick = lambda t: take(t, sel6)
    t6 = eng.eval_pairs(*(pick(d[k]) for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A', 'B')), TN, RN, precision='fp32', want_terms=True,
                        augment=cfg, segB=pick(d['segB']), pair_index=pick(idx))[3]
    assert same(t6, take(t8, sel6))
    # one graph across batches: new pair indices in the same buffer replay it, with two launches more than the plain step
    outs = dict(out_trans=torch.empty(n, 3, device=eng.device), out_rot=torch.empty(n, 3, device=eng.device),
                out_sums=torch.empty(2, device=eng.device), out_rgbB=torch.empty_like(d['rgbB']), out_depthB=torch.empty_like(d['depthB']))
    args = [d[k] for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A', 'B')] + [TN, RN]
    eng.eval_pairs(*args, precision='bf16x3', out_trans=outs['out_trans'], out_rot=outs['out_rot'], out_sums=outs['out_sums'])
    plain_launches = eng.last_launch_count()
    buf = idx.clone()
    for start in (0, 500, 9000):
        buf.copy_(torch.arange(start, start + n, dtype=torch.int64, device=eng.device))
        eng.eval_pairs(*args, precision='bf16x3', augment=cfg, segB=d['segB'], pair_index=buf, **outs)
        if start:
            assert eng.last_step_was_graph() and eng.last_launch_count() == plain_launches + 2
        r, _ = eng.augment_crops(cfg, d['rgbB'], d['depthB'], buf.clone(), segB=d['segB'])
        assert same(outs['out_rgbB'], r)


def test_refusals(pkg, eng):
    L = importlib.import_module(PKG + '._lib')
    E = type(eng)
    p = dev(make_pairs(2, seed=1), eng)
    idx = torch.arange(2, dtype=torch.int64, device=eng.device)
    bad = [(E.augment_config(blur=dict(max_kernel=8, prob=0.4)), L.ERR_INVALID, 'outside {3, 5, 7}'),
           (E.augment_config(blur=dict(max_kernel=1, prob=0.4)), L.ERR_INVALID, 'outside {3, 5, 7}'),
           (E.augment_config(hsv=dict(h=15, s=15, v=15, prob=1.5)), L.ERR_INVALID, '[0, 1]'),
           (E.augment_config(noise=dict(rgb=-1, depth=5, prob=0.5)), L.ERR_INVALID, 'noise')]
    dm = E.augment_config(cover=dict(prob=0.2)); dm.depth_missing = 1
    bad.append((dm, L.ERR_UNSUPPORTED, 'DepthMissing'))
    for cfg, code, msg in bad:
        for call in (lambda: eng.augment_draws(cfg, p['depthB'], idx),
                     lambda: eng.eval_pairs(p['rgbA'], p['depthA'], p['rgbB'], p['depthB'], p['A'], p['B'], TN, RN, augment=cfg,
                                            pair_index=idx)):
            with pytest.raises(L.Se3tnError) as e:
                call()
            assert e.value.code == code and msg in str(e.value)
    with pytest.raises(L.Se3tnError) as e:                         # a chain without a stage
        eng.augment_draws(E.augment_config(seed=1), p['depthB'], idx)
    assert e.value.code == L.ERR_INVALID and 'no stage' in str(e.value)
    for call in (lambda: eng.augment_crops(chain(), p['rgbB'], p['depthB'], idx, out_rgbB=p['rgbB']),     # in place
                 lambda: eng.eval_pairs(p['rgbA'], p['depthA'], p['rgbB'], p['depthB'], p['A'], p['B'], TN, RN, augment=chain(),
                                        pair_index=idx, out_depthB=p['depthB']),
                 lambda: eng.augment_crops(chain(), p['rgbB'], p['depthB'], idx, out_rgbB=p['rgbA'],          # outputs overlap
                                           out_depthB=p['rgbA'].view(-1)[:2 * 176 * 176 * 2].view(torch.uint16).view(2, 176, 176))):
        with pytest.raises(L.Se3tnError) as e:
            call()
        assert e.value.code == L.ERR_INVALID and 'overlap' in str(e.value)
    small = pkg.Engine(max_batch=1)
    with pytest.raises(L.Se3tnError) as e:
        small.augment_draws(chain(), p['depthB'], idx)
    assert e.value.code == L.ERR_INVALID
    small.close()
    with pytest.raises(ValueError, match='pair_index'):
        eng.eval_pairs(p['rgbA'], p['depthA'], p['rgbB'], p['depthB'], p['A'], p['B'], TN, RN, augment=chain())


def test_draw_statistics(eng):
    """>= 10^5 pairs: every branch frequency within 5 sigma of its probability, the magnitudes uniform (KS), k even over
    {3, 5, 7}, the noise N(0, std), and BlackCover never at its cap."""
    N, n = 100_000, 200
    depth = torch.full((n, 176, 176), 1000, dtype=torch.uint16, device=eng.device)
    cfg = chain(seed=11)
    ps = []
    for s in range(0, N, n):
        ps.append(eng.augment_draws(cfg, depth, torch.arange(s, s + n, dtype=torch.int64, device=eng.device))[0].cpu().numpy())
    P = np.concatenate(ps)
    for k, prob in ((R.HSV_BRANCH, .5), (R.HSV_BRANCH + 1, .5), (R.HSV_BRANCH + 2, .5), (R.NOISE_RGB_BRANCH, .5),
                    (R.NOISE_DEPTH_BRANCH, .5), (R.BLUR_RGB_BRANCH, .4), (R.BLUR_DEPTH_BRANCH, .4), (R.COVER_BRANCH, .2)):
        assert abs(P[:, k].mean() - prob) <= 5 * np.sqrt(prob * (1 - prob) / N), k
    for k, lo, hi in ((R.HSV_MAG, -15, 15), (R.HSV_MAG + 1, -15, 15), (R.HSV_MAG + 2, -15, 15), (R.BRIGHT, .5, 1.5),
                      (R.NOISE_RGB_STD, 0, 2), (R.NOISE_DEPTH_STD, 0, 5)):
        assert stats.kstest(P[:, k], 'uniform', args=(lo, hi - lo)).pvalue > 1e-4, k
    for k in (R.BLUR_RGB_K, R.BLUR_DEPTH_K):
        counts = np.array([(P[:, k] == v).sum() for v in (3, 5, 7)])
        assert counts.sum() == N and (np.abs(counts - N / 3) <= 5 * np.sqrt(N * 2 / 9)).all()
    cov = P[P[:, R.COVER_BRANCH] > 0]
    assert (cov[:, R.COVER_QUADRANT] >= 0).all() and cov[:, R.COVER_CORNERS].max() < 64
    for k in (R.COVER_U, R.COVER_V):
        assert stats.kstest(cov[:, k] + 0.5, 'uniform', args=(0, 176)).pvalue > 1e-4
    # the noise fields: N(0, std) with the drawn std
    params, nr, nd = eng.augment_draws(cfg, depth, torch.arange(n, dtype=torch.int64, device=eng.device), want_noise=True)
    params = params.cpu().numpy()
    for field, k in ((nr, R.NOISE_RGB_STD), (nd, R.NOISE_DEPTH_STD)):
        f = field.cpu().numpy().reshape(n, -1)
        z = (f / params[:, k:k + 1]).ravel()
        M = z.size
        assert abs(z.mean()) <= 5 / np.sqrt(M) and abs(z.var() - 1) <= 5 * np.sqrt(2 / M)


def write_folder(d, p):
    os.makedirs(d, exist_ok=True)
    for i in range(len(p['A'])):
        stem = os.path.join(d, '%05d' % i)
        cv2.imwrite(stem + 'rgbA.png', cv2.cvtColor(p['rgbA'][i], cv2.COLOR_RGB2BGR))
        cv2.imwrite(stem + 'rgbB.png', cv2.cvtColor(p['rgbB'][i], cv2.COLOR_RGB2BGR))
        cv2.imwrite(stem + 'depthA.png', p['depthA'][i]); cv2.imwrite(stem + 'depthB.png', p['depthB'][i])
        if i % 3:                                        # some pairs without segB: maskB = depthB > 100
            cv2.imwrite(stem + 'segB.png', p['segB'][i])
        np.savez(stem + 'meta.npz', A_in_cam=p['A'][i], B_in_cam=p['B'][i])


def test_problem_validate_and_cli_equal_engine_level(pkg, eng, synth, tmp_path, capsys):
    P = importlib.import_module(PKG + '.problems')
    D = importlib.import_module(PKG + '.datasets')
    n = 13
    p = make_pairs(n, seed=44)
    folder = str(tmp_path / 'val')
    write_folder(folder, p)
    mean, std = synth.default_mean_std()
    info = {'resolution': 176, 'max_translation': TN, 'max_rotation': 15,
            'camera': {'focalX': 1066.778, 'focalY': 1067.487, 'centerX': 312.9869, 'centerY': 241.3109}}
    ds = D.TrackDataset(folder, 'val', mean, std, None, A().from_config(REF_CONFIG), None, dataset_info=info, trans_normalizer=TN,
                        rot_normalizer=RN, engine=eng, augment_seed=7)
    cfg = chain(seed=7)
    d = dev(p, eng)
    seg_host = np.where((np.arange(n) % 3 != 0)[:, None, None], p['segB'], (p['depthB'] > 100).astype(np.uint8))
    seg = torch.from_numpy(np.ascontiguousarray(seg_host)).to(eng.device)
    idx = torch.arange(n, dtype=torch.int64, device=eng.device)
    rB, dB = eng.augment_crops(cfg, d['rgbB'], d['depthB'], idx, segB=seg)
    params = eng.augment_draws(cfg, d['depthB'], idx, segB=seg)[0].cpu().numpy()
    for i in (0, 1, 5):                                  # __getitem__: the augmented rgbB and maskB of the 8-tuple
        item = ds[i]
        assert np.array_equal(item[5], rB[i].cpu().numpy())
        mask = seg[i].cpu().numpy().copy()
        if params[i, R.COVER_BRANCH]:
            mask[R.cover_slices(*(int(params[i, k]) for k in (R.COVER_U, R.COVER_V, R.COVER_QUADRANT)))] = 0
        assert np.array_equal(item[7], mask)
    model = pkg.Se3TrackNet(engine=eng, weight_id=0)
    model.load_state_dict(synth.make_state_dict(0))
    loader = torch.utils.data.DataLoader(ds, batch_size=5, shuffle=False)
    prob = P.Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}})
    for m in ('fp32', 'bf16x3'):
        r = prob.validation_losses(m, keep_predictions=True)
        sums, preds = [], []
        for s in range(0, n, 5):
            e = min(n, s + 5)
            tr, ro, sm, _, _ = eng.eval_pairs(*(d[k][s:e] for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A', 'B')), TN, RN, precision=m,
                                              augment=cfg, segB=seg[s:e].contiguous(), pair_index=idx[s:e].contiguous())
            sums.append(sm.cpu().numpy()); preds.append(torch.cat((tr, ro), 1).cpu().numpy())
        assert np.array_equal(r['predictions'], np.concatenate(preds)), m
        bt, br = P.batch_means(np.stack(sums), P.batch_plan(n, 5, 5))
        assert np.array_equal(r['batch_trans'], bt) and np.array_equal(r['batch_rot'], br), m
    # fp8: the scales come from the first batch as the steps see it, augmented
    eng2 = pkg.Engine(max_batch=8)
    m2 = pkg.Se3TrackNet(engine=eng2, weight_id=0)
    m2.load_state_dict(synth.make_state_dict(0))
    P.evaluate(m2, ds, 5, precision='fp8')
    got = eng2.fp8_scales(0)
    eng2.load_state_dict(synth.make_state_dict(0), 0)               # drops the scales
    r5, d5 = eng2.augment_crops(cfg, d['rgbB'][:5], d['depthB'][:5], idx[:5].contiguous(), segB=seg[:5].contiguous())
    eng2.calibrate_fp8_pairs(d['rgbA'][:5], d['depthA'][:5], r5, d5, d['A'][:5])
    assert np.array_equal(got, eng2.fp8_scales(0))
    eng2.close()
    # the command line: the same numbers, labelled as augmented
    ck = tmp_path / 'ck'; ck.mkdir()
    torch.save({'state_dict': synth.make_state_dict(0)}, str(ck / 'model.pth.tar'))
    np.save(str(ck / 'mean.npy'), mean); np.save(str(ck / 'std.npy'), std)
    with open(ck / 'info.yml', 'w') as f:
        yaml.safe_dump(info, f)
    with open(ck / 'config.yml', 'w') as f:
        yaml.safe_dump(REF_CONFIG, f)
    P.main(['--val_dir', folder, '--ckpt', str(ck / 'model.pth.tar'), '--mean_std_path', str(ck), '--dataset_info', str(ck / 'info.yml'),
            '--augment', str(ck / 'config.yml'), '--seed', '7', '--batch_size', '5', '--precision', 'fp32'])
    out = capsys.readouterr().out
    assert 'augmented' in out
    r = prob.validation_losses('fp32')
    assert ('%14.8g' % r['trans']) in out
