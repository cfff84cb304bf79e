"""CPU-only: the validation pass's host logic -- pair discovery and naming, __len__, the batch arithmetic of Problem.validate
(the mean of per-batch means, the partial last batch, batches cut into device steps) -- and the new entry points' header
declarations against the ctypes binding."""
import importlib, os, re
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = 'iros20-6d-pose-tracking_b200'


def _write_pair(d, stem, size=176, seg=True, seed=0):
    import cv2
    rng = np.random.default_rng(seed)
    for name in ('rgbA', 'rgbB'):
        cv2.imwrite(os.path.join(d, stem + name + '.png'), rng.integers(0, 256, (size, size, 3), dtype=np.uint8))
    for name in ('depthA', 'depthB'):
        cv2.imwrite(os.path.join(d, stem + name + '.png'), rng.integers(300, 1800, (size, size)).astype(np.uint16))
    if seg:
        cv2.imwrite(os.path.join(d, stem + 'segB.png'), (rng.random((size, size)) > 0.5).astype(np.uint8))
    A = np.eye(4); A[2, 3] = 0.6
    B = A.copy(); B[0, 3] += 0.01
    np.savez(os.path.join(d, stem + 'meta.npz'), A_in_cam=A, B_in_cam=B)
    return A, B


def test_file_discovery_naming_and_len(tmp_path):
    D = importlib.import_module(PKG + '.datasets')
    d = tmp_path / 'A_val_A'                          # 'A' in the directory: only the basename is rewritten
    d.mkdir()
    for i in (3, 1, 2):
        _write_pair(str(d), '%06d' % i, seg=(i != 2), seed=i)
    ds = D.TrackDataset(str(d), 'val', np.zeros(8, np.float32), np.ones(8, np.float32), dataset_info={
        'resolution': 176, 'camera': {'focalX': 1, 'focalY': 1, 'centerX': 0, 'centerY': 0}})
    assert len(ds) == 3
    assert [os.path.basename(f) for f in ds.rgbA_files] == ['000001rgbA.png', '000002rgbA.png', '000003rgbA.png']
    p = D.pair_paths(ds.rgbA_files[0])
    assert p['rgbB'] == os.path.join(str(d), '000001rgbB.png') and p['meta'] == os.path.join(str(d), '000001meta.npz')
    assert p['depthA'].endswith('000001depthA.png') and p['depthB'].endswith('000001depthB.png') and p['segB'].endswith('000001segB.png')
    pair = D.read_pair(ds.rgbA_files[1])
    assert pair['segB'] is None                       # optional, as cv2.imread's None in the reference
    assert pair['rgbA'].shape == (176, 176, 3) and pair['rgbA'].dtype == np.uint8
    assert pair['depthB'].dtype == np.uint16 and pair['A_in_cam'].shape == (4, 4)
    import cv2
    raw = cv2.imread(ds.rgbA_files[1], cv2.IMREAD_COLOR)
    assert np.array_equal(pair['rgbA'], raw[..., ::-1])   # RGB order, as PIL gives the reference
    assert len(D.TrackDataset(str(tmp_path / 'empty'), 'val', np.zeros(8), np.ones(8))) == 0


@pytest.mark.parametrize('n,bs,cap,drop', [(450, 200, 64, False), (450, 200, 200, False), (400, 200, 256, False), (450, 200, 64, True), (7, 3, 2, False)])
def test_batch_plan_covers_the_loader_batches(n, bs, cap, drop):
    P = importlib.import_module(PKG + '.problems')
    steps = P.batch_plan(n, bs, cap, drop)
    n_batches = n // bs if drop else -(-n // bs)
    assert steps[-1][0] == n_batches - 1
    covered = []
    for b, s, e in steps:
        assert 0 < e - s <= cap and b * bs <= s < e <= min(n, (b + 1) * bs)
        covered += list(range(s, e))
    assert covered == list(range(n_batches * bs if drop else n))


def test_batch_means_is_the_mean_of_per_batch_means():
    """problems.py:122-129 on a DataLoader(batch_size=200, drop_last=False): a partial last batch counts as one batch."""
    P = importlib.import_module(PKG + '.problems')
    rng = np.random.default_rng(0)
    n, bs, cap = 450, 200, 64
    sq = rng.random((n, 6)).astype(np.float32)
    steps = P.batch_plan(n, bs, cap)
    step_sums = np.array([[sq[s:e, :3].sum(dtype=np.float64), sq[s:e, 3:].sum(dtype=np.float64)] for _, s, e in steps], dtype=np.float32)
    bt, br = P.batch_means(step_sums, steps)
    assert bt.dtype == np.float32 and len(bt) == 3
    ref_t = [sq[b0:b0 + bs, :3].mean(dtype=np.float64) for b0 in range(0, n, bs)]
    ref_r = [sq[b0:b0 + bs, 3:].mean(dtype=np.float64) for b0 in range(0, n, bs)]
    np.testing.assert_allclose(bt, ref_t, rtol=1e-6)
    np.testing.assert_allclose(br, ref_r, rtol=1e-6)
    assert P._mean_over_batches(bt) == pytest.approx(np.mean(ref_t), rel=1e-6)
    # a batch cut into steps adds their float32 sums in order, then divides by its 3 x pairs elements in float32
    t0 = np.float32(0)
    for (b, s, e), v in zip(steps, step_sums):
        if b == 0:
            t0 = np.float32(t0 + v[0])
    assert bt[0] == np.float32(t0 / np.float32(600))


def test_rgb_crops_must_be_8bit_three_channel(tmp_path):
    """The reference's PIL would return an RGBA, grayscale or 16-bit rgb crop as an array of another shape or depth, which
    processData does not handle: read_pair rejects such files instead of converting them."""
    import cv2
    D = importlib.import_module(PKG + '.datasets')
    for i, bad in enumerate((np.zeros((176, 176, 4), np.uint8), np.zeros((176, 176), np.uint8), np.zeros((176, 176, 3), np.uint16))):
        d = tmp_path / str(i)
        d.mkdir()
        _write_pair(str(d), '000000')
        cv2.imwrite(str(d / '000000rgbB.png'), bad)
        with pytest.raises(ValueError, match='8-bit three-channel'):
            D.read_pair(str(d / '000000rgbA.png'))


def test_training_is_refused():
    P = importlib.import_module(PKG + '.problems')
    prob = P.Problem.__new__(P.Problem)
    with pytest.raises(NotImplementedError):
        prob.train(0)
    with pytest.raises(NotImplementedError):
        prob.loop(1, '/nonexistent')


def _decl(src, name):
    m = re.search(r'\bint\s+' + name + r'\s*\(([^)]*)\)\s*;', src)
    assert m, name + ' is not declared'
    return [p.strip() for p in m.group(1).split(',')]


def test_validation_entry_points_declared_and_bound():
    src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)
    L = importlib.import_module(PKG + '._lib')
    kinds = {'se3tn_ctx*': L._vp, 'int': L._i, 'double': L._d, 'void*': L._vp}
    for name in ('se3tn_eval_pairs', 'se3tn_pair_loss'):
        params = _decl(src, name)
        res, args = L.SIGNATURES[name]
        assert res is L._i and len(args) == len(params)
        for p, a in zip(params, args):
            t = p.rsplit(None, 1)[0].replace('const ', '').replace(' *', '*')
            assert a is (L._vp if t.endswith('*') else kinds[t]), (name, p)
    assert int(re.search(r'SE3TN_PROFILE_SLOTS\s+(\d+)', src).group(1)) == L.PROFILE_SLOTS
