"""The pair generator's host half (produce_train_pair_data.py) without a device: the seeded perturbation draws against the
reference's own Utils (golden_pairs.npz, oracle/make_golden_pairs.py), the oracle's seg crop against the reference's crop_bbox, the
visibility thresholds, and completeBlender's validation split and file names."""
import importlib, os, random
import numpy as np
import pytest

import pairs_oracle as PO

PKG = 'iros20-6d-pose-tracking_b200'


@pytest.fixture(scope='module')
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'golden_pairs.npz'))


@pytest.fixture(scope='module')
def U():
    return importlib.import_module(PKG + '.Utils')


@pytest.fixture(scope='module')
def PP():
    return importlib.import_module(PKG + '.produce_train_pair_data')


def test_random_gaussian_magnitude_matches_reference(golden, U):
    for seed, mt, mr, k in golden['rng_cases']:
        seed, k = int(seed), int(k)
        for fn in (U.random_gaussian_magnitude, PO.random_gaussian_magnitude):
            random.seed(seed); np.random.seed(seed)
            got = np.stack([fn(mt, mr) for _ in range(k)])
            assert np.array_equal(got, golden['rgm_%d' % seed]), (fn.__module__, seed)
        random.seed(seed)
        assert np.array_equal(np.stack([U.random_direction() for _ in range(k)]), golden['dir_%d' % seed])


def test_oracle_seg_crop_matches_reference(golden, synth):
    rgb, depth = synth.raw_frame(3, 120, 160)
    seg = golden['seg']
    for i in range(int(golden['n_crops'])):
        r, d, s = PO.crop_bbox_seg(rgb, depth, golden['crop_bb_%d' % i], (176, 176), seg)
        assert np.array_equal(r, golden['crop_rgb_%d' % i]), i
        assert np.array_equal(d, golden['crop_depth_%d' % i]), i
        assert np.array_equal(s, golden['crop_seg_%d' % i]) and s.dtype == np.uint8, i


def test_visibility_thresholds(PP):
    assert not PP.visible_enough(100, 50)                   # num_visible <= 100
    assert PP.visible_enough(101, 1000)                     # 0.101
    assert not PP.visible_enough(101, 1011)                 # 0.0999
    assert PP.visible_enough(500, 0)                        # inf: kept, as numpy's scalar division gives it
    for v, c in ((101, 1010), (150, 1500), (3000, 7)):
        assert PP.visible_enough(v, c) == PO.visible_enough(v, c)


def test_draw_order_matches_oracle(PP, synth):
    """ProducerPurturb.draw consumes the RNG as the reference's loop: the same A_in_cam sequence and centre verdicts as the oracle."""
    K = synth.CAMERA_K.copy(); K[:2] *= 0.25
    info = {'max_translation': 0.06, 'max_rotation': 20.0, 'camera': {'focalX': K[0, 0], 'focalY': K[1, 1], 'centerX': K[0, 2],
                                                                        'centerY': K[1, 2], 'height': 120, 'width': 160}}
    stub = type('P', (), {})()
    stub.dataset_info = info; stub.cam_K = PP._cam_K32(info)
    B = synth.raw_poses(1, seed=3)[0]; B[:3, 3] = (-0.13, 0.0, 0.5)
    random.seed(4); np.random.seed(4)
    got = PP.ProducerPurturb.draw(stub, B, 30)
    random.seed(4); np.random.seed(4)
    want = []
    for _ in range(30):
        A = B.dot(np.linalg.inv(PO.random_gaussian_magnitude(0.06, 20.0)))
        p = stub.cam_K.dot(A[:3, 3].reshape(3, 1)).reshape(-1)
        u, v = p[0] / p[2], p[1] / p[2]
        want.append((A, not (u < 0 or u >= 160 or v < 0 or v >= 120)))
    assert all(np.array_equal(a, b) and f == g for (a, f), (b, g) in zip(got, want))
    assert any(f for _, f in got) and not all(f for _, f in got)


def test_blender_split_and_names(PP, tmp_path):
    """completeBlender's validation split: the val_samples last pairs in name order, newest first, renumbered from 0; the names
    are rewritten in the basename only, so a folder with an 'A' in its path keeps it."""
    train = str(tmp_path / 'A_set' / 'train_data_blender_DR') + '/'
    val = str(tmp_path / 'A_set' / 'validation_data_blender_DR') + '/'
    os.makedirs(train); os.makedirs(val)
    kinds = ('rgbA.png', 'rgbB.png', 'depthA.png', 'depthB.png', 'meta.npz', 'segB.png')
    for i in range(5):
        for k in kinds:
            with open(train + '%07d%s' % (i, k), 'w') as f:
                f.write('%d %s' % (i, k))
    PP.split_validation(train, val, 2)
    assert sorted(os.listdir(val)) == sorted('%07d%s' % (i, k) for i in range(2) for k in kinds)
    for i, src in ((0, 4), (1, 3)):
        for k in kinds:
            assert open(val + '%07d%s' % (i, k)).read() == '%d %s' % (src, k)
    assert sorted(os.listdir(train)) == sorted('%07d%s' % (i, k) for i in range(3) for k in kinds)
    with pytest.raises(ValueError, match='val_samples'):
        PP.split_validation(train, val, 4)
    assert PP._sub('/d/rgbA_dir/0001rgb.png', 'rgb', 'depth') == '/d/rgbA_dir/0001depth.png'


def test_blender_pose(PP, synth):
    """B_in_cam of a Blender frame (produce_train_pair_data.py:196-200): inv(cvcam_in_blendercam) . inv(cam_in_world) . ob_in_world."""
    P = synth.raw_poses(3, seed=1)
    cam = synth.raw_poses(1, seed=2)[0]
    meta = {'class_ids': np.array([2, 0, 1]), 'poses_in_world': P, 'blendercam_in_world': cam}
    want = np.linalg.inv(PP.GLCAM_IN_CVCAM).dot(np.linalg.inv(cam).dot(P[1]))
    assert np.array_equal(PP._blender_B_in_cam(meta, 0), want)


def test_cli_refuses_missing_arguments(PP):
    with pytest.raises(SystemExit):
        PP.main(['--mode', 'blender'])
    with pytest.raises(SystemExit):
        PP.main(['--mode', 'ycbv', '--ycb_dir', 'x'])
