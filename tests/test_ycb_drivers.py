"""Host logic of the YCB-Video drivers (reference predict.py:89-123, 299-575): initialisation sources, keyframe search, data-set
layout discovery, mesh vertex merging.  CPU only; the tracked poses themselves are checked on the GPU (test_gpu_parity.py)."""
import importlib, os
import numpy as np
import pytest


@pytest.fixture(scope='module')
def pr():
    return importlib.import_module('iros20-6d-pose-tracking_b200.predict')


def test_quaternion_matrix_matches_scipy_and_identity(pr):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(0)
    for _ in range(20):
        q = rng.normal(size=4)                                       # (w, x, y, z), not normalised: transformations.py normalises
        R = pr.quaternion_matrix3(q)
        ref = Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix()
        assert np.abs(R - ref).max() < 1e-12
    assert np.array_equal(pr.quaternion_matrix3([1, 0, 0, 0]), np.eye(3))
    assert np.array_equal(pr.quaternion_matrix3([0, 0, 0, 0]), np.eye(3))      # degenerate: identity, as transformations.py


def test_nearest_keyframe_searches_outwards(pr):
    kf = ['0048/000001', '0048/000036', '0048/000047', '0049/000010']
    assert pr.nearest_keyframe(kf, 48, 36) == ('0048/000036', 1, 36)
    assert pr.nearest_keyframe(kf, 48, 40)[2] == 36                  # 4 below beats 7 above
    assert pr.nearest_keyframe(kf, 48, 43)[2] == 47
    assert pr.nearest_keyframe(kf, 49, 0) == ('0049/000010', 3, 10)
    with pytest.raises(ValueError):
        pr.nearest_keyframe(kf, 50, 5)


def test_posecnn_result_file_and_reinit_lookup(pr, tmp_path):
    import scipy.io
    ycb = tmp_path / 'ycb'
    (ycb / 'image_sets').mkdir(parents=True)
    (ycb / 'YCB_Video_toolbox' / 'results_PoseCNN_RSS2018').mkdir(parents=True)
    (ycb / 'image_sets' / 'keyframe.txt').write_text('0048/000001\n0048/000011\n0049/000001\n')
    q = np.array([0.5, 0.5, -0.5, 0.5]); t = np.array([0.1, -0.2, 0.8])
    rois = np.zeros((2, 6)); rois[0, 1] = 3; rois[1, 1] = 7
    poses_icp = np.stack([np.r_[1.0, 0, 0, 0, 0, 0, 1], np.r_[q, t]])
    scipy.io.savemat(str(ycb / 'YCB_Video_toolbox' / 'results_PoseCNN_RSS2018' / '000001.mat'), {'rois': rois, 'poses_icp': poses_icp})
    pose = pr.use_posecnn_res(7, '0048/000009', str(ycb))            # nearest keyframe of 9 is 11 = index 1
    assert np.allclose(pose[:3, 3], t) and np.allclose(pose[:3, :3], pr.quaternion_matrix3(q)) and np.array_equal(pose[3], [0, 0, 0, 1])
    with pytest.raises(ValueError):
        pr.use_posecnn_res(5, '0048/000009', str(ycb))               # class not detected in that frame


def test_find_class_videos_and_poserbpf(pr, tmp_path):
    data = tmp_path / 'data_organized'
    for seq, classes in ((47, [4]), (48, [4, 9]), (50, [9]), (59, [4]), (60, [4])):
        for c in classes:
            (data / ('%04d' % seq) / 'pose_gt' / str(c)).mkdir(parents=True)
    assert pr.findClassContainedVideosYcb(4, str(data), testset=True) == [48, 59]
    assert pr.findClassContainedVideosYcb(4, str(data), testset=False) == [47, 48, 59, 60]
    assert pr.findClassContainedVideosYcb(9, str(data)) == [48, 50]
    res = tmp_path / 'YCB_Video_toolbox' / 'PoseRBPF_Results' / 'YCB_results_RGBD'
    for k in range(1, 5):
        (res / ('%02d_obj' % k) / 'seq_2').mkdir(parents=True)
    (res / '04_obj' / 'seq_2' / 'Pose_x.txt').write_text('1 4 0.1 0.2 0.9 1 0 0 0\n5 4 0 0 0 1 0 0 0\n')
    pose = pr.poserbpf_pose(str(tmp_path), 4, 59, [48, 59])
    assert np.allclose(pose[:3, 3], [0.1, 0.2, 0.9]) and np.allclose(pose[:3, :3], np.eye(3))


def test_load_vertices_merges_duplicates_like_trimesh(pr, tmp_path):
    """ADVICE r1: trimesh.load(process=True) merges duplicate vertices before the reference voxel-down-samples them."""
    pts = np.array([[0, 0, 0], [0.01, 0, 0], [0, 0.01, 0], [0.01, 0, 0], [0, 0, 0.02], [0, 0, 0]], dtype=np.float64)
    ply = tmp_path / 'dup.ply'
    with open(ply, 'w') as f:
        f.write('ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nend_header\n' % len(pts))
        for p in pts:
            f.write('%g %g %g\n' % tuple(p))
    merged = pr.load_vertices(str(ply))
    assert merged.shape == (4, 3) and np.allclose(merged, pts[[0, 1, 2, 4]])           # first occurrences, file order
    assert pr.load_vertices(str(ply), merge=False).shape == (6, 3)
    obj = tmp_path / 'dup.obj'
    obj.write_text(''.join('v %g %g %g\n' % tuple(p) for p in pts) + 'f 1 2 3\n')
    assert np.allclose(pr.load_vertices(str(obj)), merged)
    # the duplicates would have shifted the voxel means (0.005 m voxels: points 1 and 3 share a voxel only with each other)
    a = pr.PointCloud(merged).voxel_down_sample(0.005).points
    b = pr.PointCloud(pts).voxel_down_sample(0.005).points
    assert a.shape == b.shape and np.allclose(np.sort(a, 0), np.sort(b, 0))            # same voxels here; means of identical points are unchanged

