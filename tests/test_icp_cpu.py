"""The depth refinement without a GPU: se3tn_icp_opts in include/se3tn.h against _lib.IcpOpts,
oracle/icp_ref.py's Jacobian against central finite differences, its convergence on synthetic frames (which sets the bounds the
GPU test holds the kernels to), and Engine.icp_spec's parsing."""
import ctypes as C
import importlib
import os
import re
import sys
import numpy as np
import pytest

PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import icp_ref  # noqa: E402
import se3_oracle as so  # noqa: E402

# what the zero-head test on the GPU requires after 10 iterations from starts perturbed by 5-10 mm and 2-5 degrees (the
# oracle below lands at 0.6-0.9 mm and at most 0.2 degrees; the pyrender-drawn frames sample each pixel's ray half a pixel off
# K^-1 (p_x, p_y, 1), which leaves a bias of that order besides the 1 mm depth quantisation).  The solve is an undamped
# Gauss-Newton step: on synthetic_scene(seed=5) one start of eight (8.7 mm, 4.2 degrees) overshoots in its first iteration and
# ends 47 mm away, in the oracle exactly as on the GPU.
ADD_BOUND_MM = 1.5
ROT_BOUND_DEG = 0.5
H, W = 480, 640


def _header():
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)


def test_icp_opts_matches_the_header():
    m = re.search(r'\bstruct\s+se3tn_icp_opts\s*\{([^}]*)\}\s*se3tn_icp_opts\s*;', _header())
    assert m, 'struct se3tn_icp_opts is not defined'
    fields = []
    for decl in filter(None, (d.strip() for d in m.group(1).split(';'))):
        typ, names = decl.split(None, 1)
        assert typ == 'int32_t'
        fields += [(name.strip(), C.c_int32) for name in names.split(',')]
    L = importlib.import_module(PKG + '._lib')
    assert L.IcpOpts._fields_ == fields
    assert [f[0] for f in fields] == ['iterations', 'tau_mm', 'min_inliers', 'reserved'] and C.sizeof(L.IcpOpts) == 16
    src = open(os.path.join(ROOT, 'include', 'se3tn.h')).read()
    assert int(re.search(r'#define SE3TN_MAX_ICP_ITERATIONS (\d+)', src).group(1)) == L.MAX_ICP_ITERATIONS
    assert int(re.search(r'#define SE3TN_ICP_COLS (\d+)', src).group(1)) == L.ICP_COLS


def test_jacobian_matches_central_differences():
    rng = np.random.default_rng(0)
    for _ in range(20):
        n = rng.normal(size=3); n /= np.linalg.norm(n)
        q = rng.normal(size=3) * 0.05 + np.array([0, 0, 0.7])
        o = q + rng.normal(size=3) * 0.004
        J = icp_ref.jacobian(q, n)[0]
        h = 1e-6
        fd = np.array([(icp_ref.residual(h * np.eye(6)[k], q, n, o) - icp_ref.residual(-h * np.eye(6)[k], q, n, o)) / (2 * h)
                       for k in range(6)])
        assert np.allclose(fd, J, rtol=1e-6, atol=1e-6 * np.abs(J).max())


def test_solve_skips_keep_the_pose():
    pose = np.eye(4); pose[2, 3] = 0.7
    S = np.zeros(29)
    assert icp_ref.solve(S, pose, 6)[0] is pose                        # no inliers
    S[28] = 50.0
    for k in (0, 6, 11, 15, 18, 20):                                   # the diagonal of J^T J
        S[k] = 1.0
    assert icp_ref.solve(S, pose, 100)[0] is pose                      # count < min_inliers
    out, st = icp_ref.solve(S, pose, 6)
    assert out is not pose and st[0] == 50 and st[2] == 0 and st[3] == 0   # J^T e = 0: no motion
    S[20] = 1e-13                                                      # a pivot below 1e-12 x the largest diagonal entry
    assert icp_ref.solve(S, pose, 6)[0] is pose


synthetic_scene = icp_ref.synthetic_scene


def errors(synth, pose, gt):
    """-> (ADD mm on synth.model_points, rotation error degrees)."""
    pts = synth.model_points()
    add = np.linalg.norm(pts @ pose[:3, :3].T + pose[:3, 3] - pts @ gt[:3, :3].T - gt[:3, 3], axis=1).mean() * 1000
    rot = np.degrees(np.arccos(np.clip((np.trace(pose[:3, :3].T @ gt[:3, :3]) - 1) / 2, -1, 1)))
    return add, rot


def test_oracle_converges_on_synthetic_frames(synth):
    mesh, gts, starts, D = synthetic_scene(synth, 8)                     # the GPU test's scene
    for P, S in zip(gts, starts):
        poses, stats = icp_ref.icp(S, synth.CAMERA_K, 200.0, mesh, D, 20, 100, 10, 'pyrender', H, W)
        add, rot = errors(synth, poses[-1], P)
        assert add <= ADD_BOUND_MM and rot <= ROT_BOUND_DEG, (add, rot)
        assert errors(synth, S, P)[0] > 4 * add
        assert stats[-1, 2] < stats[0, 2] and stats[-1, 3] < stats[0, 3] and stats[-1, 0] >= 100


def test_icp_spec():
    E = importlib.import_module(PKG + '.engine').Engine
    assert E.icp_spec(None) is None and E.icp_spec(0) is None
    o = E.icp_spec(3)
    assert (o.iterations, o.tau_mm, o.min_inliers, o.reserved) == (3, E.ICP_TAU_DEFAULT, E.ICP_MIN_INLIERS_DEFAULT, 0)
    o = E.icp_spec({'iterations': 16, 'tau_mm': 1000, 'min_inliers': 6})
    assert (o.iterations, o.tau_mm, o.min_inliers) == (16, 1000, 6)
    for bad in (17, -1, True, 2.0, '3', {'iterations': 2, 'tau': 3}, {'tau_mm': 5}, {'iterations': 1, 'min_inliers': 5},
                {'iterations': 1, 'tau_mm': 1001}, {'iterations': 1, 'min_inliers': 176 * 176 + 1}):
        with pytest.raises(ValueError, match='icp'):
            E.icp_spec(bad)
