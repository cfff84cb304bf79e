"""Pins oracle/se3_oracle.py against fixtures produced by the reference's own code
(oracle/make_golden.py, run in the build container).  CPU only."""
import hashlib, os
import numpy as np
import cv2
import torch
import se3_oracle as O


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_model_forward_matches_reference(synth, golden_dir):
    g = np.load(os.path.join(golden_dir, 'golden_model.npz'))
    sd = synth.make_state_dict(0)
    A, B = synth.tensor_pairs(2, seed=0)
    out, inter = O.forward(sd, A, B, return_intermediates=True)
    # same library, same ops, same order -> bit-identical
    assert np.array_equal(out['trans'].numpy(), g['trans'])
    assert np.array_equal(out['rot'].numpy(), g['rot'])
    assert sha(out['feature'].numpy()) == str(g['feature_sha'])
    names = dict(convA1='a1', poolA1='a1p', convA2='a2', convB1='b1', poolB1='b1p', convB2='b2',
                 convB3='b3', convAB1='ab1', convAB2='ab2', trans_conv1='trans1',
                 trans_conv2='trans2', rot_conv1='rot1', rot_conv2='rot2')
    for ref_name, mine in names.items():
        assert np.array_equal(inter[mine][:, ::8, ::5, ::5].numpy(), g['act_' + ref_name + '_sub']), ref_name


def test_config1_end_to_end(synth, golden_dir):
    g = np.load(os.path.join(golden_dir, 'golden_model.npz'))
    rgbA = cv2.imread(os.path.join(golden_dir, 'c1_rgbA.png'))[..., ::-1].copy()
    rgbB = cv2.imread(os.path.join(golden_dir, 'c1_rgbB.png'))[..., ::-1].copy()
    depthA, depthB = synth.depth_from_rgb(rgbA), synth.depth_from_rgb(rgbB)
    mean, std = synth.default_mean_std()
    pose = synth.config1_pose()
    (dA, dB), _ = O.process_data(rgbA, depthA, pose, rgbB, depthB, np.eye(4), mean, std)
    assert sha(dA) == str(g['c1_dataA_sha']) and sha(dB) == str(g['c1_dataB_sha'])
    sd = synth.make_state_dict(0)
    out = O.forward(sd, torch.from_numpy(dA)[None], torch.from_numpy(dB)[None])
    assert np.array_equal(out['trans'].numpy(), g['c1_trans'])
    assert np.array_equal(out['rot'].numpy(), g['c1_rot'])
    pose_out = O.process_predict(pose, (out['trans'][0].numpy(), out['rot'][0].numpy()))
    assert np.array_equal(pose_out, g['c1_pose_out'])


def test_bbox_and_crop_small_frame(synth, golden_dir):
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    rgb, depth, K = p['small_rgb'], p['small_depth'], p['K_small']
    n = len(p['object_width'])
    for i in range(n):
        bb = O.compute_bbox(p['poses'][i], K, p['object_width'][i], scale=(1000, 1000, 1000))
        assert bb.dtype == np.int32 and np.array_equal(bb, p[f'bb_{i}'])
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        assert rB.dtype == np.uint8 and dB.dtype == np.uint16
        assert sha(rB) == str(p[f'rgbB_sha_{i}']) and sha(dB) == str(p[f'depthB_sha_{i}']), i
        if i < 2:
            assert np.array_equal(rB, p[f'rgbB_{i}']) and np.array_equal(dB, p[f'depthB_{i}'])
    bb = O.compute_bbox(p['poses'][1], K, 200., scale=(1000, -1000, 1000))
    assert np.array_equal(bb, p['bb_gl_0'])


def test_crop_full_frame(synth, golden_dir):
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    rgb, depth = synth.raw_frame(0)
    assert sha(rgb) == str(p['full_rgb_sha']) and sha(depth) == str(p['full_depth_sha'])
    poses = synth.raw_poses(8, seed=0)
    assert np.array_equal(poses, p['full_poses'])
    for i in range(8):
        bb = O.compute_bbox(poses[i], synth.CAMERA_K, 200., scale=(1000, 1000, 1000))
        assert np.array_equal(bb, p[f'full_bb_{i}'])
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        assert sha(rB) == str(p[f'full_rgbB_sha_{i}']) and sha(dB) == str(p[f'full_depthB_sha_{i}'])


def test_process_data_both_dtype_chains(synth, golden_dir):
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    rgb, depth, K = p['small_rgb'], p['small_depth'], p['K_small']
    n = len(p['object_width'])
    poses = p['poses']
    rgbAs, depthAs = synth.rendered_views(n, poses, seed=7)
    mean, std = synth.default_mean_std()
    stats = {'f32': (mean, std), 'f64': (mean.astype(np.float64) + 0.123, std.astype(np.float64) * 1.01)}
    for i in range(n):
        bb = O.compute_bbox(poses[i], K, p['object_width'][i], scale=(1000, 1000, 1000))
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        for tag, (m, s) in stats.items():
            (dA_, dB_), (tl, rl) = O.process_data(rgbAs[i], depthAs[i], poses[i].copy(), rB, dB,
                                                  p[f'gtB_{i}'].copy(), m, s)
            assert dA_.dtype == np.float32
            assert sha(dA_) == str(p[f'dataA_sha_{tag}_{i}']), (tag, i)
            assert sha(dB_) == str(p[f'dataB_sha_{tag}_{i}']), (tag, i)
            assert np.array_equal(dA_[:, ::11, ::11], p[f'dataA_sub_{tag}_{i}'])
        assert np.array_equal(tl, p[f'label_trans_{i}']) and np.array_equal(rl, p[f'label_rot_{i}'])


def test_process_predict_and_normalize(golden_dir):
    p = np.load(os.path.join(golden_dir, 'golden_pre.npz'))
    n = len(p['pu_poses'])
    for i in range(n):
        o5 = O.process_predict(p['pu_poses'][i], (p['pu_trans'][i], p['pu_rot'][i]))
        o30 = O.process_predict(p['pu_poses'][i], (p['pu_trans'][i], p['pu_rot'][i]),
                                rot_normalizer=30 * np.pi / 180)
        assert o5.dtype == np.float64
        assert np.array_equal(o5, p['pu_out_5deg'][i]) and np.array_equal(o30, p['pu_out_30deg'][i])
        assert np.array_equal(O.normalize_rotation_matrix(p['nrm_in'][i].copy()), p['nrm_out'][i])
    assert np.array_equal(p['pu_out_5deg'][0], p['pu_poses'][0])     # zero residual = identity update


def test_known_answers_rodrigues():
    # SURVEY 8c known-answer checks on the third-party op the path leans on
    assert np.array_equal(cv2.Rodrigues(np.zeros(3))[0], np.eye(3))
    w = np.array([0.3, -0.2, 0.5])
    assert np.allclose(cv2.Rodrigues(cv2.Rodrigues(w)[0])[0].ravel(), w, atol=1e-12)
    assert cv2.Rodrigues(np.zeros(3, np.float32))[0].dtype == np.float32       # F10


def test_numpy1_legacy_depth_differs_by_at_most_one_ulp_of_offset(synth):
    rng = np.random.default_rng(0)
    d = rng.integers(0, 3000, size=(64, 64)).astype(np.uint16)
    pose = np.eye(4); pose[2, 3] = 0.7123456789
    a = O.normalize_depth(d, pose); b = O.normalize_depth(d, pose, legacy_numpy1=True)
    # the two differ by the rounding of the offset z*1000 to float32 (+ one result rounding)
    bound = 2 * np.spacing(np.float32(pose[2, 3] * 1000))
    assert np.all(np.abs(a.astype(np.float64) - b) <= bound)


def test_metrics_oracle_vs_reference(synth, golden_dir):
    """ADD / ADD-S / VOCap restatements against values produced by the reference's own Utils.add / Utils.adi /
    eval_ycb.VOCap (oracle/make_golden.py)."""
    g = np.load(os.path.join(golden_dir, 'golden_metrics.npz'))
    model = synth.model_points(2620, seed=0)
    pred, gt = synth.pose_pairs(12, seed=0)
    pred[0] = gt[0]
    add = np.array([O.add(pred[i], gt[i], model) for i in range(12)])
    adi = np.array([O.adi(pred[i], gt[i], model) for i in range(12)])
    assert np.allclose(add, g['add'], rtol=1e-13, atol=0) and add[0] == 0.0
    assert np.allclose(adi, g['adi'], rtol=1e-13, atol=0) and adi[0] == 0.0
    assert np.all(adi <= add + 1e-15)                      # nearest neighbour can only be closer
    for k in ('mixed', 'all_below', 'dups', 'single', 'sorted_add'):
        assert abs(O.vocap(g['curve_' + k]) - float(g['vocap_' + k])) < 1e-13, k


def test_render_uniforms_vs_reference(synth, golden_dir):
    """Window, projection matrix, view matrix and light direction of the renderer against the reference's own
    update_cam_mat / render_image / compute_bbox (oracle/make_golden.py runs them with vispy stubbed)."""
    g = np.load(os.path.join(golden_dir, 'golden_render.npz'))
    for i, pose in enumerate(g['poses']):
        u = O.render_uniforms(pose, synth.CAMERA_K, float(g['object_width']))
        assert [u['left'], u['right'], u['top'], u['bottom']] == list(g['window'][i])
        assert np.array_equal(u['proj64'], g['proj64'][i])
        assert np.array_equal(u['view32'], g['view'][i].astype(np.float32))           # the GL upload casts to float32
        assert np.array_equal(u['light32'], g['light32'][i]) and g['light32'].dtype == np.float32


def test_render_oracle_properties(synth):
    """The rasterisation restatement itself (no GL here: parity unpinned) must at least behave like a renderer."""
    mesh = synth.mesh(2, seed=0)
    pose = np.eye(4); pose[:3, 3] = (0.03, -0.02, 0.6)
    rgb, dep = O.render_window(pose, synth.CAMERA_K, 200.0, mesh)
    fg = dep > 0
    assert 1500 < fg.sum() < 12000 and rgb[~fg].max() == 0 and rgb[fg].max() > 100
    assert 600 - 30 <= dep[fg].min() and dep[fg].max() <= 600 + 30                      # a 5 x 3.5 x 2.5 cm half-extent body at z = 0.6 m
    ys, xs = np.nonzero(fg)                                                             # centred in its own window
    assert abs(xs.mean() - 88) < 6 and abs(ys.mean() - 88) < 6
    # the same object twice as far away covers a quarter of the pixels of a window that is half as large in pixels ... i.e. the same share
    pose2 = pose.copy(); pose2[:3, 3] *= 2
    _, dep2 = O.render_window(pose2, synth.CAMERA_K, 200.0, mesh)
    assert abs((dep2 > 0).sum() - fg.sum()) < 0.05 * fg.sum()
    # front-most surface wins: every depth is no farther than the object's centre plus its smallest half-extent
    assert (dep[fg] <= 600 + 26).all()
    # degenerate window -> empty image
    rgb0, dep0 = O.render_window(pose, synth.CAMERA_K, 0.0, mesh)
    assert rgb0.max() == 0 and dep0.max() == 0


def test_fill_depth_oracle_vs_reference(golden_dir):
    """Depth hole filling restated (cv2 calls in the reference's order) against the reference's own Utils.fill_depth."""
    g = np.load(os.path.join(golden_dir, 'golden_fill.npz'))
    for k in 'ab':
        mm, m = O.fill_depth_mm(g['in_' + k])
        assert np.array_equal(m, g['out_m_' + k]) and np.array_equal(mm, g['out_mm_' + k])
        assert (g['in_' + k] == 0).mean() > 0.1 and (mm == 0).mean() < 0.02          # the holes are actually filled
        # the optional branches (Utils.py:486-497 extrapolate, :506-510 gaussian), alone and together
        for tag, ex, blur in (('ex', True, 'bilateral'), ('ga', False, 'gaussian'), ('exga', True, 'gaussian')):
            assert np.array_equal(O.fill_depth(g['in_' + k] / 1e3, 2.0, extrapolate=ex, blur_type=blur), g['out_m_%s_%s' % (k, tag)])
        assert not np.array_equal(g['out_m_%s_ex' % k], g['out_m_' + k]) and not np.array_equal(g['out_m_%s_ga' % k], g['out_m_' + k])


def _ray_cast_depth(mesh, pose, K, u, S=176):
    """Pinhole ray through every pixel centre of the crop window against the posed triangles (Moeller-Trumbore, float64);
    -> camera-space depth (S, S), inf where nothing is hit between the near (0.1 m) and far (2 m) planes.  A triangle wholly in
    front of the eye is tested against the rays of its projected box (one pixel of margin) only; any other against all rays."""
    cols = u['left'] + (np.arange(S) + 0.5) * (u['right'] - u['left']) / S
    # the window rows live in the y-flipped image v' = 2*cy - v (compute_bbox with scale -1000); array row 0 is v' = bottom
    vflip = u['bottom'] - (np.arange(S) + 0.5) * (u['bottom'] - u['top']) / S
    rows = 2 * K[1, 2] - vflip
    dx = (cols - K[0, 2]) / K[0, 0]; dy = (rows - K[1, 2]) / K[1, 1]
    D = np.stack(np.broadcast_arrays(dx[None, :], dy[:, None], np.ones((S, S))), -1).reshape(-1, 3)     # ray directions, origin 0
    P = mesh['pos'].astype(np.float64) @ pose[:3, :3].T + pose[:3, 3]
    with np.errstate(divide='ignore', invalid='ignore'):            # window column / row of each vertex (valid where z > 0)
        pi = (K[0, 0] * P[:, 0] / P[:, 2] + K[0, 2] - u['left']) * S / (u['right'] - u['left']) - 0.5
        pj = (K[1, 1] * P[:, 1] / P[:, 2] + K[1, 2] - 2 * K[1, 2] + u['bottom']) * S / (u['bottom'] - u['top']) - 0.5
    everything = np.arange(S * S)
    best = np.full(len(D), np.inf)
    for f in mesh['faces']:
        if (P[f, 2] > 1e-3).all():
            ia, ib = max(0, int(np.floor(pi[f].min())) - 1), min(S - 1, int(np.ceil(pi[f].max())) + 1)
            ja, jb = max(0, int(np.floor(pj[f].min())) - 1), min(S - 1, int(np.ceil(pj[f].max())) + 1)
            if ia > ib or ja > jb:
                continue
            sel = (np.arange(ja, jb + 1)[:, None] * S + np.arange(ia, ib + 1)[None, :]).ravel()
        else:
            sel = everything
        Ds = D[sel]
        v0, v1, v2 = P[f[0]], P[f[1]], P[f[2]]
        e1, e2 = v1 - v0, v2 - v0
        pv = np.cross(Ds, e2); det = pv @ e1
        with np.errstate(divide='ignore', invalid='ignore'):
            inv = 1.0 / det
            tv = -v0
            uu = (pv @ tv) * inv
            qv = np.cross(tv, e1)
            vv = (Ds @ qv) * inv
            t = (qv @ e2) * inv
        hit = (np.abs(det) > 1e-15) & (uu >= 0) & (vv >= 0) & (uu + vv <= 1) & (t > 0.1) & (t < 2.0)
        best[sel] = np.where(hit & (t < best[sel]), t, best[sel])
    return best.reshape(S, S)                                       # direction z-component is 1: t is the camera-space depth


def _assert_same_surface(dep, z, min_pixels):
    import cv2
    ray_fg, ras_fg = np.isfinite(z), dep > 0
    assert ras_fg.sum() > min_pixels
    edge = cv2.dilate(ray_fg.astype(np.uint8), np.ones((3, 3), np.uint8)) != cv2.erode(ray_fg.astype(np.uint8), np.ones((3, 3), np.uint8))
    assert (ray_fg == ras_fg)[~edge].all() and (ray_fg != ras_fg).sum() < 0.02 * ras_fg.sum()
    both = ray_fg & ras_fg & ~edge
    assert np.abs(dep[both].astype(np.float64) - z[both] * 1000).max() < 1.5


def test_render_oracle_vs_ray_casting(synth):
    """Independent geometric cross-check of the rasterisation restatement (no GL here): cast a pinhole ray through every pixel
    centre of the crop window and intersect it with the posed triangles.  The rasteriser must see the same surface: identical
    coverage away from silhouette edges, depth within 1 mm (uint16 truncation + float32 z-buffer).  An 80-face model with large
    triangles, and a 20,480-face one (level 5) whose triangles are mostly below a pixel, as real models' are."""
    K = synth.CAMERA_K
    pose = synth.raw_poses(3, seed=21)[2]
    u = O.render_uniforms(pose, K, 200.0)
    for level in (1, 5):
        mesh = synth.mesh(level, seed=2)
        rgb, dep = O.render_window(pose, K, 200.0, mesh)
        _assert_same_surface(dep, _ray_cast_depth(mesh, pose, K, u), 3000)


def test_render_oracle_nan_normals_count_as_zero_lambert(synth):
    """A NaN vertex normal (what load_ply_mesh makes of a stored (0, 0, 0)) gives a NaN Lambert term, which counts as 0 as the
    GPU's max instruction and fmax take it: all normals NaN draws exactly what all normals zero draws (n.l = 0), and a model
    with some NaN normals casts no NaN to uint8 and shows no black fragment."""
    import warnings
    mesh = synth.mesh(2, seed=0)
    pose = synth.raw_poses(3, seed=21)[2]
    K = synth.CAMERA_K
    nan_all, zero_all, some = dict(mesh), dict(mesh), dict(mesh)
    nan_all['nrm'] = np.full_like(mesh['nrm'], np.nan); zero_all['nrm'] = np.zeros_like(mesh['nrm'])
    some['nrm'] = mesh['nrm'].copy(); some['nrm'][::7] = np.nan
    with warnings.catch_warnings():
        warnings.simplefilter('error')                                 # an invalid cast would warn
        a, b, c = (O.render_window(pose, K, 200.0, m) for m in (nan_all, zero_all, some))
        plain = O.render_window(pose, K, 200.0, mesh)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(c[1], plain[1])
    fg = c[1] > 0
    assert fg.sum() > 2000 and (c[0][fg].max(-1) > 0).all() and (c[0] != plain[0]).any(-1).sum() > 100


def _long_mesh(synth, level, seed, stretch=24.0):
    """A synthetic model stretched along its z axis until it reaches from behind the camera to well in front of it."""
    mesh = dict(synth.mesh(level, seed=seed))
    mesh['pos'] = (mesh['pos'] * np.array([1.0, 1.0, stretch], np.float32)).astype(np.float32)
    return mesh


def test_render_oracle_near_plane_clipping_vs_ray_casting(synth):
    """Triangles with vertices behind the eye plane (w <= 0) and in front of the near plane are cut AT the near plane, as GL's
    polygon clipping does: the visible part must coincide with what rays limited to t in (0.1 m, 2 m) see."""
    import cv2
    K = synth.CAMERA_K
    for level, rvec, tr in ((1, (0.05, 0.02, 0.1), (0.045, 0.0, 0.45)), (2, (0.0, 0.08, 0.5), (0.045, 0.0, 0.45))):
        mesh = _long_mesh(synth, level, seed=2)
        pose = np.eye(4); pose[:3, :3] = cv2.Rodrigues(np.array(rvec))[0]; pose[:3, 3] = tr
        zcam = mesh['pos'].astype(np.float64) @ pose[2, :3] + pose[2, 3]
        assert zcam.min() < -0.05 and zcam.max() > 0.8                      # the model really passes through the eye plane
        f = mesh['faces']; zf = zcam[f]
        assert ((zf.min(1) <= 1e-6) & (zf.max(1) > 0.1)).sum() >= 4          # ... and some triangles straddle it
        u = O.render_uniforms(pose, K, 200.0)
        rgb, dep = O.render_window(pose, K, 200.0, mesh)
        z = _ray_cast_depth(mesh, pose, K, u)
        _assert_same_surface(dep, z, 3000)
        # the test bites: without the straddling triangles a visible part of the surface would be missing
        kept = dict(mesh); kept['faces'] = f[~((zf.min(1) <= 1e-6) & (zf.max(1) > 0.1))]
        with np.errstate(invalid='ignore'):
            lost = np.isfinite(z) & ~(np.abs(z - _ray_cast_depth(kept, pose, K, u)) < 1e-6)   # a closed model: the far side shows instead
        assert lost.sum() > 300 and (dep[lost] > 0).mean() > 0.98
        assert rgb[dep > 0].max() > 0


def test_render_full_frame_unlit_vs_ray_casting(synth):
    """The pyrender-style producer of input A (offscreen_renderer.py:77-83; no pyrender here: parity unpinned): the full camera
    image must show the surface a pinhole ray through every pixel centre (u + 0.5, v + 0.5) hits, with the metric depth pyrender
    reports, unlit colours, and Tracker.render_window's crop (predict.py:210-214) must be crop_bbox of exactly that image."""
    import cv2
    mesh = synth.mesh(1, seed=2)
    K = synth.CAMERA_K
    H, W = 480, 640
    pose = synth.raw_poses(3, seed=21)[2]
    color, depth = O.render_full_frame_unlit(pose, K, mesh, H, W)
    assert color.shape == (H, W, 3) and depth.dtype == np.float32
    ys, xs = np.nonzero(depth > 0)
    assert len(ys) > 500
    y0, y1, x0, x1 = max(ys.min() - 6, 0), min(ys.max() + 7, H), max(xs.min() - 6, 0), min(xs.max() + 7, W)
    uu, vv = np.meshgrid(np.arange(x0, x1) + 0.5, np.arange(y0, y1) + 0.5)
    D = np.stack([(uu - K[0, 2]) / K[0, 0], (vv - K[1, 2]) / K[1, 1], np.ones_like(uu)], -1).reshape(-1, 3)
    P = mesh['pos'].astype(np.float64) @ pose[:3, :3].T + pose[:3, 3]
    best = np.full(len(D), np.inf)
    for f in mesh['faces']:
        v0, v1, v2 = P[f[0]], P[f[1]], P[f[2]]
        e1, e2 = v1 - v0, v2 - v0
        pv = np.cross(D, e2); det = pv @ e1
        with np.errstate(divide='ignore', invalid='ignore'):
            inv = 1.0 / det; tv = -v0
            a = (pv @ tv) * inv; qv = np.cross(tv, e1); b = (D @ qv) * inv; t = (qv @ e2) * inv
        hit = (np.abs(det) > 1e-15) & (a >= 0) & (b >= 0) & (a + b <= 1) & (t > 0.1) & (t < 2.0)
        best = np.where(hit & (t < best), t, best)
    z = best.reshape(y1 - y0, x1 - x0)
    sub = depth[y0:y1, x0:x1]
    ray_fg, ras_fg = np.isfinite(z), sub > 0
    edge = cv2.dilate(ray_fg.astype(np.uint8), np.ones((3, 3), np.uint8)) != cv2.erode(ray_fg.astype(np.uint8), np.ones((3, 3), np.uint8))
    assert (ray_fg == ras_fg)[~edge].all() and (ray_fg != ras_fg).sum() < 0.05 * ras_fg.sum()
    both = ray_fg & ras_fg & ~edge
    assert np.abs(sub[both].astype(np.float64) - z[both]).max() < 2e-4          # float32 z-buffer + float32 linearisation
    outside = np.ones((H, W), bool); outside[y0:y1, x0:x1] = False
    assert not depth[outside].any() and not color[outside].any()
    # unlit: every foreground colour lies within the hull of the model's vertex colours
    fg = color[depth > 0].astype(int)
    assert fg.min() >= int(mesh['col'].min()) - 1 and fg.max() <= int(mesh['col'].max()) + 1
    # the crop: what predict.py:210-214 does with that image
    rgbA, depthA = O.render_window_pyrender(pose, K, 200.0, mesh, H, W)
    bbox = O.compute_bbox(pose, K, 200.0, scale=(1000, 1000, 1000))
    want = O.crop_bbox(color, (depth * np.float32(1000)).astype(np.uint16), bbox, (176, 176))
    assert rgbA.shape == (176, 176, 3) and depthA.dtype == np.uint16
    assert np.array_equal(rgbA, want[0]) and np.array_equal(depthA, want[1]) and (depthA > 0).sum() > 1500
