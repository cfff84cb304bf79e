"""The rasteriser (csrc/render.cu through Engine.render, Engine.visibility and Engine.init_poses) bit for bit against the oracle
(se3_oracle.render_window / render_window_pyrender / render_full_frame_unlit) where the suite's small meshes never take it:

  * models of 20,480 to 327,680 faces (synth.mesh(5..7)), near, mid, far and over the image border, and a model crossing the
    near plane: sub-pixel triangles, many faces per pixel, window-z ties, triangles snapped to zero area, a projected-vertex
    stride 60-250x the small meshes';
  * meshes built for the rules a rasteriser decides (oracle/render_cases.py): vertices on sample centres (the top-left rule,
    checked also against the coverage any watertight rule gives), coincident and z-tied layers (depth test LESS, the first
    drawn wins), faces without area and unused vertices (nothing drawn), NaN vertex normals (a NaN Lambert term counts as 0);
  * launch shapes: batch sizes across warp and CTA multiples, level-0 and level-7 models in one launch, a context whose
    workspace grows under captured steps;
  * the consumers at that density: the visibility check's coverage counts and the initialiser's candidate rows.

Every comparison is exact.  Oracle results are cached per module so that each (level, mode, pose) is drawn once."""
import importlib
import os
import sys
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
PKG = 'iros20-6d-pose-tracking_b200'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_ref  # noqa: E402
import render_cases as rc  # noqa: E402
import se3_oracle as so  # noqa: E402

synth_mod = importlib.import_module(PKG + '.synth')
K = synth_mod.CAMERA_K
HW = (480, 640)
WIDTH = 200.0
TN, RN = 0.03, 5 * np.pi / 180
# near: window larger than 176 px; far: 1.4-1.9 m, where snapping collapses triangles; border: the window hangs over the
# right / top edge of the camera image
PLACES = {'near': (0.05, -0.04, 0.33), 'mid': (-0.03, 0.02, 0.7), 'far': (-0.08, 0.06, 1.7), 'border': (0.13, -0.09, 0.55)}
DENSE = {(5, 'vispy'): ('near', 'far'), (5, 'pyrender'): ('near', 'border'),
         (6, 'vispy'): ('near', 'mid', 'far'), (6, 'pyrender'): ('mid', 'far'),
         (7, 'vispy'): ('near', 'far'), (7, 'pyrender'): ('far', 'border')}


def place(name):
    p = synth_mod.raw_poses(4, seed=31)[list(PLACES).index(name)].copy()
    p[:3, 3] = PLACES[name]
    return p


def _hw(mode):
    return HW if mode == 'pyrender' else None


def oracle_render(mode, pose, mesh):
    if mode == 'vispy':
        return so.render_window(pose, K, WIDTH, mesh)
    return so.render_window_pyrender(pose, K, WIDTH, mesh, *HW)


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


def render(e, mode, poses, ids, widths=None):
    """Engine.render of poses (n,4,4) with mesh ids (n) -> numpy (rgb, depth)."""
    n = len(poses)
    ow = torch.full((n,), WIDTH, dtype=torch.float64, device=e.device) if widths is None else _dev(e, widths)
    rgb, dep = e.render(K, _dev(e, poses), ow, _dev(e, np.asarray(ids, np.int32)), mode=mode, image_hw=_hw(mode))
    return rgb.cpu().numpy(), dep.cpu().numpy()


def assert_same(got, want, what):
    (rgb, dep), (rrgb, rdep) = got, want
    assert np.array_equal(dep, rdep), '%s: %d depth pixels differ' % (what, (dep != rdep).sum())
    assert np.array_equal(rgb, rrgb), '%s: %d colour values differ' % (what, (rgb != rrgb).sum())


@pytest.fixture(scope='module')
def meshes(synth):
    return {lv: synth.mesh(lv, seed=lv) for lv in (0, 1, 5, 6, 7)}


@pytest.fixture(scope='module')
def oracle(meshes):
    """oracle(level, mode, place) -> (rgb, depth), each drawn once per module."""
    cache = {}

    def get(level, mode, name):
        key = (level, mode, name)
        if key not in cache:
            cache[key] = oracle_render(mode, place(name), meshes[level])
        return cache[key]
    return get


@pytest.fixture(scope='module')
def eng(pkg, meshes):
    e = pkg.Engine(max_batch=8)
    for lv, m in meshes.items():
        e.set_mesh(m, lv)                         # mesh id = level
    yield e
    e.close()


# ------------------------------------------------------------------------------------------------ 1. dense meshes
@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
@pytest.mark.parametrize('level', [5, 6, 7])
def test_dense_mesh_bit_exact(eng, meshes, oracle, level, mode):
    names = DENSE[(level, mode)]
    poses = np.stack([place(nm) for nm in names])
    rgb, dep = render(eng, mode, poses, [level] * len(names))
    for i, nm in enumerate(names):
        assert_same((rgb[i], dep[i]), oracle(level, mode, nm), 'level %d %s %s' % (level, mode, nm))
        assert (dep[i] > 0).sum() > 2000
    if 'far' in names:                            # the regime: sub-pixel triangles, and at levels 6 and 7 some snap to zero area
        view32, proj32, vw, vh = rc.viewport(place('far'), K, WIDTH, mode, *HW)
        X, Y = rc.snapped(meshes[level]['pos'], view32, proj32, vw, vh)
        f = meshes[level]['faces']
        area2 = np.abs((X[f[:, 1]] - X[f[:, 0]]) * (Y[f[:, 2]] - Y[f[:, 0]]) - (X[f[:, 2]] - X[f[:, 0]]) * (Y[f[:, 1]] - Y[f[:, 0]]))
        assert np.median(area2) < 2 * so.SUBPIXEL ** 2
        assert level < 6 or (area2 == 0).sum() > 0


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_dense_mesh_crossing_the_near_plane(eng, meshes, mode):
    """The stretched model of test_render_near_plane_clipping_bit_exact at level 5: many small triangles behind the eye
    (dropped: at this density none reaches past the near plane) and many crossing the near plane (cut per pixel by the depth
    test)."""
    import cv2
    mesh = rc.stretched(meshes[5])
    p = np.eye(4); p[:3, :3] = cv2.Rodrigues(np.array((0.05, 0.02, 0.1)))[0]; p[:3, 3] = (0.045, 0.0, 0.45)
    zf = (mesh['pos'].astype(np.float64) @ p[2, :3] + p[2, 3])[mesh['faces']]
    assert (zf.min(1) <= 1e-6).sum() >= 64 and ((zf.min(1) < 0.1) & (zf.max(1) > 0.1)).sum() >= 64
    eng.set_mesh(mesh, 9)
    rgb, dep = render(eng, mode, p[None], [9])
    assert_same((rgb[0], dep[0]), oracle_render(mode, p, mesh), 'near plane %s' % mode)
    assert (dep[0] > 0).sum() > 3000


# ------------------------------------------------------------------------------------------------ 2. constructed meshes
GRIDS = [('vispy', 'mid', 0.7), ('pyrender', 'near', 0.33), ('pyrender', 'far', 1.7)]


@pytest.mark.parametrize('mode,name,zc', GRIDS, ids=['vispy', 'pyrender-near', 'pyrender-far'])
def test_sample_centre_grid(eng, mode, name, zc):
    """Every sample on an edge or a vertex of the grid.  Each face has its own colour, so the rgb shows which face won every
    sample: it must be the oracle's.  Independently of the oracle: the top-left rule with window y up covers the samples of
    the half-open box [x0, x1) x (y0, y1] -- every sample strictly inside, the left column and the top row without their far
    ends -- and nothing else."""
    pose = place(name)
    cols, rows = rc.window_samples(pose, K, WIDTH, mode, *HW)
    if mode == 'vispy':
        x0, x1, y0, y1 = 30, 146, 40, 136
    else:                                        # grid edges on camera pixels the crop samples, so they show in the output
        vc, vr = np.unique(cols[cols >= 0]), np.unique(rows[rows >= 0])
        x0, y0 = int(vc[12]), int(vr[10])
        x1 = int([c for c in vc if c > x0 + 60 and (c - x0) % 2 == 0][0])
        y1 = int([r for r in vr if r > y0 + 50 and (r - y0) % 2 == 0][0])
    mesh = rc.sample_grid(pose, K, WIDTH, mode, x0, x1, y0, y1, zc, *HW)
    eng.set_mesh(mesh, 9)
    rgb, dep = render(eng, mode, pose[None], [9])
    assert_same((rgb[0], dep[0]), oracle_render(mode, pose, mesh), 'grid %s %s' % (mode, name))
    ok = (cols[None, :] >= 0) & (rows[:, None] >= 0)
    jj, ii = np.broadcast_arrays(rows[:, None], cols[None, :])
    strict = ok & (ii > x0) & (ii < x1) & (jj > y0) & (jj < y1)
    outside = ~ok | (ii < x0) | (ii > x1) | (jj < y0) | (jj > y1)
    top_left = ok & (ii >= x0) & (ii < x1) & (jj > y0) & (jj <= y1)
    cov = dep[0] > 0
    assert cov[strict].all() and not cov[outside].any()
    assert np.array_equal(cov, top_left)
    assert (top_left & ~strict).sum() > 20                     # boundary samples are in the picture
    # the faces that win: 4 per cell at most, and samples on shared edges or vertices each pick one of them
    assert len(np.unique(rgb[0][cov].reshape(-1, 3), axis=0)) > cov.sum() // 3


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_coincident_layers_first_drawn_wins(eng, synth, mode):
    """The faces drawn twice over identical positions with other colours: every pixel ties in window z, so the first drawn
    shows -- the original image with the copy appended after it, the copy's image with it placed before.  A copy moved
    3e-8 m away from the eye, below float32 window-z resolution, ties at most pixels with unequal positions: placed first, it
    shows there, and the original only where the nearer surface wins in float32."""
    base = synth.mesh(4, seed=3)
    other = dict(base, col=(255 - base['col']).astype(np.uint8))
    pose = place('mid')
    eng.set_mesh(base, 9); alone = render(eng, mode, pose[None], [9])
    eng.set_mesh(other, 9); alone_other = render(eng, mode, pose[None], [9])
    for order, want in (('after', alone), ('before', alone_other)):
        m = rc.layered(base, other['col'], order)
        eng.set_mesh(m, 9)
        got = render(eng, mode, pose[None], [9])
        assert_same(got, want, 'layers %s' % order)
        ref = oracle_render(mode, pose, m)
        assert_same((got[0][0], got[1][0]), ref, 'layers %s vs oracle' % order)
    m = rc.layered(base, other['col'], 'before', shift=3e-8, pose=pose)
    eng.set_mesh(m, 9)
    got = render(eng, mode, pose[None], [9])
    assert_same((got[0][0], got[1][0]), oracle_render(mode, pose, m), 'shifted layer')
    cov = got[1][0] > 0
    copy_shows = (got[0][0] == alone_other[0][0]).all(-1) & cov
    base_shows = (got[0][0] == alone[0][0]).all(-1) & cov
    assert copy_shows.sum() > 0.5 * cov.sum() and base_shows.sum() > 0
    # the positions really differ and the window z really ties: the copy drawn alone has other float32 positions and the
    # same z32 as the original at most pixels
    assert not np.array_equal(m['pos'][len(base['pos']):], base['pos'])
    view32, proj32, vw, vh = rc.viewport(pose, K, WIDTH, mode, *HW)
    k0 = so._rasterise(base, view32, proj32, vw, vh)[0] >> np.uint64(32)
    k1 = so._rasterise(dict(base, pos=m['pos'][len(base['pos']):]), view32, proj32, vw, vh)[0] >> np.uint64(32)
    hit = k0 != np.uint64(0x3F800000)
    assert (k0 == k1)[hit].mean() > 0.5 and (k0 != k1)[hit].any()


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_degenerate_faces_and_unused_vertices_draw_nothing(eng, synth, mode):
    """Faces with a repeated index, faces whose vertices snap onto one row, column or diagonal of samples in front of the
    model, and vertices no face uses: the image is the model's own, bit for bit."""
    base = synth.mesh(4, seed=6)
    pose = place('mid')
    m = rc.with_degenerates(base, pose, K, WIDTH, mode, *HW)
    assert len(m['faces']) == len(base['faces']) + 8 and len(m['pos']) > len(base['pos'])
    eng.set_mesh(base, 9); want = render(eng, mode, pose[None], [9])
    eng.set_mesh(m, 9); got = render(eng, mode, pose[None], [9])
    assert_same(got, want, 'degenerates')
    assert_same((got[0][0], got[1][0]), oracle_render(mode, pose, m), 'degenerates vs oracle')
    assert_same((got[0][0], got[1][0]), oracle_render(mode, pose, base), 'model vs oracle')


def test_nan_normals_count_as_zero_lambert(eng, synth, tmp_path):
    """A vertex stored with normal (0, 0, 0) loads as NaN (load_ply_mesh normalises as vispy_renderer.py:121 does).  Its
    fragments' Lambert term is NaN, which counts as 0: the ambient 0.65 alone, never the undefined cast of a NaN colour."""
    mio = importlib.import_module(PKG + '.mesh_io')
    base = synth.mesh(2, seed=0)
    pose = place('mid')
    front = np.argsort(so._project_vertices(base['pos'], *rc.viewport(pose, K, WIDTH, 'vispy'))[2])[:40]     # visible ones
    stored = dict(base, nrm=base['nrm'].copy())
    stored['nrm'][front] = 0.0
    path = str(tmp_path / 'zero_normals.ply')
    mio.save_ply_mesh(path, stored)
    with np.errstate(invalid='ignore'):
        loaded = mio.load_ply_mesh(path)
    assert np.isnan(loaded['nrm'][front]).all() and np.isfinite(np.delete(loaded['nrm'], front, 0)).all()
    eng.set_mesh(base, 9)
    plain = render(eng, 'vispy', pose[None], [9])
    eng.set_mesh(loaded, 9)
    got = render(eng, 'vispy', pose[None], [9])
    want = oracle_render('vispy', pose, loaded)
    assert_same((got[0][0], got[1][0]), want, 'nan normals')
    cov = got[1][0] > 0
    assert cov.sum() > 1000 and (got[0][0][cov].max(-1) > 0).all()
    assert np.array_equal(got[1], plain[1]) and (got[0] != plain[0]).any(-1).sum() > 100     # the shading changed, nothing else
    # all normals NaN draws what all normals zero draws (n.l = 0): ambient only, on both sides
    nan_all, zero_all = synth.mesh(2, seed=0), synth.mesh(2, seed=0)
    nan_all['nrm'] = np.full_like(base['nrm'], np.nan); zero_all['nrm'] = np.zeros_like(base['nrm'])
    eng.set_mesh(nan_all, 9); a = render(eng, 'vispy', pose[None], [9])
    eng.set_mesh(zero_all, 9); b = render(eng, 'vispy', pose[None], [9])
    assert_same(a, b, 'nan vs zero normals')
    assert_same((a[0][0], a[1][0]), oracle_render('vispy', pose, nan_all), 'nan normals vs oracle')


# ------------------------------------------------------------------------------------------------ 3. launch shapes
@pytest.fixture(scope='module')
def batch_eng(pkg, meshes):
    e = pkg.Engine(max_batch=160)
    e.set_mesh(meshes[5], 0)
    yield e
    e.close()


@pytest.mark.parametrize('mode', ['vispy', 'pyrender'])
def test_batch_rows_equal_single_renders(batch_eng, meshes, mode):
    """n in {1, 2, 63, 64, 65, max_batch}: every row of a batched render equals its pose drawn alone; a seeded sample of
    rows equals the oracle."""
    e = batch_eng
    nmax = e.max_batch
    poses = synth_mod.raw_poses(nmax, seed=77)
    for i, nm in enumerate(('near', 'far', 'border')):
        poses[5 + 40 * i] = place(nm)
    widths = np.full(nmax, WIDTH); widths[3::7] = 150.0
    single = [render(e, mode, poses[i:i + 1], [0], widths[i:i + 1]) for i in range(nmax)]
    for n in (1, 2, 63, 64, 65, nmax):
        rgb, dep = render(e, mode, poses[:n], [0] * n, widths[:n])
        for i in range(n):
            assert np.array_equal(rgb[i], single[i][0][0]) and np.array_equal(dep[i], single[i][1][0]), (mode, n, i)
    for i in np.random.default_rng(3).choice(nmax, 3, replace=False):
        want = (so.render_window(poses[i], K, widths[i], meshes[5]) if mode == 'vispy'
                else so.render_window_pyrender(poses[i], K, widths[i], meshes[5], *HW))
        assert_same((single[i][0][0], single[i][1][0]), want, 'row %d' % i)


def test_level0_and_level7_in_one_launch(eng, meshes, oracle):
    """Tracks of a 12-vertex model at the 163,842-vertex stride of a level-7 model in the same launch."""
    names = ['near', 'far', 'far', 'near', 'mid', 'near']
    ids = [7, 0, 7, 0, 0, 7]
    poses = np.stack([place(nm) for nm in names])
    rgb, dep = render(eng, 'vispy', poses, ids)
    for i, (nm, lv) in enumerate(zip(names, ids)):
        alone = render(eng, 'vispy', poses[i:i + 1], [lv])
        assert np.array_equal(rgb[i], alone[0][0]) and np.array_equal(dep[i], alone[1][0]), i
        assert_same((rgb[i], dep[i]), oracle(lv, 'vispy', nm), 'row %d (level %d)' % (i, lv))


def test_workspace_growth_under_captured_steps(pkg, synth, meshes, oracle):
    """A context that has captured render-tracking steps with small models grows its projected-vertex workspace when a
    level-7 model is set: the next step and render equal the oracle's render and a fresh context's step."""
    def make(models):
        e = pkg.Engine(max_batch=4)
        mean, std = synth.default_mean_std()
        for wid, m in models.items():
            e.load_state_dict(synth.make_state_dict(wid), wid); e.set_stats(mean, std, wid); e.set_mesh(m, wid)
        return e
    names = ['near', 'far']
    poses = np.stack([place(nm) for nm in names])
    rgb_f, depth_f = synth.raw_frame(5)
    wid = np.array([0, 1], np.int32)
    small = {0: meshes[1], 1: meshes[0]}
    grown = {0: meshes[7], 1: meshes[0]}

    def step(e, outs=None):
        ow = torch.full((2,), WIDTH, dtype=torch.float64, device=e.device)
        r = e.track_render(_dev(e, rgb_f), _dev(e, depth_f), K, _dev(e, poses), ow, TN, RN, weight_ids_host=wid,
                           weight_ids_dev=_dev(e, wid), **(outs or {}))
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in r]
    e = make(small)
    try:
        outs = dict(out_poses=torch.empty(2, 4, 4, dtype=torch.float64, device=e.device),
                    out_trans=torch.empty(2, 3, device=e.device), out_rot=torch.empty(2, 3, device=e.device))
        for _ in range(2):
            before = step(e, outs)
        assert e.last_step_was_graph()
        e.set_mesh(meshes[7], 0)
        after = step(e, outs)
        rgb, dep = render(e, 'vispy', poses, wid)
        f = make(grown)
        try:
            fresh = step(f)
            frgb, fdep = render(f, 'vispy', poses, wid)
        finally:
            f.close()
    finally:
        e.close()
    assert all(np.array_equal(x, y) for x, y in zip(after, fresh))
    assert not np.array_equal(after[0], before[0])
    assert np.array_equal(rgb, frgb) and np.array_equal(dep, fdep)
    assert_same((rgb[0], dep[0]), oracle(7, 'vispy', 'near'), 'grown row 0')
    assert_same((rgb[1], dep[1]), oracle(0, 'vispy', 'far'), 'grown row 1')


# ------------------------------------------------------------------------------------------------ 4. consumers
def test_visibility_coverage_at_level6(eng, meshes):
    """Engine.visibility's covered counts (a coverage pass of its own over the whole camera image) equal the pixels of
    render_full_frame_unlit whose depth is > 0.1 m; visible counts the class's labels."""
    names = ['near', 'mid', 'border']
    poses = np.stack([place(nm) for nm in names])
    seg = np.random.default_rng(8).integers(0, 4, HW).astype(np.uint8)
    cid = np.array([1, 2, 3], np.int32)
    vis, cov = eng.visibility(_dev(eng, seg), K, _dev(eng, poses), _dev(eng, cid), mesh_ids=np.full(3, 6, np.int32))
    vis, cov = vis.cpu().numpy(), cov.cpu().numpy()
    for i in range(3):
        _, depth = so.render_full_frame_unlit(poses[i], K, meshes[6], *HW)
        assert cov[i] == int((depth > np.float32(0.1)).sum()) and cov[i] > 1000, (i, cov[i])
        assert vis[i] == int((seg == cid[i]).sum())


def test_init_at_its_defaults(pkg, synth, meshes):
    """V 300, R 24, K 8 on a level-5 model, three objects, max_batch 64: 21,600 candidate rows in 338 chunks, the last one
    partial, chunks across object boundaries.  The kept rows are the rank order of the call's own candidate rows; a seeded
    sample of candidate rows, with rows on both sides of chunk boundaries, equals the oracle's score (pyrender mode)."""
    _, gts, _, D, seg = init_ref.labelled_scene(synth, 3, seed=0)
    e = pkg.Engine(max_batch=64)
    try:
        e.set_mesh(meshes[5], 0)
        spec = e.INIT_DEFAULTS
        V, R, Kk = spec['viewpoints'], spec['inplane'], spec['keep']
        VR, n = V * R, 3
        assert (n * VR) % e.max_batch != 0 and VR % e.max_batch != 0
        out = dict(stats=torch.full((n, 6), -7, dtype=torch.int64, device=e.device),
                   t0=torch.full((n, 3), float('nan'), dtype=torch.float64, device=e.device),
                   cand_rows=torch.full((n, VR, 8), -7, dtype=torch.int32, device=e.device),
                   kept_rows=torch.full((n, Kk, 8), -7, dtype=torch.int32, device=e.device))
        ow = torch.full((n,), WIDTH, dtype=torch.float64, device=e.device)
        P, rows = e.init_poses(_dev(e, D), _dev(e, seg), K, [1, 2, 3], ow, mode='pyrender', image_hw=HW, init=None, out=out)
        torch.cuda.synchronize()
        o = {k: v.cpu().numpy() for k, v in out.items()}
    finally:
        e.close()
    rng = np.random.default_rng(12)
    B = 64
    for i in range(n):
        assert o['stats'][i][0] == 0
        cand = o['cand_rows'][i]
        assert (cand[:, 1] == np.arange(VR)).all()
        order = init_ref.rank_order(cand)
        assert np.array_equal(o['kept_rows'][i], cand[order[:Kk]])
        # candidates on both sides of the chunk boundaries nearest the object's start and end, and random ones
        first = (-(i * VR)) % B                                # first candidate of this object that starts a chunk
        last = ((i + 1) * VR - 1) // B * B - i * VR            # last chunk start inside the object
        picks = {first - 1, first, last - 1, last} | set(int(c) for c in rng.choice(VR, 4, replace=False))
        picks = sorted(c for c in picks if 0 <= c < VR)
        for c in picks:
            pose = np.eye(4); pose[:3, :3] = init_ref.grid_rotation(c, V, R); pose[:3, 3] = o['t0'][i]
            want = init_ref.row(0, c, init_ref.score_pose(pose, K, WIDTH, meshes[5], D, seg, i + 1, spec['tau_mm'], 'pyrender', *HW))
            assert np.array_equal(cand[c], want), (i, c, cand[c], want)
