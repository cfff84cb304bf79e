"""Start poses from a mask and the depth frame (se3tn_init_poses, include/se3tn.h; csrc/init.cu) restated in numpy.

  stats    mask = #(seg == l), depth_px = #(seg == l, depth > 0), sum_u / sum_v over the mask pixels, z_med = the lower median of
           the mask's depths > 0; status 1: mask = 0, 2: depth_px < min_pixels; t0 = z_med / 1000 K^-1 (u, v, 1), (u, v) the
           mask's centroid; (0, 0, 1) when the status is not 0
  grid     candidate c = v R + r: the Fibonacci-sphere direction d_v mapped to the camera's -z axis (up +z, +y when |d_v.z| >
           0.99), then turned about the camera's z by 2 pi r / R; every candidate at t0
  score    per rendered row, over the 176 x 176 crop of its own window: model, maskc, overlap, pairs, S = sum (O - R) over the
           pairs, delta = (2 S + pairs) // (2 pairs), inlier #(|O - (R + delta)| <= tau)
  rank     the higher inlier / union (union = model + maskc - overlap, 0 scores 0), the higher overlap, the lower candidate
  keep     the K best; each kept pose moves along its ray: t = t0 (1 + delta / (1000 t0_z))
  refine   icp_ref.icp on the kept poses, each rescored at delta 0, the best kept
The rasteriser is se3_oracle's restatement (its depth, vectorised here from the same visibility keys)."""
import functools

import numpy as np

import icp_ref
import se3_oracle as so

SIZE = 176
COLS = ('status', 'candidate', 'model', 'maskc', 'overlap', 'pairs', 'inlier', 'delta')


def mask_stats(depth, seg, label, min_pixels, K):
    """-> (stats int64 [status, mask, depth_px, sum_u, sum_v, z_med], t0 float64 (3,))."""
    v, u = np.nonzero(seg == label)
    d = depth[v, u].astype(np.int64)
    dz = np.sort(d[d > 0])
    mask, depth_px = len(u), len(dz)
    z_med = int(dz[(depth_px - 1) // 2]) if depth_px else 0
    status = 1 if mask == 0 else (2 if depth_px < min_pixels else 0)
    su, sv = int(u.astype(np.int64).sum()), int(v.astype(np.int64).sum())
    stats = np.array([status, mask, depth_px, su, sv, z_med], np.int64)
    if status:
        return stats, np.array([0.0, 0.0, 1.0])
    m = float(mask)
    uu, vv, z = su / m, sv / m, z_med / 1000.0
    return stats, np.array([z * ((uu - K[0, 2]) / K[0, 0]), z * ((vv - K[1, 2]) / K[1, 1]), z])


def viewpoint(v, V):
    z = 1.0 - (2.0 * v + 1.0) / V
    rad = np.sqrt(1.0 - z * z)
    phi = v * (np.pi * (3.0 - np.sqrt(5.0)))
    return np.array([rad * np.cos(phi), rad * np.sin(phi), z])


def grid_rotation(c, V, R):
    """The candidate's rotation (object -> camera)."""
    v, r = divmod(c, R)
    d = viewpoint(v, V)
    up = np.array([0.0, 1.0, 0.0]) if abs(d[2]) > 0.99 else np.array([0.0, 0.0, 1.0])
    zc = -d
    xc = np.cross(zc, up)
    xc = xc * (1.0 / np.sqrt((xc[0] * xc[0] + xc[1] * xc[1]) + xc[2] * xc[2]))
    yc = np.cross(zc, xc)
    th = (2.0 * np.pi) * r / R
    ct, st = np.cos(th), np.sin(th)
    return np.stack([ct * xc - st * yc, st * xc + ct * yc, zc])


def grid(V, R, t0):
    """-> (V R, 4, 4) candidate poses at t0."""
    P = np.tile(np.eye(4), (V * R, 1, 1))
    for c in range(V * R):
        P[c, :3, :3] = grid_rotation(c, V, R)
        P[c, :3, 3] = t0
    return P


def shift(pose, delta):
    """The kept pose moved along its ray by delta mm."""
    out = np.array(pose, np.float64).copy()
    f = 1.0 + float(delta) / (1000.0 * pose[2, 3])
    out[:3, 3] = pose[:3, 3] * f
    return out


def render_depth(pose, K, width, mesh, mode='vispy', H=None, W=None):
    """The render's uint16 depth (176, 176) mm at pose, vectorised from se3_oracle's visibility keys (render_window /
    render_window_pyrender compute the same values pixel by pixel)."""
    if mode == 'vispy':
        u = so.render_uniforms(pose, K, width)
        if u['right'] == u['left'] or u['top'] == u['bottom'] or not np.all(np.isfinite(u['proj32'])):
            return np.zeros((SIZE, SIZE), np.uint16)
        key = so._rasterise(mesh, u['view32'], u['proj32'], SIZE, SIZE)[0]
        hit = (key & np.uint64(0xFFFFFFFF)) != np.uint64(0xFFFFFFFF)
        A, B = u['proj64'][2, 2], u['proj64'][2, 3]
        d32 = (key >> np.uint64(32)).astype(np.uint32).view(np.float32)
        tt = (d32 * np.float32(-2.0)).astype(np.float32) + np.float32(1.0)
        dist = (B / (tt.astype(np.float64) - A)) * -1
        out = np.where(hit & (dist < B / (A + 1)), dist * 1000, 0)
        return out.astype(np.uint16)
    full = full_depth(pose, K, mesh, H, W)
    bbox = so.compute_bbox(pose, K, width, scale=(1000, 1000, 1000))
    return so.crop_bbox(np.zeros((H, W, 3), np.uint8), full, bbox, (SIZE, SIZE))[1]


def full_depth(pose, K, mesh, H, W):
    """The pyrender-mode render of the whole H x W camera image as uint16 mm (render_full_frame_unlit's depth x 1000)."""
    u = so.pyrender_uniforms(pose, K, H, W)
    key = so._rasterise(mesh, u['view32'], u['proj32'], W, H)[0][::-1]
    hit = (key & np.uint64(0xFFFFFFFF)) != np.uint64(0xFFFFFFFF)
    d32 = (key >> np.uint64(32)).astype(np.uint32).view(np.float32)
    zn, zf = np.float32(so.NEAR_PLANE), np.float32(so.FAR_PLANE)
    zn_ = (np.float32(2.0) * d32).astype(np.float32) - np.float32(1.0)
    den = np.float32(zf + zn) - (zn_ * np.float32(zf - zn)).astype(np.float32)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        d = (np.float32(np.float32(2.0) * zn * zf) / den).astype(np.float32)
        return np.where(hit, (d * np.float32(1000)), np.float32(0)).astype(np.uint16)


def crop(pose, K, width, depth, seg, label):
    """(O uint16, M bool) (176, 176): the observed depth and the mask under each crop pixel of pose's window, 0 outside."""
    O, M = np.zeros((SIZE, SIZE), np.uint16), np.zeros((SIZE, SIZE), bool)
    top, left, ch, cw = so.crop_window(so.compute_bbox(pose, K, width, scale=(1000, 1000, 1000)))
    if ch <= 0 or cw <= 0:
        return O, M
    H, W = depth.shape
    fy, fx = icp_ref.window_indices(top, left, ch, cw, SIZE)
    iy, ix = np.nonzero((fy >= 0) & (fy < H))[0], np.nonzero((fx >= 0) & (fx < W))[0]
    O[np.ix_(iy, ix)] = depth[np.ix_(fy[iy], fx[ix])]
    M[np.ix_(iy, ix)] = seg[np.ix_(fy[iy], fx[ix])] == label
    return O, M


def score(Rd, O, M, tau, fixed_delta=False):
    """-> [model, maskc, overlap, pairs, inlier, delta] of a rendered depth against its crop."""
    Rd, O = Rd.astype(np.int64), O.astype(np.int64)
    r = Rd > 0
    pair = r & M & (O > 0)
    model, maskc, overlap, pairs = int(r.sum()), int(M.sum()), int((r & M).sum()), int(pair.sum())
    S = int((O - Rd)[pair].sum())
    delta = 0 if fixed_delta or pairs == 0 else (2 * S + pairs) // (2 * pairs)
    inlier = int((pair & (np.abs(O - (Rd + delta)) <= tau)).sum())
    return [model, maskc, overlap, pairs, inlier, delta]


def row(status, cand, counts):
    model, maskc, overlap, pairs, inlier, delta = counts
    return np.array([status, cand, model, maskc, overlap, pairs, inlier, delta], np.int64)


def ranks_above(x, y):
    """True when score row x ranks strictly above row y."""
    ux, uy = int(x[2]) + int(x[3]) - int(x[4]), int(y[2]) + int(y[3]) - int(y[4])
    lhs, rhs = int(x[6]) * max(uy, 1), int(y[6]) * max(ux, 1)
    if lhs != rhs:
        return lhs > rhs
    if x[4] != y[4]:
        return x[4] > y[4]
    return x[1] < y[1]


def rank_order(rows):
    """Indices of rows, best first."""
    cmp = lambda a, b: -1 if ranks_above(rows[a], rows[b]) else (1 if ranks_above(rows[b], rows[a]) else 0)
    return sorted(range(len(rows)), key=functools.cmp_to_key(cmp))


def score_pose(pose, K, width, mesh, depth, seg, label, tau, mode='vispy', H=None, W=None, fixed_delta=False):
    Rd = render_depth(pose, K, width, mesh, mode, H, W)
    O, M = crop(pose, K, width, depth, seg, label)
    return score(Rd, O, M, tau, fixed_delta)


def init_object(depth, seg, K, label, width, mesh, V, R, keep, tau, min_pixels, icp=None, mode='vispy', H=None, W=None,
                grid_poses=None):
    """Stages 1-6 for one object.  icp: (iterations, tau, min_inliers) or None.  grid_poses: the candidates to score (the
    device's, to compare rows exactly), else grid(V, R, t0).  -> dict stats, t0, grid, rows (V R, 8), kept (K,), kept_poses,
    kept_rows, icp_poses, icp_rows, pose (4, 4), row (8,)."""
    stats, t0 = mask_stats(depth, seg, label, min_pixels, K)
    G = grid(V, R, t0) if grid_poses is None else grid_poses
    rows = np.stack([row(stats[0], c, score_pose(G[c], K, width, mesh, depth, seg, label, tau, mode, H, W)) for c in range(V * R)])
    kept = rank_order(rows)[:keep]
    kept_poses = np.stack([shift(G[c], rows[c, 7]) for c in kept])
    out = dict(stats=stats, t0=t0, grid=G, rows=rows, kept=np.array(kept), kept_poses=kept_poses, kept_rows=rows[kept])
    cand_rows, cand_poses = out['kept_rows'], kept_poses
    if icp is not None:
        it, itau, imin = icp
        ip = np.stack([icp_ref.icp(P, K, width, mesh, depth, itau, imin, it, mode, H, W)[0][-1] for P in kept_poses])
        ir = np.stack([row(stats[0], c, score_pose(P, K, width, mesh, depth, seg, label, tau, mode, H, W, fixed_delta=True))
                       for c, P in zip(kept, ip)])
        out.update(icp_poses=ip, icp_rows=ir)
        cand_rows, cand_poses = ir, ip
    best = rank_order(cand_rows)[0]
    out['row'] = cand_rows[best]
    out['pose'] = cand_poses[best] if stats[0] == 0 else np.full((4, 4), np.nan)
    return out


def labelled_scene(synth, n, seed=0):
    """icp_ref.synthetic_scene with a label image: each pixel labelled k + 1 by the object k whose depth won it, 0 for none.
    -> (mesh, gts (n, 4, 4), starts, depth uint16 (480, 640), seg uint8 (480, 640))."""
    mesh, gts, starts, D = icp_ref.synthetic_scene(synth, n, seed)
    K = synth.CAMERA_K
    D2, L = np.zeros_like(D), np.zeros(D.shape, np.uint8)
    for k, P in enumerate(gts):
        d = full_depth(P, K, mesh, *D.shape)
        win = (d > 0) & ((D2 == 0) | (d < D2))
        D2 = np.where(win, d, D2)
        L = np.where(win, np.uint8(k + 1), L)
    assert np.array_equal(D2, D), 'the label image was drawn from another depth than the scene'
    return mesh, gts, starts, D, L
