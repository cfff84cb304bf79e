"""Start poses from a 2D box and the depth frame (se3tn_init_boxes, include/se3tn.h; csrc/init.cu) restated in numpy, on top of
init_ref's mask rule.

  box      int (x0, y0, x1, y1), half-open: the pixels x0 <= u < x1, y0 <= v < y1, inside the frame; x1 == x0 or y1 == y0 is
           empty (status 1)
  stats    init_ref.mask_stats' columns over the box's pixels: mask = the box's pixel count, depth_px, sum_u, sum_v, z_med the
           lower median; status 1 / 2 as for a mask
  depths   D candidates: z_d = the sorted depth at k_d = max(0, floor(((2 d + 1) depth_px - D) / (2 D))), d < D (the quantiles
           (2 d + 1) / 2 D; D = 1 is the lower median); t0_d = z_d / 1000 K^-1 (u, v, 1) on the ray through the box centre;
           (0, 0, 1) for each d when the status is not 0
  grid     candidate c = d V R + v R + r: init_ref.grid_rotation(v R + r) at t0_d
  score    init_ref.score with M = "the crop pixel's source frame pixel lies in the box"
  keep / refine / choose   init_ref's, over the D V R rows of the object"""
import numpy as np

import icp_ref
import init_ref
import se3_oracle as so


def quantile_index(d, D, depth_px):
    """The sorted index of depth candidate d of D among depth_px depths."""
    return max(0, ((2 * d + 1) * depth_px - D) // (2 * D))


def candidate(d, v, r, V, R):
    """The candidate number of depth d, viewpoint v and in-plane angle r."""
    return (d * V + v) * R + r


def box_mask(box, H, W):
    """The box's pixels as a bool (H, W) image."""
    x0, y0, x1, y1 = (int(x) for x in box)
    m = np.zeros((H, W), bool)
    m[y0:y1, x0:x1] = True
    return m


def box_stats(depth, box, min_pixels, K, D):
    """-> (stats int64 [status, mask, depth_px, sum_u, sum_v, z_med], t0 float64 (D, 3))."""
    stats, _ = init_ref.mask_stats(depth, box_mask(box, *depth.shape).astype(np.uint8), 1, min_pixels, K)
    if stats[0]:
        return stats, np.tile([0.0, 0.0, 1.0], (D, 1))
    x0, y0, x1, y1 = (int(x) for x in box)
    d = depth[y0:y1, x0:x1].astype(np.int64).reshape(-1)
    dz = np.sort(d[d > 0])
    m = float(stats[1])
    uu, vv = int(stats[3]) / m, int(stats[4]) / m
    t0 = []
    for q in range(D):
        z = int(dz[quantile_index(q, D, len(dz))]) / 1000.0
        t0.append([z * ((uu - K[0, 2]) / K[0, 0]), z * ((vv - K[1, 2]) / K[1, 1]), z])
    return stats, np.array(t0)


def grid(V, R, t0):
    """-> (D V R, 4, 4) candidate poses, depth d's block at t0[d]."""
    return np.concatenate([init_ref.grid(V, R, t) for t in t0])


def crop(pose, K, width, depth, box):
    """(O uint16, M bool) (176, 176): the observed depth and box membership under each crop pixel of pose's window."""
    H, W = depth.shape
    O = init_ref.crop(pose, K, width, depth, np.zeros((H, W), np.uint8), 1)[0]
    M = np.zeros((init_ref.SIZE, init_ref.SIZE), bool)
    top, left, ch, cw = so.crop_window(so.compute_bbox(pose, K, width, scale=(1000, 1000, 1000)))
    if ch <= 0 or cw <= 0:
        return O, M
    fy, fx = icp_ref.window_indices(top, left, ch, cw, init_ref.SIZE)
    x0, y0, x1, y1 = (int(x) for x in box)
    M[:] = ((fy >= y0) & (fy < y1) & (fy >= 0) & (fy < H))[:, None] & ((fx >= x0) & (fx < x1) & (fx >= 0) & (fx < W))[None, :]
    return O, M


def score_pose(pose, K, width, mesh, depth, box, tau, mode='vispy', H=None, W=None, fixed_delta=False):
    Rd = init_ref.render_depth(pose, K, width, mesh, mode, H, W)
    O, M = crop(pose, K, width, depth, box)
    return init_ref.score(Rd, O, M, tau, fixed_delta)


def init_object(depth, box, K, width, mesh, V, R, keep, tau, min_pixels, D, icp=None, mode='vispy', H=None, W=None):
    """Stages 1-6 for one object from its box, as init_ref.init_object.  -> dict stats, t0 (D, 3), grid, rows (D V R, 8),
    kept, kept_poses, kept_rows, icp_poses, icp_rows, pose (4, 4), row (8,)."""
    stats, t0 = box_stats(depth, box, min_pixels, K, D)
    G = grid(V, R, t0)
    rows = np.stack([init_ref.row(stats[0], c, score_pose(G[c], K, width, mesh, depth, box, tau, mode, H, W)) for c in range(len(G))])
    kept = init_ref.rank_order(rows)[:keep]
    kept_poses = np.stack([init_ref.shift(G[c], rows[c, 7]) for c in kept])
    out = dict(stats=stats, t0=t0, grid=G, rows=rows, kept=np.array(kept), kept_poses=kept_poses, kept_rows=rows[kept])
    cand_rows, cand_poses = out['kept_rows'], kept_poses
    if icp is not None:
        it, itau, imin = icp
        ip = np.stack([icp_ref.icp(P, K, width, mesh, depth, itau, imin, it, mode, H, W)[0][-1] for P in kept_poses])
        ir = np.stack([init_ref.row(stats[0], c, score_pose(P, K, width, mesh, depth, box, tau, mode, H, W, fixed_delta=True))
                       for c, P in zip(kept, ip)])
        out.update(icp_poses=ip, icp_rows=ir)
        cand_rows, cand_poses = ir, ip
    best = init_ref.rank_order(cand_rows)[0]
    out['row'] = cand_rows[best]
    out['pose'] = cand_poses[best] if stats[0] == 0 else np.full((4, 4), np.nan)
    return out


def tight_box(seg, label):
    """The tight half-open box of seg == label: (min u, min v, max u + 1, max v + 1); (0, 0, 0, 0) without pixels."""
    v, u = np.nonzero(seg == label)
    if len(u) == 0:
        return np.zeros(4, np.int32)
    return np.array([u.min(), v.min(), u.max() + 1, v.max() + 1], np.int32)


def with_background(depth, K, near=1.1, far=1.3):
    """depth with a tilted plane behind the scene wherever it is 0: z runs from `near` m at the top row to `far` m at the
    bottom row, so every box around an object also holds background depth.  uint16 mm."""
    H, W = depth.shape
    v = np.arange(H, dtype=np.float64)[:, None] + np.zeros((1, W))
    u = np.arange(W, dtype=np.float64)[None, :] + np.zeros((H, 1))
    z = near + (far - near) * (v / (H - 1)) + 0.02 * (u / (W - 1) - 0.5)
    plane = np.round(z * 1000).astype(np.uint16)
    return np.where(depth == 0, plane, depth).astype(np.uint16)
