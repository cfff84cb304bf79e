"""The depth refinement of a tracking step (se3tn_icp_opts, include/se3tn.h; csrc/icp.cu) restated in numpy fp64.

One iteration at pose T = (R, t) (object -> OpenCV camera, metres):
  tri      the triangle each 176 x 176 crop pixel of the model rendered at T shows (-1: none), from the bit-exact rasteriser
           restatement of se3_oracle.py (its visibility keys; what it returns is unchanged)
  window   compute_bbox at scale 1000 and cv2's nearest source indices, as the fit check and K0 crop B
  terms    per crop pixel with tri >= 0 whose frame pixel p is inside the frame and d_obs = depth[p] > 0:
           r = K^-1 (p_x, p_y, 1); the triangle's camera-frame vertices a_k = R v_k + t and unit normal n of (a1 - a0) x (a2 - a0);
           q = r (n.a0) / (n.r), d_model = 1000 q_z; skipped when |n.r| / |r| < 0.1 or d_model <= 0; inlier when
           |d_obs - d_model| <= tau; o = r d_obs / 1000; e = n.(q - o); J = [(q x n)^T, n^T]
  sums     the upper 21 entries of J^T J (row-major), J^T e, sum e^2, the inlier count
  solve    Cholesky of J^T J; fewer than min_inliers inliers or a pivot <= 1e-12 x the largest diagonal entry: the pose stays;
           else xi = -(J^T J)^-1 J^T e and R <- Exp(w) R, t <- Exp(w) t + v (Rodrigues)
Every per-pixel operation is written in the association icp.cu uses (no fused multiply-adds there), so each term and each
inlier decision equals the kernel's bit for bit; only the order of the sums differs."""
import numpy as np

import se3_oracle as so

SIZE = 176


def tri_window(ob2cam, K, object_width, mesh, mode='vispy', H=None, W=None, size=SIZE):
    """-> int32 (size, size): the triangle index each pixel of the render at ob2cam shows, -1 for background, in the layout of
    the render's depth (se3_oracle.render_window in the vispy mode, render_window_pyrender in the pyrender mode)."""
    tri = np.full((size, size), -1, np.int32)
    if mode == 'vispy':
        u = so.render_uniforms(ob2cam, K, object_width)
        if u['right'] == u['left'] or u['top'] == u['bottom'] or not np.all(np.isfinite(u['proj32'])):
            return tri
        key, _, _ = so._rasterise(mesh, u['view32'], u['proj32'], size, size)
        t = (key & np.uint64(0xFFFFFFFF)).astype(np.int64)
        return np.where(t == 0xFFFFFFFF, -1, t).astype(np.int32)
    u = so.pyrender_uniforms(ob2cam, K, H, W)
    key, _, _ = so._rasterise(mesh, u['view32'], u['proj32'], W, H)
    t = (key & np.uint64(0xFFFFFFFF)).astype(np.int64)[::-1]                    # image rows top-down
    full = np.where(t == 0xFFFFFFFF, -1, t).astype(np.int32)
    top, left, ch, cw = so.crop_window(so.compute_bbox(ob2cam, K, object_width, scale=(1000, 1000, 1000)))
    if ch <= 0 or cw <= 0:
        return tri
    fy, fx = window_indices(top, left, ch, cw, size)
    iy, ix = np.nonzero((fy >= 0) & (fy < H))[0], np.nonzero((fx >= 0) & (fx < W))[0]
    tri[np.ix_(iy, ix)] = full[np.ix_(fy[iy], fx[ix])]
    return tri


def window_indices(top, left, ch, cw, size=SIZE):
    """Frame rows and columns the crop's rows and columns read: cv2 INTER_NEAREST's floor(dst * (1 / (size / n))), clamped."""
    sy = np.minimum(np.floor(np.arange(size) * (1.0 / (size / ch))).astype(np.int64), ch - 1)
    sx = np.minimum(np.floor(np.arange(size) * (1.0 / (size / cw))).astype(np.int64), cw - 1)
    return top + sy, left + sx


def pixel_terms(pose, K, object_width, mesh, tri, depth, tau):
    """-> dict(e (m,), J (m, 6), q, n, o (m, 3), pix (m, 2) crop (row, column)) of the inliers of one iteration, crop pixels in
    row-major order."""
    empty = dict(e=np.zeros(0), J=np.zeros((0, 6)), q=np.zeros((0, 3)), n=np.zeros((0, 3)), o=np.zeros((0, 3)),
                 pix=np.zeros((0, 2), np.int64))
    top, left, ch, cw = so.crop_window(so.compute_bbox(pose, K, object_width, scale=(1000, 1000, 1000)))
    if ch <= 0 or cw <= 0:
        return empty
    H, W = depth.shape
    fy, fx = window_indices(top, left, ch, cw, tri.shape[0])
    jj, ii = np.nonzero(tri >= 0)
    t = tri[jj, ii].astype(np.int64)
    keep = t < len(mesh['faces'])
    py, px = fy[jj], fx[ii]
    keep &= (py >= 0) & (py < H) & (px >= 0) & (px < W)
    jj, ii, t, py, px = jj[keep], ii[keep], t[keep], py[keep], px[keep]
    obs = depth[py, px].astype(np.int64)
    keep = obs != 0
    jj, ii, t, py, px, obs = jj[keep], ii[keep], t[keep], py[keep], px[keep], obs[keep]
    P = np.asarray(pose, np.float64).reshape(16)
    pos = mesh['pos'].astype(np.float64)
    f = mesh['faces'][t]
    v = []
    for k in range(3):
        x, y, z = pos[f[:, k], 0], pos[f[:, k], 1], pos[f[:, k], 2]
        v.append([((P[4 * r] * x + P[4 * r + 1] * y) + P[4 * r + 2] * z) + P[4 * r + 3] for r in range(3)])
    e1 = [v[1][r] - v[0][r] for r in range(3)]
    e2 = [v[2][r] - v[0][r] for r in range(3)]
    c = [e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]]
    with np.errstate(divide='ignore', invalid='ignore'):
        length = np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])
        il = 1.0 / length
        nx, ny, nz = c[0] * il, c[1] * il, c[2] * il
        fxK, fyK, cxK, cyK = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
        rx = (px.astype(np.float64) - cxK) / fxK
        ry = (py.astype(np.float64) - cyK) / fyK
        ndr = (nx * rx + ny * ry) + nz
        rl = np.sqrt((rx * rx + ry * ry) + 1.0)
        nda = (nx * v[0][0] + ny * v[0][1]) + nz * v[0][2]
        s = nda / ndr
        dmodel = 1000.0 * s
        dobs = obs.astype(np.float64)
        ok = (length > 0.0) & (np.abs(ndr / rl) >= 0.1) & (dmodel > 0.0) & (np.abs(dobs - dmodel) <= float(tau))
    rx, ry, s, dobs, nx, ny, nz = rx[ok], ry[ok], s[ok], dobs[ok], nx[ok], ny[ok], nz[ok]
    zo = dobs / 1000.0
    q = np.stack([rx * s, ry * s, s], 1)
    o = np.stack([rx * zo, ry * zo, zo], 1)
    n = np.stack([nx, ny, nz], 1)
    e = (nx * (q[:, 0] - o[:, 0]) + ny * (q[:, 1] - o[:, 1])) + nz * (q[:, 2] - o[:, 2])
    J = jacobian(q, n)
    return dict(e=e, J=J, q=q, n=n, o=o, pix=np.stack([jj[ok], ii[ok]], 1))


def jacobian(q, n):
    """J = [(q x n)^T, n^T] per row: the derivative of residual() at xi = 0."""
    q, n = np.atleast_2d(q), np.atleast_2d(n)
    qx, qy, qz, nx, ny, nz = q[:, 0], q[:, 1], q[:, 2], n[:, 0], n[:, 1], n[:, 2]
    return np.stack([qy * nz - qz * ny, qz * nx - qx * nz, qx * ny - qy * nx, nx, ny, nz], 1)


def residual(xi, q, n, o):
    """e(xi) = n . (Exp(w) q + v - o): the point-to-plane residual after the left increment xi = (w, v), the plane's normal
    held fixed (the Gauss-Newton model the solve linearises)."""
    E = exp_so3(np.asarray(xi[:3], np.float64))
    return float(np.dot(n, E @ q + np.asarray(xi[3:], np.float64) - o))


def exp_so3(w):
    """Rodrigues: cos th I + sin th [k]x + (1 - cos th) k k^T, k = w / th (the identity at th = 0)."""
    th = float(np.sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]))
    if th == 0.0:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.cos(th) * np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * np.outer(k, k)


def sums(terms):
    """-> float64 (29,): JtJ upper (21, row-major), Jte (6), sum e^2, count."""
    J, e = terms['J'], terms['e']
    A = J.T @ J
    up = [A[r, c] for r in range(6) for c in range(r, 6)]
    return np.array(up + list(J.T @ e) + [float(e @ e), float(len(e))])


def solve(S, pose, min_inliers):
    """One solve from the sums: -> (new pose (4, 4), stats [inliers, rms_mm, step_mm, step_deg]).  A skipped update returns
    the pose itself (the same array)."""
    A = np.zeros((6, 6))
    k = 0
    for r in range(6):
        for c in range(r, 6):
            A[r, c] = A[c, r] = S[k]
            k += 1
    b, e2, cnt = S[21:27], S[27], S[28]
    stats = [cnt, np.sqrt(e2 / cnt) * 1000.0 if cnt > 0 else 0.0, 0.0, 0.0]
    maxd = float(np.max(np.diag(A)))
    if not (cnt >= min_inliers and maxd > 0 and np.isfinite(maxd)):
        return pose, stats
    L = np.zeros((6, 6))
    for j in range(6):
        d = A[j, j] - sum(L[j, q] * L[j, q] for q in range(j))
        if not d > 1e-12 * maxd:
            return pose, stats
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, 6):
            L[i, j] = (A[i, j] - sum(L[i, q] * L[j, q] for q in range(j))) / L[j, j]
    y = np.zeros(6)
    for i in range(6):
        y[i] = (-b[i] - sum(L[i, q] * y[q] for q in range(i))) / L[i, i]
    xi = np.zeros(6)
    for i in range(5, -1, -1):
        xi[i] = (y[i] - sum(L[q, i] * xi[q] for q in range(i + 1, 6))) / L[i, i]
    E = exp_so3(xi[:3])
    out = np.array(pose, np.float64).copy()
    out[:3, :3] = E @ pose[:3, :3]
    out[:3, 3] = E @ pose[:3, 3] + xi[3:]
    th = float(np.linalg.norm(xi[:3]))
    stats[2] = float(np.linalg.norm(out[:3, 3] - pose[:3, 3])) * 1000.0
    stats[3] = np.degrees(th)
    return out, stats


def iterate(pose, K, object_width, mesh, depth, tau, min_inliers, mode='vispy', H=None, W=None):
    """One ICP iteration from pose: render the triangle ids, form the terms, solve.  -> (pose, stats, terms)."""
    pose = np.asarray(pose, np.float64)
    tri = tri_window(pose, K, object_width, mesh, mode, H, W)
    terms = pixel_terms(pose, K, object_width, mesh, tri, depth, tau)
    new, stats = solve(sums(terms), pose, min_inliers)
    return new, stats, terms


def icp(pose, K, object_width, mesh, depth, tau, min_inliers, iterations, mode='vispy', H=None, W=None):
    """M iterations -> (poses (M, 4, 4) after each, stats (M, 4))."""
    poses, stats = [], []
    for _ in range(iterations):
        pose, st, _ = iterate(pose, K, object_width, mesh, depth, tau, min_inliers, mode, H, W)
        poses.append(pose)
        stats.append(st)
    return np.stack(poses), np.array(stats)


def synthetic_scene(synth, n, seed=0):
    """n ground-truth poses spread over the frame, the 480 x 640 uint16 depth frame the pyrender-mode render draws of them
    (nearest surface per pixel), and starts perturbed by 5-10 mm and 2-5 degrees."""
    rng = np.random.default_rng(seed)
    mesh, K = synth.mesh(), synth.CAMERA_K
    gts, starts = [], []
    D = np.zeros((480, 640), np.uint16)
    for k in range(n):
        P = np.eye(4); P[:3, :3] = synth._random_rotations(rng, 1)[0]
        P[:3, 3] = (-0.24 + 0.16 * (k % 4), -0.08 + 0.16 * (k // 4 % 2), 0.8 + 0.02 * k)
        _, d = so.render_full_frame_unlit(P, K, mesh, 480, 640)
        d = (d * np.float32(1000)).astype(np.uint16)
        D = np.where((d > 0) & ((D == 0) | (d < D)), d, D)
        w = rng.normal(size=3); w /= np.linalg.norm(w)
        t = rng.normal(size=3); t /= np.linalg.norm(t)
        S = P.copy()
        S[:3, :3] = exp_so3(w * np.radians(rng.uniform(2, 5))) @ P[:3, :3]
        S[:3, 3] = P[:3, 3] + t * rng.uniform(0.005, 0.010)
        gts.append(P); starts.append(S)
    return mesh, np.stack(gts), np.stack(starts), D
