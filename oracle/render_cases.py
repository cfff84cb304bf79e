"""Meshes built to put the rasteriser (csrc/render.cu, se3_oracle.render_window / render_window_pyrender) where rasterisers go
wrong: vertices on sample centres, coincident and z-tied layers, degenerate faces, NaN normals.  Every mesh is the dict
Engine.set_mesh and the oracle take (pos float32 (nv,3), nrm float32 (nv,3), col uint8 (nv,3), faces int32 (nf,3))."""
import numpy as np

import icp_ref
import se3_oracle as so

SIZE = 176


def viewport(pose, K, width, mode, H=None, W=None):
    """-> (view32, proj32, vw, vh): the GL uniforms and viewport the render of pose uses (vispy: the 176 x 176 crop window;
    pyrender: the whole H x W camera image)."""
    if mode == 'vispy':
        u = so.render_uniforms(pose, K, width)
        return u['view32'], u['proj32'], SIZE, SIZE
    u = so.pyrender_uniforms(pose, K, H, W)
    return u['view32'], u['proj32'], W, H


def unproject(view32, proj32, vw, vh, xw, yw, zc):
    """float32 object-space points that project to window position (xw, yw) (pixels, y up) at camera depth zc metres, through
    the float32 uniforms.  The projection snaps to 1/256 pixel, so the float32 rounding of the result (far below that) does not
    move the snapped position; sample_grid and with_degenerates check it."""
    P, V = proj32.astype(np.float64), view32.astype(np.float64)
    assert P[3, 0] == 0 and P[3, 1] == 0
    xw, yw = np.broadcast_arrays(np.asarray(xw, np.float64), np.asarray(yw, np.float64))
    ze = -float(zc)                                                  # GL eye space looks down -z
    w = P[3, 2] * ze + P[3, 3]
    rhs = np.stack([(2.0 * xw / vw - 1.0) * w - P[0, 2] * ze - P[0, 3], (2.0 * yw / vh - 1.0) * w - P[1, 2] * ze - P[1, 3]], -1)
    xy = np.linalg.solve(P[:2, :2], rhs.reshape(-1, 2).T).T
    eye = np.concatenate([xy, np.full((len(xy), 1), ze)], 1)
    obj = (eye - V[:3, 3]) @ np.linalg.inv(V[:3, :3]).T
    return obj.reshape(xw.shape + (3,)).astype(np.float32)


def snapped(mesh_pos, view32, proj32, vw, vh):
    """-> (X, Y) int64: the sub-pixel positions the rasteriser snaps the vertices to."""
    X, Y = so._project_vertices(mesh_pos, view32, proj32, vw, vh)[:2]
    return X.astype(np.int64), Y.astype(np.int64)


def _face_colours(nf, seed):
    """A distinct colour per face for up to 2^24 faces: an odd multiplier permutes the 24-bit codes."""
    code = (np.arange(nf, dtype=np.int64) * 2654435761 + 97 * (seed + 1)) % (1 << 24)
    return np.stack([code & 255, (code >> 8) & 255, (code >> 16) & 255], 1).astype(np.uint8)


def _flat_mesh(corners, faces, face_col, normal):
    """One vertex per face corner, so every face shows its own colour: which face wins a pixel is visible in the rgb."""
    faces = np.asarray(faces, np.int64)
    pos = corners[faces].reshape(-1, 3)
    col = np.repeat(face_col, 3, axis=0)
    nrm = np.tile(np.asarray(normal, np.float32), (len(pos), 1))
    return dict(pos=pos.astype(np.float32), nrm=nrm, col=col, faces=np.arange(len(pos), dtype=np.int32).reshape(-1, 3))


def sample_grid(pose, K, width, mode, x0, x1, y0, y1, zc, H=None, W=None, seed=0):
    """A planar grid whose vertices sit on sample centres: corner vertices on the samples (i, j) with i - x0 and j - y0 even,
    x0 <= i <= x1, y0 <= j <= y1 (window sample indices, y up: the window's pixels in the vispy mode, the camera pixels in the
    pyrender mode), and each 2 x 2 cell split along both diagonals at the vertex on its centre sample.  Every sample of the
    grid's box then lies on an edge or a vertex.  Each face has its own vertices and colour.  -> mesh."""
    assert (x1 - x0) % 2 == 0 and (y1 - y0) % 2 == 0 and x1 > x0 and y1 > y0
    view32, proj32, vw, vh = viewport(pose, K, width, mode, H, W)
    ii, jj = np.meshgrid(np.arange(x0, x1 + 1), np.arange(y0, y1 + 1))           # every sample of the box, row-major
    pts = unproject(view32, proj32, vw, vh, ii + 0.5, jj + 0.5, zc).reshape(-1, 3)
    X, Y = snapped(pts, view32, proj32, vw, vh)
    assert np.array_equal(X, (ii.reshape(-1) * so.SUBPIXEL + so.SUBPIXEL // 2)) and \
        np.array_equal(Y, (jj.reshape(-1) * so.SUBPIXEL + so.SUBPIXEL // 2)), 'a grid vertex missed its sample centre'
    nx = x1 - x0 + 1
    at = lambda i, j: (j - y0) * nx + (i - x0)
    faces = []
    for j in range(y0, y1, 2):
        for i in range(x0, x1, 2):
            a, b, c, d, m = at(i, j), at(i + 2, j), at(i + 2, j + 2), at(i, j + 2), at(i + 1, j + 1)
            faces += [(a, b, m), (b, c, m), (c, d, m), (d, a, m)]
    normal = np.linalg.inv(view32.astype(np.float64)[:3, :3]) @ np.array([0.0, 0.0, 1.0])       # towards the eye
    return _flat_mesh(pts, faces, _face_colours(len(faces), seed), normal)


def window_samples(pose, K, width, mode, H=None, W=None):
    """-> (cols, rows) int64 (176,): the window sample (x index, y index with y up) each output column / row shows.
    vispy: the window pixels themselves (output row r is window row r); pyrender: the camera pixel crop_bbox's resize reads,
    -1 where it lies outside the image."""
    if mode == 'vispy':
        return np.arange(SIZE), np.arange(SIZE)
    top, left, ch, cw = so.crop_window(so.compute_bbox(pose, K, width, scale=(1000, 1000, 1000)))
    fy, fx = icp_ref.window_indices(top, left, ch, cw, SIZE)
    cols = np.where((fx >= 0) & (fx < W), fx, -1)
    rows = np.where((fy >= 0) & (fy < H), H - 1 - fy, -1)
    return cols, rows


def layered(mesh, recolour, order, shift=0.0, pose=None):
    """The faces of `mesh` drawn twice: once over its own vertices and once over a copy with the colours `recolour` (uint8
    (nv,3)), the copy moved `shift` metres along the camera's viewing axis of pose (away from the eye for shift > 0).
    order 'after': the original faces first; 'before': the copy's first.  -> mesh."""
    nv = len(mesh['pos'])
    pos2 = mesh['pos'].astype(np.float64)
    if shift:
        pos2 = pos2 + np.asarray(pose)[:3, :3].T @ np.array([0.0, 0.0, shift])
    pos = np.concatenate([mesh['pos'], pos2.astype(np.float32)])
    nrm = np.concatenate([mesh['nrm'], mesh['nrm']])
    col = np.concatenate([mesh['col'], recolour.astype(np.uint8)])
    f, f2 = mesh['faces'], mesh['faces'] + nv
    faces = np.concatenate([f, f2] if order == 'after' else [f2, f])
    return dict(pos=pos.astype(np.float32), nrm=nrm.astype(np.float32), col=col, faces=faces.astype(np.int32))


def with_degenerates(mesh, pose, K, width, mode, H=None, W=None, zc=None):
    """`mesh` with faces that have no area inserted before, among and after its own (their relative order kept): repeated
    indices (a a b, a b b, a a a over visible vertices) and collinear faces whose three vertices snap onto one row, one column
    and one diagonal of samples in front of the model; plus vertices no face uses, placed in front of it.  -> mesh with the
    same image as `mesh`."""
    view32, proj32, vw, vh = viewport(pose, K, width, mode, H, W)
    X, Y = snapped(mesh['pos'], view32, proj32, vw, vh)
    nv = len(mesh['pos'])
    zc = float(pose[2, 3]) - 0.08 if zc is None else zc                              # nearer the eye than the model
    cx, cy = int(np.median(X) // so.SUBPIXEL), int(np.median(Y) // so.SUBPIXEL)      # a sample the model covers
    line = [(cx - 6, cy), (cx, cy), (cx + 6, cy), (cx, cy - 5), (cx, cy), (cx, cy + 7), (cx - 4, cy - 4), (cx, cy), (cx + 3, cy + 3)]
    lp = unproject(view32, proj32, vw, vh, np.array([p[0] for p in line]) + 0.5, np.array([p[1] for p in line]) + 0.5, zc)
    lx, ly = snapped(lp, view32, proj32, vw, vh)
    assert np.array_equal(lx, np.array([p[0] for p in line]) * 256 + 128) and np.array_equal(ly, np.array([p[1] for p in line]) * 256 + 128)
    spare = unproject(view32, proj32, vw, vh, np.array([cx + 0.5, cx - 10.5, cx + 20.25]), np.array([cy + 0.5, cy + 9.5, cy - 3.75]), zc)
    a, b = int(np.argmin(np.abs(X - cx * 256) + np.abs(Y - cy * 256))), int(mesh['faces'][0, 1])
    deg = np.array([(a, a, b), (a, b, b), (a, a, a), (b, a, a),
                    (nv, nv + 1, nv + 2), (nv + 3, nv + 4, nv + 5), (nv + 6, nv + 7, nv + 8), (nv + 2, nv, nv + 1)], np.int32)
    f = mesh['faces']
    h = len(f) // 2
    faces = np.concatenate([deg[:3], f[:h], deg[3:6], f[h:], deg[6:]])
    pos = np.concatenate([mesh['pos'], lp, spare]).astype(np.float32)
    nrm = np.concatenate([mesh['nrm'], np.tile(mesh['nrm'][:1], (len(lp) + len(spare), 1))]).astype(np.float32)
    col = np.concatenate([mesh['col'], np.full((len(lp) + len(spare), 3), 255, np.uint8)])
    return dict(pos=pos, nrm=nrm, col=col, faces=faces.astype(np.int32))


def with_nan_normals(mesh, vertices):
    """`mesh` with the normals of `vertices` NaN: what load_ply_mesh makes of a vertex stored with normal (0, 0, 0)."""
    out = dict(mesh)
    nrm = mesh['nrm'].copy()
    nrm[vertices] = np.nan
    out['nrm'] = nrm
    return out


def stretched(mesh, stretch=24.0):
    """`mesh` stretched along its z axis until, at the poses the near-plane tests use, it reaches from behind the eye to well
    in front of it."""
    out = dict(mesh)
    out['pos'] = (mesh['pos'] * np.array([1.0, 1.0, stretch], np.float32)).astype(np.float32)
    return out
