"""CPU oracle for the se(3)-TrackNet per-frame inference hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package imports this file.
Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import it, and only as the checker / the timed
CPU baseline -- never as a fallback for the CUDA path.

What it restates (file:line are relative to the upstream reference tree,
wenbowen123/iros20-6d-pose-tracking @ 18dc5bac):

  compute_bbox                 Utils.py:302-316
  crop_bbox                    Utils.py:320-359
  normalize_rotation_matrix    Utils.py:363-367
  normalize_depth              data_augmentation.py:134-144   (OffsetDepth)
  normalize_channels           data_augmentation.py:154-164   (NormalizeChannels)
  to_tensor                    data_augmentation.py:179-189   (ToTensor)
  process_data                 datasets.py:115-156            (TrackDataset.processData)
  crop_bbox_indexed            Utils.py:320-359 through cv2's nearest-neighbour index formula (no canvas)
  process_predict              datasets.py:159-175            (TrackDataset.processPredict)
  process_predict_exact        datasets.py:159-175 with its float32 roundings and the product's association pinned
  forward                      se3_tracknet.py:81-112 + network_modules.py:59-66,86-120
  on_track                     predict.py:217-296 (render_window output taken as an input)
  add / adi                    Utils.py:72-98     (ADD, ADD-S; scipy cKDTree for the nearest neighbour)
  vocap                        eval_ycb.py:45-64  (VOCap)

Third-party arithmetic the reference delegates to, and which the oracle calls
directly because the same libraries are importable here:
  * conv / batch-norm / pooling / linear -> PyTorch CPU fp32 (reference pins
    torch==1.10.2+cu113, docker/dockerfile:34; here torch 2.11 CPU)
  * so(3) exp / log -> cv2.Rodrigues (datasets.py:148,173)
  * nearest resize -> cv2.resize(INTER_NEAREST) (Utils.py:343-344)

Parity pinning: the reference ships no tests and no golden vectors (SURVEY.md
section 8c).  The oracle is therefore pinned against OUTPUTS OF THE REFERENCE
ITSELF RUN IN THE BUILD CONTAINER: ``oracle/make_golden.py`` imports the
reference's own ``se3_tracknet.py`` (unchanged) and its ``Utils.py`` /
``data_augmentation.py`` / ``datasets.py`` (with the missing third-party
imports stubbed and ``np.float`` aliased, nothing else touched), runs them on
seeded inputs and writes ``tests/golden/*.npz``.  ``tests/test_oracle_golden.py``
checks this file against those fixtures bit-for-bit.

numpy note: ``depth -= pose[2,3]*1000`` (data_augmentation.py:139-141) is an
in-place op between a float32 array and a float64 scalar.  Under numpy >= 2
(NEP 50, what runs here) the subtraction happens in float64 and is rounded once
to float32; numpy 1.x converted the scalar to float32 first.  The two differ by
at most ~1 ulp of float32(z*1000), i.e. < 1.3e-4 mm for z < 2 m.  The oracle follows the numpy >= 2 behaviour because
that is what the reference does when run in this image; `legacy_numpy1=True`
selects the other.
"""
import numpy as np
import cv2
import torch
import torch.nn.functional as F

IMAGE_SIZE = 176

# ----------------------------------------------------------------------------
# geometry / cropping  (Utils.py)
# ----------------------------------------------------------------------------

def compute_bbox(pose, K, scale_size=230, scale=(1, 1, 1)):
    """Utils.py:302-316.  The four corners (x-+half, y-+half) of a metric square
    of side `scale_size` centred on the (scaled) object position, at the object's
    depth, pushed through the pinhole model in float64 and rounded with np.round
    (half-to-even) to int32.  Row order: (-,-), (-,+), (+,-), (+,+); columns (v,u)."""
    centre = np.array([pose[0, 3] * scale[0], pose[1, 3] * scale[1], pose[2, 3] * scale[2]],
                      dtype=np.float64)
    half = scale_size / 2
    signs = np.array([[-1, -1], [-1, 1], [1, -1], [1, 1]], dtype=np.float64)
    xs = centre[0] + signs[:, 0] * half
    ys = centre[1] + signs[:, 1] * half
    zs = np.full(4, centre[2])
    vu = np.empty((4, 2), dtype=np.float64)
    vu[:, 0] = ys * K[1, 1] / zs + K[1, 2]
    vu[:, 1] = xs * K[0, 0] / zs + K[0, 2]
    return np.round(vu).astype(np.int32)


def crop_window(boundingbox):
    """(top, left, crop_h, crop_w) of the window crop_bbox cuts: Utils.py:321-328."""
    top, left = int(boundingbox[:, 0].min()), int(boundingbox[:, 1].min())
    bottom, right = int(boundingbox[:, 0].max()), int(boundingbox[:, 1].max())
    return top, left, bottom - top, right - left


def crop_bbox(color, depth, boundingbox, output_size=(100, 100)):
    """Utils.py:320-359 (seg=None).  The window [top,bottom) x [left,right) of the
    frame is copied into a zero canvas (pixels outside the frame stay 0), then both
    canvases are resized with cv2 INTER_NEAREST; the depth canvas is float64
    (Utils.py:330) and is cast to uint16 after the resize (Utils.py:353).  The
    trailing `* mask` multiplies (Utils.py:351-355) are identities."""
    top, left, crop_h, crop_w = crop_window(boundingbox)
    H, W = color.shape[:2]
    rgb_canvas = np.zeros((crop_h, crop_w, 3), dtype=color.dtype)
    z_canvas = np.zeros((crop_h, crop_w), dtype=np.float64)
    # intersection of the window with the frame, in frame and in canvas coordinates
    y0, y1 = max(top, 0), min(top + crop_h, H)
    x0, x1 = max(left, 0), min(left + crop_w, W)
    cy0, cx0 = abs(min(top, 0)), abs(min(left, 0))
    cy1 = min(crop_h - (top + crop_h - H), crop_h)
    cx1 = min(crop_w - (left + crop_w - W), crop_w)
    rgb_canvas[cy0:cy1, cx0:cx1, :] = color[y0:y1, x0:x1, :]
    z_canvas[cy0:cy1, cx0:cx1] = depth[y0:y1, x0:x1]
    rgb_out = cv2.resize(rgb_canvas, output_size, interpolation=cv2.INTER_NEAREST)
    z_out = cv2.resize(z_canvas, output_size, interpolation=cv2.INTER_NEAREST).astype(np.uint16)
    return rgb_out * (rgb_out != 0), z_out * (z_out != 0)


def crop_bbox_indexed(color, depth, boundingbox, output_size=(100, 100)):
    """crop_bbox without the canvas, for windows too large to allocate one (tens of thousands of pixels a side when the
    object is millimetres from the camera).  cv2's INTER_NEAREST takes output pixel (y, x) from canvas pixel
    (min(floor(y * (1 / (dh / h))), h - 1), min(floor(x * (1 / (dw / w))), w - 1)), the factors in float64; the canvas
    pixel is frame pixel (top + sy, left + sx), zero outside the frame.  An empty window (object_width 0) gives zeros:
    that is what the crop kernels cut, while the reference's cv2.resize refuses an empty canvas."""
    top, left, crop_h, crop_w = crop_window(boundingbox)
    out_w, out_h = output_size
    H, W = color.shape[:2]
    rgb = np.zeros((out_h, out_w, 3), dtype=color.dtype)
    z = np.zeros((out_h, out_w), dtype=depth.dtype)
    if crop_h <= 0 or crop_w <= 0:
        return rgb, z
    sy = np.minimum(np.floor(np.arange(out_h) * (1.0 / (out_h / crop_h))).astype(np.int64), crop_h - 1)
    sx = np.minimum(np.floor(np.arange(out_w) * (1.0 / (out_w / crop_w))).astype(np.int64), crop_w - 1)
    fy, fx = top + sy, left + sx
    iy, ix = np.nonzero((fy >= 0) & (fy < H))[0], np.nonzero((fx >= 0) & (fx < W))[0]
    rgb[np.ix_(iy, ix)] = color[np.ix_(fy[iy], fx[ix])]
    z[np.ix_(iy, ix)] = depth[np.ix_(fy[iy], fx[ix])]
    return rgb, z


def normalize_rotation_matrix(R):
    """Utils.py:363-367 (in place, column-normalise)."""
    R[:, 0] = R[:, 0] / np.linalg.norm(R[:, 0])
    R[:, 1] = R[:, 1] / np.linalg.norm(R[:, 1])
    R[:, 2] = R[:, 2] / np.linalg.norm(R[:, 2])
    return R


# ----------------------------------------------------------------------------
# post-transforms  (data_augmentation.py)
# ----------------------------------------------------------------------------

def normalize_depth(depth, pose, legacy_numpy1=False):
    """data_augmentation.py:134-144."""
    depth = depth.astype(np.float32)
    invalid_mask = np.logical_or(depth <= 100, depth >= 2000)
    z = pose[2, 3] * 1000
    if legacy_numpy1:
        z = np.float32(z)
    if pose[2, 3] < 0:   # gl pose
        depth += z
    else:
        depth -= z
    depth[invalid_mask] = 2000
    return depth


def normalize_channels(rgb, depth, mean, std):
    """data_augmentation.py:159-163."""
    rgb = rgb.transpose(2, 0, 1)
    rgb = (rgb - mean[:3, np.newaxis, np.newaxis]) / std[:3, np.newaxis, np.newaxis]
    depth = (depth - mean[3, np.newaxis, np.newaxis]) / std[3, np.newaxis, np.newaxis]
    return rgb, depth


def to_tensor(rgbA, depthA, rgbB, depthB):
    """data_augmentation.py:179-189 -> two float32 (4,H,W) arrays."""
    bufferA = np.zeros((4, rgbA.shape[1], rgbA.shape[2]), dtype=np.float32)
    bufferA[0:3] = rgbA
    bufferA[3] = depthA
    bufferB = np.zeros((4, rgbA.shape[1], rgbA.shape[2]), dtype=np.float32)
    bufferB[0:3] = rgbB
    bufferB[3] = depthB
    return bufferA, bufferB


def post_transforms(rgbA, depthA, rgbB, depthB, A_in_cam, mean, std, legacy_numpy1=False):
    """Compose([OffsetDepth(), NormalizeChannels(mean,std), ToTensor()]) as
    built at predict.py:189.  Both depths are offset by A's z (F12)."""
    dA = normalize_depth(depthA, A_in_cam, legacy_numpy1)
    dB = normalize_depth(depthB, A_in_cam, legacy_numpy1)
    rA = rgbA.astype(np.float32)
    rB = rgbB.astype(np.float32)
    rA, dA = normalize_channels(rA, dA, mean[:4], std[:4])
    rB, dB = normalize_channels(rB, dB, mean[4:], std[4:])
    return to_tensor(rA, dA, rB, dB)


# ----------------------------------------------------------------------------
# TrackDataset.processData / processPredict  (datasets.py)
# ----------------------------------------------------------------------------

def process_data(rgbA, depthA, A_in_cam, rgbB, depthB, B_in_cam, mean, std,
                 trans_normalizer=0.03, rot_normalizer=5 * np.pi / 180, legacy_numpy1=False):
    """datasets.py:115-156 with pretransforms=augmentations=None (predict.py:191).
    Returns ([dataA, dataB], [trans_label, rot_label])."""
    dataA, dataB = post_transforms(rgbA, depthA, rgbB, depthB, A_in_cam, mean, std, legacy_numpy1)
    trans_label = B_in_cam[:3, 3] - A_in_cam[:3, 3]
    trans_label = trans_label / trans_normalizer
    A2B = B_in_cam[:3, :3].dot(A_in_cam[:3, :3].T)
    A2B = normalize_rotation_matrix(A2B)
    rod = cv2.Rodrigues(A2B)[0].reshape(-1)
    rot_label = rod / rot_normalizer
    return [dataA, dataB], [trans_label, rot_label]


def process_predict(A_in_cam, predB, trans_normalizer=0.03, rot_normalizer=5 * np.pi / 180):
    """datasets.py:159-175.  dtype chain (F10): net output float32 * python float
    stays float32; cv2.Rodrigues(float32) returns float32; .dot(float64) -> float64."""
    B_in_cam = np.eye(4)
    trans_pred = predB[0] * trans_normalizer
    B_in_cam[:3, 3] = trans_pred + A_in_cam[:3, 3]
    rot_pred = predB[1] * rot_normalizer
    A2B = cv2.Rodrigues(rot_pred)[0].reshape(3, 3)
    B_in_cam[:3, :3] = A2B.dot(A_in_cam[:3, :3])
    return B_in_cam


def pose_compose_exact(A_in_cam, R, t):
    """B = [R . A_R | float64(t) + A_t] for a batch (n,4,4), (n,3,3), (n,3): each product entry in scalar float64 as
    (r0 a0 + r1 a1) + r2 a2, every operation rounded on its own (numpy ufuncs; np.dot may fuse or reorder in BLAS)."""
    A = np.asarray(A_in_cam, dtype=np.float64)
    R = np.asarray(R, dtype=np.float64)
    B = np.zeros_like(A)
    for r in range(3):
        for c in range(3):
            B[:, r, c] = (R[:, r, 0] * A[:, 0, c] + R[:, r, 1] * A[:, 1, c]) + R[:, r, 2] * A[:, 2, c]
    B[:, :3, 3] = np.asarray(t).astype(np.float64) + A[:, :3, 3]
    B[:, 3, 3] = 1.0
    return B


def process_predict_exact(A_in_cam, trans, rot, trans_normalizer=0.03, rot_normalizer=5 * np.pi / 180):
    """process_predict for a batch, every rounding pinned: the dtype chain of datasets.py:159-175 (F9 / F10) with the
    rotation product in the association the pose update uses.
      trans_pred = float32 trans * float32(tn)               (float32 array times a Python float stays float32)
      R32        = cv2.Rodrigues(float32 rot * float32(rn))  (float32 in, float32 out: OpenCV's float64 result rounded)
      B          = pose_compose_exact(A, R32, trans_pred)"""
    t32 = np.asarray(trans, dtype=np.float32) * np.float32(trans_normalizer)
    r32 = np.asarray(rot, dtype=np.float32) * np.float32(rot_normalizer)
    R32 = np.stack([cv2.Rodrigues(r)[0] for r in r32])
    assert t32.dtype == np.float32 and R32.dtype == np.float32
    return pose_compose_exact(A_in_cam, R32, t32)


# ----------------------------------------------------------------------------
# Se3TrackNet.forward  (se3_tracknet.py:81-112) as a pure function of state_dict
# ----------------------------------------------------------------------------

SELU_ALPHA = 1.6732632423543772
SELU_SCALE = 1.0507009873554805
BN_EPS = 1e-5

def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'],
                        sd[p + '.weight'], sd[p + '.bias'], False, 0.0, BN_EPS)

def _conv_bn_selu(x, sd, p, stride, pad):
    """network_modules.py:59-66: Conv -> BN(eval) -> SELU (F1)."""
    x = F.conv2d(x, sd[p + '.0.weight'], sd[p + '.0.bias'], stride=stride, padding=pad)
    return F.selu(_bn(x, sd, p + '.1'))

def _basic_block(x, sd, p):
    """network_modules.py:105-120, stride 1, no downsample (F2)."""
    out = F.conv2d(x, sd[p + '.conv1.weight'], sd[p + '.conv1.bias'], padding=1)
    out = F.relu(_bn(out, sd, p + '.bn1'))
    out = F.conv2d(out, sd[p + '.conv2.weight'], sd[p + '.conv2.bias'], padding=1)
    out = _bn(out, sd, p + '.bn2')
    return F.relu(out + x)

@torch.no_grad()
def forward(sd, A, B, return_intermediates=False):
    """A, B: float32 (N,4,H,W) torch CPU tensors; sd: reference-format state_dict."""
    inter = {}
    a = _conv_bn_selu(A, sd, 'convA1', 2, 3); inter['a1'] = a
    a = F.max_pool2d(a, 3, 2, 1); inter['a1p'] = a
    a = _basic_block(a, sd, 'convA2'); inter['a2'] = a
    b = _conv_bn_selu(B, sd, 'convB1', 2, 3); inter['b1'] = b
    b = F.max_pool2d(b, 3, 2, 1); inter['b1p'] = b
    b = _basic_block(b, sd, 'convB2'); inter['b2'] = b
    b = _basic_block(b, sd, 'convB3'); inter['b3'] = b
    ab = torch.cat((a, b), 1).contiguous()
    ab = _conv_bn_selu(ab, sd, 'convAB1', 2, 1); inter['ab1'] = ab
    ab = _basic_block(ab, sd, 'convAB2'); inter['ab2'] = ab
    out = {'feature': ab}
    for head in ('trans', 'rot'):
        h = _conv_bn_selu(ab, sd, head + '_conv1', 2, 1); inter[head + '1'] = h
        h = _basic_block(h, sd, head + '_conv2'); inter[head + '2'] = h
        h = F.adaptive_avg_pool2d(h, 1).reshape(A.shape[0], -1)
        h = torch.tanh(F.linear(h, sd[head + '_out.0.weight'], sd[head + '_out.0.bias']))
        out[head] = h.contiguous()
    if return_intermediates:
        return out, inter
    return out


# ----------------------------------------------------------------------------
# Tracker.on_track  (predict.py:217-296), renderer output supplied by the caller
# ----------------------------------------------------------------------------

def on_track(sd, prev_pose, current_rgb, current_depth, rgbA, depthA, K, object_width,
             mean, std, trans_normalizer=0.03, rot_normalizer=5 * np.pi / 180,
             image_size=IMAGE_SIZE, return_all=False):
    """predict.py:217-296 with samples=1, imshow removed and render_window's
    result (rgbA u8 HxWx3, depthA u16 mm) passed in."""
    A_in_cam = prev_pose.copy()
    bb = compute_bbox(A_in_cam, K, object_width, scale=(1000, 1000, 1000))
    rgbB, depthB = crop_bbox(current_rgb, current_depth, bb, (image_size, image_size))
    sample, _ = process_data(rgbA, depthA, A_in_cam, rgbB, depthB, np.eye(4), mean, std,
                             trans_normalizer, rot_normalizer)
    dataA = torch.from_numpy(sample[0]).unsqueeze(0).float()
    dataB = torch.from_numpy(sample[1]).unsqueeze(0).float()
    pred = forward(sd, dataA, dataB)
    trans = pred['trans'][0].numpy()
    rot = pred['rot'][0].numpy()
    out = process_predict(A_in_cam, (trans, rot), trans_normalizer, rot_normalizer)
    if return_all:
        return out, dict(bb=bb, rgbB=rgbB, depthB=depthB, dataA=sample[0], dataB=sample[1],
                         trans=trans, rot=rot)
    return out


# ----------------------------------------------------------------------------
# metrics  (Utils.py:72-98, eval_ycb.py:45-64)  -- SURVEY.md 8(f) row 1
# ----------------------------------------------------------------------------

def _transform(points, T):
    """open3d PointCloud.transform: p -> R p + t (float64)."""
    return points @ T[:3, :3].T + T[:3, 3]


def add(pred, gt, model_pts):
    """Utils.py:72-82."""
    return np.linalg.norm(_transform(model_pts, pred) - _transform(model_pts, gt), axis=1).mean()


def adi(pred, gt, model_pts):
    """Utils.py:84-98 (cKDTree.query(k=1); `n_jobs=` was renamed `workers=` in scipy 1.6 and later removed)."""
    from scipy import spatial
    nn_index = spatial.cKDTree(_transform(model_pts, pred).copy())
    nn_dists, _ = nn_index.query(_transform(model_pts, gt).copy(), k=1)
    return nn_dists.mean()


def vocap(rec):
    """eval_ycb.py:45-64.  Forward running max over precision values that are already increasing."""
    rec = np.sort(np.asarray(rec, dtype=np.float64).reshape(-1))
    n = len(rec)
    prec = np.arange(1, n + 1) / float(n)
    keep = rec < 0.1
    rec, prec = rec[keep], prec[keep]
    mrec = np.concatenate(([0.0], rec, [0.1]))
    mpre = np.maximum.accumulate(np.concatenate(([0.0], prec, [prec[-1]])))
    i = np.where(mrec[1:] != mrec[:-1])[0] + 1
    return np.sum((mrec[i] - mrec[i - 1]) * mpre[i]) * 10


# =============================================================================================
# Input A: the rendered view of the object at the previous pose (SURVEY.md 8f row 2)
#   window + matrices   predict.py:193-215 (Tracker.render_window), vispy_renderer.py:135-150 (update_cam_mat)
#   light               vispy_renderer.py:171-173 (render_image)
#   shaders             vispy_renderer.py:56-105
#   read-back, depth    vispy_renderer.py:152-169 (on_draw)
# The reference hands the triangles to OpenGL (vispy/gloo); no GL exists in this container, so the rasterisation
# itself is a restatement of the OpenGL pipeline the reference configures: 176x176 viewport, depth test LESS, NO
# face culling (on_draw only calls set_cull_face, which selects the culled side; GL_CULL_FACE is never enabled),
# clear colour 0 / depth 1, smooth (perspective-correct) varyings, float->unorm8 colour conversion, and
# glReadPixels rows bottom-up taken as array rows top-down (which, with the y-flipped orthographic window, is an
# upright image).  PARITY UNPINNED for the rasterisation rules a GL implementation is free to choose (sub-pixel
# snapping: 8 bits here; tie rule on edges: top-left; depth-buffer format: float32 here).  The uniforms (window,
# projection matrix, view matrix, light direction) ARE pinned against the reference's own code
# (tests/golden/golden_render.npz, oracle/make_golden.py).
# Near-plane clipping (GL clips polygons at z_clip = -w): triangles in front of the eye are cut per pixel by the depth test;
# triangles crossing the eye plane take the homogeneous path in render_window (_straddler_setup).  The geometry of both is
# cross-checked against ray casting in tests/test_oracle_golden.py.
# =============================================================================================
GLCAM_IN_CVCAM = np.diag([1.0, -1.0, -1.0, 1.0])
NEAR_PLANE, FAR_PLANE = 0.1, 2.0
SUBPIXEL = 256


def render_uniforms(ob2cam, K, object_width):
    """-> dict(left,right,top,bottom, view32 (4,4) float32 [math convention: clip = P.V.p], proj64, proj32, light32)."""
    bbox = compute_bbox(ob2cam, K, object_width, scale=(1000, -1000, 1000))          # predict.py:202
    left, right = np.min(bbox[:, 1]), np.max(bbox[:, 1])                                # np.int32 scalars, as in the reference
    top, bottom = np.min(bbox[:, 0]), np.max(bbox[:, 0])
    ob2cam_gl = np.linalg.inv(GLCAM_IN_CVCAM).dot(ob2cam)                              # predict.py:203
    n, f = NEAR_PLANE, FAR_PLANE
    proj = np.array([[K[0, 0], 0, -K[0, 2], 0], [0, K[1, 1], -K[1, 2], 0], [0, 0, n + f, n * f], [0, 0, -1, 0]])
    with np.errstate(divide='ignore', invalid='ignore'):
        ortho = np.array([[2. / (right - left), 0, 0, -(right + left) / (right - left)],
                          [0, 2. / (top - bottom), 0, -(top + bottom) / (top - bottom)],
                          [0, 0, -2 / (f - n), -(f + n) / (f - n)], [0, 0, 0, 1]]).astype(np.float32)
    proj64 = ortho.dot(proj)                                                            # = projection_matrix.T
    light = np.dot(np.linalg.inv(ob2cam_gl.T), np.array([0, 0.1, -0.9, 1]))[:3]         # vispy_renderer.py:172
    return dict(left=int(left), right=int(right), top=int(top), bottom=int(bottom), view32=ob2cam_gl.astype(np.float32),
                proj64=proj64, proj32=proj64.astype(np.float32), light32=light.astype(np.float32))


def _project_vertices(pos32, view32, proj32, width, height):
    """float64 arithmetic on the float32 uniforms / attributes, fixed association (mirrored by render.cu)."""
    p = pos32.astype(np.float64); V = view32.astype(np.float64); P = proj32.astype(np.float64)
    v = [((V[i, 0] * p[:, 0] + V[i, 1] * p[:, 1]) + V[i, 2] * p[:, 2]) + V[i, 3] for i in range(4)]
    c = [((P[i, 0] * v[0] + P[i, 1] * v[1]) + P[i, 2] * v[2]) + P[i, 3] * v[3] for i in range(4)]
    w = c[3]
    with np.errstate(divide='ignore', invalid='ignore'):
        xw = (c[0] / w + 1.0) * (width * 0.5)
        yw = (c[1] / w + 1.0) * (height * 0.5)
        zw = (c[2] / w + 1.0) * 0.5
        X = np.rint(xw * SUBPIXEL); Y = np.rint(yw * SUBPIXEL)
    return X, Y, zw, w, c


def _near_clipped_box(cl, width, height):
    """Pixel box (ia, ib, ja, jb) that contains the part of a clip-space triangle beyond the near plane (z + w >= 0),
    one pixel of margin; the whole viewport when the arithmetic does not stay finite.  Only has to be conservative."""
    pts = []
    for a in range(3):
        b = (a + 1) % 3
        da, db = cl[a][2] + cl[a][3], cl[b][2] + cl[b][3]
        if da >= 0: pts.append((cl[a][0], cl[a][1], cl[a][3]))
        if (da >= 0) != (db >= 0):
            s = da / (da - db)
            pts.append(tuple(cl[a][k] + s * (cl[b][k] - cl[a][k]) for k in (0, 1, 3)))
    if not pts: return None
    with np.errstate(all='ignore'):
        xs = [(x / w + 1.0) * (width * 0.5) for x, y, w in pts]; ys = [(y / w + 1.0) * (height * 0.5) for x, y, w in pts]
    if not all(np.isfinite(v) and abs(v) < 1e9 for v in xs + ys): return 0, width - 1, 0, height - 1
    return (max(0, int(np.floor(min(xs))) - 1), min(width - 1, int(np.ceil(max(xs))) + 1),
            max(0, int(np.floor(min(ys))) - 1), min(height - 1, int(np.ceil(max(ys))) + 1))


def _straddler_setup(clip, i0, i1, i2, width, height):
    """Adjugate of M = [[x0 x1 x2], [y0 y1 y2], [w0 w1 w2]] (clip space), fixed association (mirrored by render.cu)."""
    cl = [tuple(float(clip[k][i]) for k in range(4)) for i in (i0, i1, i2)]
    if not all(np.isfinite(v) for c in cl for v in c): return None
    if all(c[2] + c[3] < 0 for c in cl): return None                                 # wholly on the eye side of the near plane
    box = _near_clipped_box(cl, width, height)
    if box is None or box[0] > box[1] or box[2] > box[3]: return None
    (x0, y0, z0, w0), (x1, y1, z1, w1), (x2, y2, z2, w2) = cl
    A = (y1 * w2 - y2 * w1, y2 * w0 - y0 * w2, y0 * w1 - y1 * w0)
    B = (x2 * w1 - x1 * w2, x0 * w2 - x2 * w0, x1 * w0 - x0 * w1)
    C = (x1 * y2 - x2 * y1, x2 * y0 - x0 * y2, x0 * y1 - x1 * y0)
    det = (x0 * A[0] + x1 * A[1]) + x2 * A[2]
    if det == 0 or not np.isfinite(det): return None
    return dict(idx=(i0, i1, i2), A=A, B=B, C=C, idet=1.0 / det, z=(z0, z1, z2), w=(w0, w1, w2), box=box)


def _rasterise(mesh, view32, proj32, width, height):
    """Visibility pass of the GL pipeline restated (see the header of this section): -> (key, setups, w).  key (height, width)
    uint64 = float32 window-z bits << 32 | triangle index (depth test LESS, first drawn wins ties), row 0 = window y 0 (bottom)."""
    X, Y, zw, w, clip = _project_vertices(mesh['pos'], view32, proj32, width, height)
    key = np.full((height, width), (np.uint64(0x3F800000) << np.uint64(32)) | np.uint64(0xFFFFFFFF), np.uint64)   # depth 1.0, no triangle
    faces = mesh['faces']
    lim = 1 << 25                      # render.cu evaluates the edge functions in float64: exact below 2^25 sub-pixels
    half = SUBPIXEL // 2
    setups = {}
    for t in range(len(faces)):
        i0, i1, i2 = (int(a) for a in faces[t])
        usable = all(w[i] > 1e-6 and np.isfinite(X[i]) and np.isfinite(Y[i]) and abs(X[i]) < lim and abs(Y[i]) < lim for i in (i0, i1, i2))
        if not usable:
            # A vertex at or behind the eye plane (or projected out of the exact-integer range): the screen-space set-up does
            # not exist.  GL clips such a triangle against the near plane; here it is rasterised in homogeneous coordinates
            # (weights beta = M^-1 (px, py, 1) with M the clip-space (x, y, w) columns -- inside iff all beta >= 0) and the
            # per-pixel depth test 0 <= z_window cuts it at the near plane, which is the same set of fragments.
            st = _straddler_setup(clip, i0, i1, i2, width, height)
            if st is None: continue
            ia, ib, ja, jb = st['box']
            px = ((2 * np.arange(ia, ib + 1) + 1 - width).astype(np.float64) / float(width))[None, :]
            py = ((2 * np.arange(ja, jb + 1) + 1 - height).astype(np.float64) / float(height))[:, None]
            with np.errstate(all='ignore'):
                beta = [((st['A'][k] * px + st['B'][k] * py) + st['C'][k]) * st['idet'] for k in range(3)]
                zc = (beta[0] * st['z'][0] + beta[1] * st['z'][1]) + beta[2] * st['z'][2]
                wc = (beta[0] * st['w'][0] + beta[1] * st['w'][1]) + beta[2] * st['w'][2]
                z32 = ((zc / wc + 1.0) * 0.5).astype(np.float32)
                ok = (beta[0] >= 0) & (beta[1] >= 0) & (beta[2] >= 0) & (z32 >= 0) & (z32 < 1)
            if not ok.any(): continue
            k = (z32.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(t)
            sub = key[ja:jb + 1, ia:ib + 1]
            upd = ok & (k < sub)
            sub[upd] = k[upd]
            setups[t] = st
            continue
        x0, y0, x1, y1, x2, y2 = (int(a) for a in (X[i0], Y[i0], X[i1], Y[i1], X[i2], Y[i2]))
        area2 = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0)
        if area2 == 0: continue
        if area2 < 0:                                                                    # no culling: make it counter-clockwise
            i1, i2, x1, y1, x2, y2, area2 = i2, i1, x2, y2, x1, y1, -area2
        ia, ib = max(0, (min(x0, x1, x2) - half + SUBPIXEL - 1) // SUBPIXEL), min(width - 1, (max(x0, x1, x2) - half) // SUBPIXEL)
        ja, jb = max(0, (min(y0, y1, y2) - half + SUBPIXEL - 1) // SUBPIXEL), min(height - 1, (max(y0, y1, y2) - half) // SUBPIXEL)
        if ia > ib or ja > jb: continue
        cx = (np.arange(ia, ib + 1, dtype=np.int64) * SUBPIXEL + half)[None, :]
        cy = (np.arange(ja, jb + 1, dtype=np.int64) * SUBPIXEL + half)[:, None]
        inside = np.ones((jb - ja + 1, ib - ia + 1), bool); E = []
        for (xa, ya, xb, yb) in ((x1, y1, x2, y2), (x2, y2, x0, y0), (x0, y0, x1, y1)):
            dx, dy = xb - xa, yb - ya
            e = dx * (cy - ya) - dy * (cx - xa)
            tl = (dy < 0) or (dy == 0 and dx < 0)                                       # top-left rule, y up, counter-clockwise
            inside &= (e > 0) | ((e == 0) & tl)
            E.append(e)
        if not inside.any(): continue
        inv_area = 1.0 / float(area2)                                                   # divisions only as reciprocals, like a GPU
        lam = [e.astype(np.float64) * inv_area for e in E]
        z = (lam[0] * zw[i0] + lam[1] * zw[i1]) + lam[2] * zw[i2]
        z32 = z.astype(np.float32)
        ok = inside & (z32 >= 0) & (z32 < 1)                                         # depth clip; LESS against the cleared 1.0
        k = (z32.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(t)
        sub = key[ja:jb + 1, ia:ib + 1]
        upd = ok & (k < sub)
        sub[upd] = k[upd]
        setups[t] = (i0, i1, i2, x0, y0, x1, y1, x2, y2, area2)
    return key, setups, w


def _fragment_weights(setup, w, i, j, width, height):
    """Perspective-correct (unnormalised) weights q0..q2 of the three vertices at pixel (i, j), and their vertex ids."""
    half = SUBPIXEL // 2
    if isinstance(setup, dict):                                                          # near-plane straddler: homogeneous weights
        i0, i1, i2 = setup['idx']
        px, py = float(2 * i + 1 - width) / float(width), float(2 * j + 1 - height) / float(height)
        q0, q1, q2 = (((setup['A'][k] * px + setup['B'][k] * py) + setup['C'][k]) * setup['idet'] for k in range(3))
        return (i0, i1, i2), (q0, q1, q2)
    i0, i1, i2, x0, y0, x1, y1, x2, y2, area2 = setup
    cx, cy = i * SUBPIXEL + half, j * SUBPIXEL + half
    e0 = (x2 - x1) * (cy - y1) - (y2 - y1) * (cx - x1)
    e1 = (x0 - x2) * (cy - y2) - (y0 - y2) * (cx - x2)
    e2 = (x1 - x0) * (cy - y0) - (y1 - y0) * (cx - x0)
    inv_area = 1.0 / float(area2)
    l0, l1, l2 = float(e0) * inv_area, float(e1) * inv_area, float(e2) * inv_area
    return (i0, i1, i2), (l0 * (1.0 / w[i0]), l1 * (1.0 / w[i1]), l2 * (1.0 / w[i2]))


def _interp_colour(mesh, ids, q):
    i0, i1, i2 = ids; q0, q1, q2 = q
    rq = 1.0 / ((q0 + q1) + q2)
    return [((q0 * float(np.float32(mesh['col'][i0, c] / 255.0)) + q1 * float(np.float32(mesh['col'][i1, c] / 255.0)))
             + q2 * float(np.float32(mesh['col'][i2, c] / 255.0))) * rq for c in range(3)]


def render_window(ob2cam, K, object_width, mesh, size=176, uniforms=None):
    """-> (rgb uint8 (size,size,3), depth uint16 (size,size) in mm, 0 = background).  mesh: dict(pos float32 (nv,3),
    nrm float32 (nv,3), col uint8 (nv,3), faces int32 (nf,3))."""
    u = uniforms if uniforms is not None else render_uniforms(ob2cam, K, object_width)
    rgb = np.zeros((size, size, 3), np.uint8); depth = np.zeros((size, size), np.uint16)
    if u['right'] == u['left'] or u['top'] == u['bottom'] or not np.all(np.isfinite(u['proj32'])):
        return rgb, depth
    key, setups, w = _rasterise(mesh, u['view32'], u['proj32'], size, size)
    A, B = u['proj64'][2, 2], u['proj64'][2, 3]
    far_dist = B / (A + 1)
    light = u['light32'].astype(np.float64)
    for j, i in zip(*np.nonzero((key & np.uint64(0xFFFFFFFF)) != np.uint64(0xFFFFFFFF))):
        t = int(key[j, i] & np.uint64(0xFFFFFFFF))
        (i0, i1, i2), (q0, q1, q2) = _fragment_weights(setups[t], w, i, j, size, size)
        rq = 1.0 / ((q0 + q1) + q2)
        def interp(a0, a1, a2): return ((q0 * a0 + q1 * a1) + q2 * a2) * rq
        pos = [interp(float(mesh['pos'][i0, c]), float(mesh['pos'][i1, c]), float(mesh['pos'][i2, c])) for c in range(3)]
        nrm = [interp(float(mesh['nrm'][i0, c]), float(mesh['nrm'][i1, c]), float(mesh['nrm'][i2, c])) for c in range(3)]
        col = _interp_colour(mesh, (i0, i1, i2), (q0, q1, q2))
        x = [(-light[c]) - pos[c] for c in range(3)]
        il = 1.0 / np.sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2])
        L = [x[c] * il for c in range(3)]
        d = (nrm[0] * L[0] + nrm[1] * L[1]) + nrm[2] * L[2]
        # max(d, 0) as the GPU's max instruction and C's fmax take it: a NaN term (a zero-length normal that load_ply_mesh
        # normalised to NaN) counts as 0, so the fragment gets the ambient 0.65 alone; Python's max would keep the NaN
        lightv = 0.4 * (d if d > 0.0 else 0.0) + 0.65
        for c in range(3):
            rgb[j, i, c] = np.uint8(np.rint(min(max(lightv * col[c], 0.0), 1.0) * 255.0))
        d32 = np.uint32(key[j, i] >> np.uint64(32)).view(np.float32)
        tt = np.float32(np.float32(d32 * np.float32(-2.0)) + np.float32(1.0))            # float32 array * python float stays float32
        dist = (B / (np.float64(tt) - A)) * -1                                          # `- A` with a float64 scalar: float64 (numpy >= 2)
        depth[j, i] = 0 if dist >= far_dist else np.uint16(dist * 1000)
    return rgb, depth


# ---------------------------------------------------------------------------------------------
# The reference's OTHER producer of input A: dataset_info['renderer'] == 'pyrenderer' (predict.py:161-164, 210-214;
# offscreen_renderer.py:47-83): pyrender renders the WHOLE camera image (IntrinsicsCamera fx fy cx cy, znear 0.1, zfar 2,
# ambient light 1 and no other light, background 0), the metric depth goes to uint16 mm and crop_bbox (Utils.py:320-359) cuts
# the 176 x 176 window out of both.  pyrender is a third-party package that is neither vendored in the reference nor installed
# here (reference docker/dockerfile: `pip install pyrender`, unpinned; 0.1.45 is the release of that time), so its part is
# restated from its published sources: camera.py IntrinsicsCamera.get_projection_matrix, renderer.py _read_main_framebuffer
# (depth linearisation), shaders/mesh.frag (colour = base colour * ambient when the scene has no lights).  PARITY UNPINNED,
# twice: the GL rasterisation rules (as above) and pyrender itself; per-fragment texture lookups (textured .obj) are replaced
# by per-vertex colours, as the reference's own vispy path does for the same models (predict.py:167-179).
# ---------------------------------------------------------------------------------------------
def pyrender_uniforms(ob2cam, K, H, W):
    n, f = NEAR_PLANE, FAR_PLANE
    P = np.zeros((4, 4))
    P[0, 0] = 2.0 * K[0, 0] / W; P[1, 1] = 2.0 * K[1, 1] / H
    P[0, 2] = 1.0 - 2.0 * K[0, 2] / W; P[1, 2] = 2.0 * K[1, 2] / H - 1.0
    P[3, 2] = -1.0
    P[2, 2] = (f + n) / (n - f); P[2, 3] = (2 * f * n) / (n - f)
    ob2cam_gl = np.linalg.inv(GLCAM_IN_CVCAM).dot(ob2cam)                              # offscreen_renderer.py:80
    return dict(view32=ob2cam_gl.astype(np.float32), proj32=P.astype(np.float32))


def render_full_frame_unlit(ob2cam, K, mesh, H, W):
    """-> (color uint8 (H,W,3), depth float32 (H,W) metres, 0 = background): what Renderer.render returns
    (offscreen_renderer.py:77-83), image rows top-down."""
    u = pyrender_uniforms(ob2cam, K, H, W)
    key, setups, w = _rasterise(mesh, u['view32'], u['proj32'], W, H)
    color = np.zeros((H, W, 3), np.uint8); depth = np.zeros((H, W), np.float32)
    zn, zf = np.float32(NEAR_PLANE), np.float32(FAR_PLANE)
    for j, i in zip(*np.nonzero((key & np.uint64(0xFFFFFFFF)) != np.uint64(0xFFFFFFFF))):
        t = int(key[j, i] & np.uint64(0xFFFFFFFF))
        ids, q = _fragment_weights(setups[t], w, i, j, W, H)
        col = _interp_colour(mesh, ids, q)
        r = H - 1 - j                                                                   # glReadPixels rows are bottom-up; pyrender flips them
        for c in range(3):
            color[r, i, c] = np.uint8(np.rint(min(max(col[c], 0.0), 1.0) * 255.0))
        d32 = np.uint32(key[j, i] >> np.uint64(32)).view(np.float32)
        zn_ = np.float32(np.float32(np.float32(2.0) * d32) - np.float32(1.0))            # float32 throughout, as numpy does on the float32 read-back
        depth[r, i] = np.float32(np.float32(np.float32(2.0) * zn * zf) / np.float32(np.float32(zf + zn) - np.float32(zn_ * np.float32(zf - zn))))
    return color, depth


def render_window_pyrender(ob2cam, K, object_width, mesh, H, W, size=176):
    """Tracker.render_window with the pyrender renderer (predict.py:210-214) -> (rgb uint8 (size,size,3), depth uint16 (size,size))."""
    bbox = compute_bbox(ob2cam, K, object_width, scale=(1000, 1000, 1000))
    rgb, depth = render_full_frame_unlit(ob2cam, K, mesh, H, W)
    depth = (depth * np.float32(1000)).astype(np.uint16)
    return crop_bbox(rgb, depth, bbox, (size, size))


# =============================================================================================
# Depth hole filling for live sensors (SURVEY.md 8f row 4): Utils.py:455-514 as predict_ros.py:38-41 calls it
#   depth_mm uint16 -> fill_depth(depth / 1e3, max_depth=2.0, extrapolate=False, blur_type='bilateral') -> (x * 1000).astype(uint16)
# Third-party arithmetic: cv2.dilate / morphologyEx / medianBlur / bilateralFilter, called directly (same library the
# reference calls; pinned by tests/golden/golden_fill.npz, which oracle/make_golden.py produces with the reference's own
# Utils.fill_depth).
# =============================================================================================
def fill_depth(depth, max_depth=2.0, extrapolate=False, blur_type='bilateral'):
    """Utils.py:455-514.  depth: metres (any float dtype) -> float32 metres."""
    depth = np.asarray(depth).astype(np.float32)
    diamond = np.array([[0, 0, 1, 0, 0], [0, 1, 1, 1, 0], [1, 1, 1, 1, 1], [0, 1, 1, 1, 0], [0, 0, 1, 0, 0]], dtype=np.uint8)
    valid = depth > 0.1
    depth[valid] = max_depth - depth[valid]                      # invert so that dilation prefers near surfaces
    depth = cv2.dilate(depth, diamond)
    depth = cv2.morphologyEx(depth, cv2.MORPH_CLOSE, np.ones((5, 5), np.uint8))
    empty = depth < 0.1
    dilated = cv2.dilate(depth, np.ones((7, 7), np.uint8))
    depth[empty] = dilated[empty]
    if extrapolate:                                              # Utils.py:486-497
        top_row = np.argmax(depth > 0.1, axis=0)
        top_val = depth[top_row, range(depth.shape[1])]
        for col in range(depth.shape[1]):
            depth[0:top_row[col], col] = top_val[col]
        empty = depth < 0.1
        dilated = cv2.dilate(depth, np.ones((31, 31), np.uint8))
        depth[empty] = dilated[empty]
    depth = cv2.medianBlur(depth, 5)
    if blur_type == 'bilateral':
        depth = cv2.bilateralFilter(depth, 5, 1.5, 2.0)
    elif blur_type == 'gaussian':                                # Utils.py:506-510
        valid = depth > 0.1
        blurred = cv2.GaussianBlur(depth, (5, 5), 0)
        depth[valid] = blurred[valid]
    valid = depth > 0.1
    depth[valid] = max_depth - depth[valid]
    return depth


def fill_depth_mm(depth_mm, extrapolate=False, blur_type='bilateral'):
    """predict_ros.py:38-41: uint16 millimetres in, uint16 millimetres out."""
    d = fill_depth(np.asarray(depth_mm).astype(np.uint16) / 1e3, max_depth=2.0, extrapolate=extrapolate, blur_type=blur_type)
    return (d * 1000).astype(np.uint16), d
