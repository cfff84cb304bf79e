"""Drop-in for the Tracker of the reference's predict.py (reference predict.py:127-296): same
constructor, attributes and on_track signature, so the reference's sequence drivers
(predict.py:299-624) and predict_ros.py:59 can call it unchanged -- with the per-frame work
(crop, depth clip, normalise, 17-conv network, pose update) running as one stream of libse3tn
kernels instead of numpy + torch.nn.

Differences, all additive:
  * on_track(..., rgbA=None, depthA=None): the rendered previous view may be passed in.  The
    OpenGL renderers (vispy_renderer.py / offscreen_renderer.py) are out of scope; when they are
    importable the Tracker uses them exactly as the reference does, otherwise rgbA/depthA (or a
    `renderer=` object with render_window(ob2cam)) must be supplied.
  * the second, visualisation-only render + cv2.imshow (predict.py:284-290) only happens with
    show=True.
  * on_track_batch(): N independent tracks of one frame in one batched launch sequence (the
    reference is batch 1, F15).  Numpy frames and poses take the host route: one se3tn_track_host /
    se3tn_track_render_host call that returns numpy poses.  Tensors and mixed inputs take the device
    route: CUDA tensors are used as they are, every other input is staged through one double-buffered
    set, and one se3tn_track_batch / se3tn_track_render step is enqueued.
  * Tracker(..., fill_depth=True): on_track takes a live sensor's raw depth frame and hole-fills it
    inside the tracking step, as the reference's ROS node does with Utils.fill_depth before every
    on_track (predict_ros.py:38-41).
  * Tracker(..., iterations=k): each frame refines every track k times inside one tracking step, exactly as k chained on_track
    calls would (the CUDA rasteriser draws input A at each round's pose).
"""
import collections
import contextlib
import os
import random
import numpy as np
import torch

from . import _lib
from . import engine as _engine            # the class itself: tests stand in for Engine, not for its static checks
from .engine import Engine, check_weight_sets_fit
from .cuda_renderer import CudaRenderer
from .se3_tracknet import Se3TrackNet
from .datasets import TrackDataset
from .staging import StagingRing, VideoSink
from . import Utils as U

_refine_iterations = Engine.refine_iterations      # the drivers check counts before any Engine exists
# Tracker(fit=True)'s tau: a starting guess for a sensor's depth noise at a metre or so, not measured on a real sensor
FIT_TAU_DEFAULT = 10

# The per-step options of a Tracker or a driver run, as step_options checks them: fit the tau in mm whose rows the caller keeps
# (None: none), tau the step's fit check in mm (None: off), icp Engine.icp_spec's argument (None: off), hypotheses S and the seed
# of their draws, reinit reinit_options' value (None: off).  A tuple, so the spawned ranks of a multi-GPU run receive it in their
# process arguments.
StepOptions = collections.namedtuple('StepOptions', 'fit tau icp hypotheses seed reinit', defaults=(None,))


def step_options(fit=None, hypotheses=1, seed=0, icp=None, icp_tau=None, fit_switch=False, reinit=None):
    """The options of every tracking step -> StepOptions, or a ValueError, checked in this order:
    fit       None or a tau in mm (Engine.fit_spec).  fit_switch (the Tracker's fit) also takes True, FIT_TAU_DEFAULT mm, and
              False, off, which refuses hypotheses.
    hypotheses  S, an integer in [1, MAX_HYPOTHESES]; seed an integer.
    icp       None / 0 off, or M iterations or a dict (Engine.icp_spec); icp_tau the gate in mm, refused without icp.  ICP inside
              hypothesis steps is not supported: refused with S > 1.
    S > 1 ranks the starts by the fit check, so the step's tau is fit, or FIT_TAU_DEFAULT when fit is None.
    reinit    None off, or reinit_options' argument: re-initialise lost tracks after every step.  It ranks starts by the fit check
              as hypotheses do: the step's tau is then fit or FIT_TAU_DEFAULT, and fit_switch's False is refused."""
    off = fit_switch and fit is False
    if fit_switch and isinstance(fit, bool):
        fit = FIT_TAU_DEFAULT if fit else None
    fit = _engine.Engine.fit_spec(fit) or None
    if isinstance(hypotheses, (bool, np.bool_)) or not isinstance(hypotheses, (int, np.integer)) or \
            not 1 <= hypotheses <= _lib.MAX_HYPOTHESES:
        raise ValueError('hypotheses must be an integer in [1, %d], not %r' % (_lib.MAX_HYPOTHESES, hypotheses))
    if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, (int, np.integer)):
        raise ValueError('seed must be an integer, not %r' % (seed,))
    if icp_tau is not None:
        if not icp:
            raise ValueError('icp_tau %r without icp: the gate of ICP iterations that do not run' % (icp_tau,))
        icp = {'iterations': icp, 'tau_mm': icp_tau}
    if _engine.Engine.icp_spec(icp) is None:
        icp = None
    elif hypotheses > 1:
        raise ValueError('icp %r with hypotheses %d: ICP inside hypothesis steps is not supported' % (icp, hypotheses))
    if off and hypotheses > 1:
        raise ValueError('hypotheses=%d ranks the starts by the fit check: fit must not be off' % hypotheses)
    reinit = reinit_options(reinit)
    if off and reinit is not None:
        raise ValueError('reinit ranks a start against the tracked pose by the fit check: fit must not be off')
    tau = fit or (FIT_TAU_DEFAULT if hypotheses > 1 or reinit is not None else None)
    return StepOptions(fit, tau, icp, int(hypotheses), int(seed), reinit)


def reinit_options(reinit):
    """Tracker(reinit=)'s value -> None (off) or a dict {'below', 'after', 'init'}: below the inlier fraction and after the frames
    in a row below it that make a track lost (Engine.reinit_spec; defaults Engine.REINIT_DEFAULTS), init Engine.init_spec's
    fields for the restart (None: its defaults).  Anything else is a ValueError."""
    if reinit is None:
        return None
    if not isinstance(reinit, dict):
        raise ValueError('reinit must be None or a dict of below, after and init, not %r' % (reinit,))
    unknown = set(reinit) - {'below', 'after', 'init'}
    if unknown:
        raise ValueError('reinit: unknown fields %s' % sorted(unknown))
    spec = dict(_engine.Engine.REINIT_DEFAULTS, init=None)
    spec.update(reinit)
    _engine.Engine.reinit_spec(spec['below'], spec['after'])
    _engine.Engine.init_spec(spec['init'])
    return spec


def reinit_keep(opts):
    """The tracks per restarted track an Engine must hold for opts' re-initialisation (its init keep), 1 without it."""
    return 1 if opts.reinit is None else Engine.init_spec(opts.reinit['init']).keep


def hypothesis_spread(info, opts, label=None):
    """The spread a class's start hypotheses are drawn with: its dataset_info's (max_translation m, max_rotation degrees), the
    bounds its training pairs were drawn with; None when opts has no hypotheses.  A ValueError, prefixed with `label`, when either
    is missing or Engine.hypothesis_spec refuses it."""
    if opts.hypotheses == 1:
        return None
    try:
        spread = float(info['max_translation']), float(info['max_rotation'])
        _engine.Engine.hypothesis_spec(opts.hypotheses, opts.seed, *spread)
    except (KeyError, TypeError, ValueError) as e:
        raise ValueError('%sdataset_info max_translation / max_rotation: %s' % ('' if label is None else label + ': ', e)) from e
    return spread


def fit_fractions(rows):
    """The derived numbers of fit-check rows (Engine.track_render's fit; (..., 6) int32: model, observed, inlier, front, behind,
    residual) -> dict of float64 arrays of the leading shape: 'inlier' inlier / model, 'front' front / model, 'behind' behind / model,
    'residual' residual / inlier in mm (the mean inlier residual).  Each is 0 where its denominator is 0.  Rows of -1 (a frame
    that was not tracked) give NaN."""
    r = rows.cpu().numpy() if torch.is_tensor(rows) else np.asarray(rows)
    r = r.astype(np.float64)
    div = lambda a, b: np.divide(a, b, out=np.zeros_like(a), where=b > 0)
    out = {'inlier': div(r[..., 2], r[..., 0]), 'front': div(r[..., 3], r[..., 0]), 'behind': div(r[..., 4], r[..., 0]),
           'residual': div(r[..., 5], r[..., 2])}
    untracked = (r == -1).all(axis=-1)
    for v in out.values():
        v[untracked] = np.nan
    return out


class PointCloud:
    """Minimal stand-in for the open3d point cloud the reference keeps in Tracker.object_cloud
    (predict.py:131-133): callers only read `.points`."""
    def __init__(self, points):
        self.points = np.asarray(points, dtype=np.float64)

    def voxel_down_sample(self, voxel_size):
        # open3d semantics: points are bucketed on a grid anchored at (min_bound - voxel/2) and each
        # occupied voxel is replaced by the mean of its points
        pts = self.points
        origin = pts.min(0) - voxel_size * 0.5
        keys = np.floor((pts - origin) / voxel_size).astype(np.int64)
        _, inv = np.unique(keys, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        sums = np.zeros((inv.max() + 1, 3)); np.add.at(sums, inv, pts)
        cnt = np.bincount(inv).astype(np.float64)[:, None]
        return PointCloud(sums / cnt)


def load_vertices(model_path, merge=True):
    """Vertices of a .ply (ascii / binary little endian) or .obj mesh, as trimesh.load(..).vertices gives them to the
    reference (predict.py:131).  trimesh loads with process=True, which MERGES duplicate vertices (positions equal to its
    tol.merge = 1e-8); duplicates would otherwise weigh twice in the voxel means of voxel_down_sample and move the
    convex-hull diameter -> object_width -> crop window.  merge=True reproduces that (first occurrence kept, file order)."""
    ext = os.path.splitext(model_path)[1].lower()
    if ext == '.obj':
        v = [list(map(float, l.split()[1:4])) for l in open(model_path) if l.startswith('v ')]
        pts = np.asarray(v, dtype=np.float64)
    elif ext == '.ply':
        pts = _ply_vertices(model_path)
    else:
        raise ValueError('unsupported mesh format: ' + model_path)
    if merge and len(pts):
        key = np.round(pts / 1e-8).astype(np.int64)
        _, first = np.unique(key, axis=0, return_index=True)
        pts = pts[np.sort(first)]
    return pts


def _ply_vertices(model_path):
    with open(model_path, 'rb') as f:
        fmt, nvert, props, in_vertex = None, 0, [], False
        while True:
            line = f.readline().decode('ascii', 'replace').strip()
            if line.startswith('format'):
                fmt = line.split()[1]
            elif line.startswith('element'):
                in_vertex = line.split()[1] == 'vertex'
                if in_vertex:
                    nvert = int(line.split()[2])
            elif line.startswith('property') and in_vertex:
                props.append((line.split()[1], line.split()[-1]))
            elif line == 'end_header':
                break
        names = [p[1] for p in props]
        ix = [names.index(a) for a in 'xyz']
        if fmt == 'ascii':
            data = np.loadtxt(f, max_rows=nvert, ndmin=2)
            return data[:, ix].astype(np.float64)
        np_t = {'float': '<f4', 'float32': '<f4', 'double': '<f8', 'float64': '<f8', 'uchar': 'u1', 'uint8': 'u1',
                'char': 'i1', 'int': '<i4', 'int32': '<i4', 'uint': '<u4', 'short': '<i2', 'ushort': '<u2'}
        dt = np.dtype([(n, np_t[t]) for t, n in props])
        data = np.frombuffer(f.read(dt.itemsize * nvert), dtype=dt, count=nvert)
        return np.stack([data['x'], data['y'], data['z']], 1).astype(np.float64)


def object_cloud(model_path):
    """Tracker.object_cloud of a mesh file: its vertices down-sampled on a 5 mm voxel grid (reference predict.py:131-133)."""
    return PointCloud(load_vertices(model_path)).voxel_down_sample(voxel_size=0.005)


def compute_obj_max_width(points):
    """Convex-hull diameter in mm (reference Utils.py:101-105, 450-451)."""
    from scipy.spatial import ConvexHull, distance_matrix
    hull = points[ConvexHull(points).vertices]
    return float(np.max(distance_matrix(hull, hull))) * 1000


def _as_numpy_pose(p):
    return np.ascontiguousarray(p, dtype=np.float64)


class Tracker:
    def __init__(self, dataset_info, images_mean, images_std, ckpt_dir, model_path=None, trans_normalizer=0.03,
                 rot_normalizer=5 * np.pi / 180, engine=None, weight_id=0, renderer=None, precision='bf16x3', max_batch=64,
                 fill_depth=False, iterations=1, fit=None, hypotheses=1, seed=0, icp=None, reinit=None):
        """fill_depth: the depth frames given to on_track / on_track_batch are raw sensor frames, hole-filled inside every
        tracking step.  True is the reference ROS node's fill_depth(depth, max_depth=2.0); a dict sets max_depth / extrapolate
        / blur_type (Engine.depth_fill_spec).
        iterations: on_track / on_track_batch refine every track k times on each frame, in one tracking step (Engine.track_render),
        exactly as k chained calls with iterations=1 would.  k > 1 needs the CUDA rasteriser drawing input A inside the step: a
        reference GL renderer is a ValueError here, and input A passed to a call is a ValueError there.
        fit: the fit check of every tracking step (Engine.track_render's fit): None / False off, True FIT_TAU_DEFAULT mm, or tau in
        mm (1..1000).  on_track / on_track_batch then leave the frame's rows (model, observed, inlier, front, behind, residual per
        track) in last_fit: numpy on the host route, an int32 CUDA tensor on the device route; fit_fractions turns them into
        fractions.  Like iterations > 1 it needs the CUDA rasteriser drawing input A inside the step.
        hypotheses: S in [1, 32].  S > 1 tracks every track from S starts per frame, its previous pose and S - 1 poses drawn
        around it with the spread the network's training pairs were drawn with (dataset_info['max_translation'] m,
        ['max_rotation'] degrees), and keeps the one whose model fits the frame best (Engine.track_hypotheses).  It turns the fit
        check on at FIT_TAU_DEFAULT mm when fit is not given, and needs the CUDA rasteriser as fit does.  last_fit then holds the
        kept rows and last_choice the kept hypotheses.  Hypothesis h of track j in the Tracker's c-th call is drawn with key
        (seed, c, j).  A Tracker that builds its Engine sizes it max_batch x S; a shared Engine must hold n x S tracks per call.
        S = 1 is the plain step (last_choice stays None).
        icp: depth refinement after the network's last round (Engine.track_render's icp): None / 0 off, M iterations of
        point-to-plane ICP at Engine.icp_spec's default gate, or a dict of its fields.  on_track / on_track_batch then leave the
        last iteration's stats (inliers, rms_mm, step_mm, step_deg per track) in last_icp: numpy on the host route, a float64
        CUDA tensor on the device route.  Like fit it needs the CUDA rasteriser drawing input A inside the step; it is refused
        with hypotheses > 1.  fit, hypotheses, seed, icp and reinit are checked by step_options and kept in opts.
        reinit: None off, or a dict {'below': f, 'after': L, 'init': {Engine.init_spec's fields}} (reinit_options): after every
        step, a track whose inlier fraction stayed below f for L frames in a row is restarted from its mask
        (Engine.reinit) when on_track / on_track_batch are given the frame's mask or label image, and the start replaces the
        tracked pose only when it fits the frame better.  The event codes of the frame's tracks (0 not below, 1 below, 2
        restarted, 3 no start, 4 start rejected) are left in last_reinit.  Each track index keeps its streak of frames below
        across calls; a call with another number of tracks, or reset_reinit(), starts them from 0.  Like hypotheses it turns the
        fit check on at FIT_TAU_DEFAULT mm when fit is not given, and needs the CUDA rasteriser; a Tracker that builds its
        Engine sizes it for max_batch x init keep tracks, which one restart of every track needs.  Each frame with reinit on
        synchronises once, to read which tracks are lost."""
        Engine.depth_fill_spec(fill_depth)                 # a bad value fails here, not at the first frame
        self.iterations = Engine.refine_iterations(iterations)
        self.opts = step_options(fit, hypotheses, seed, icp, fit_switch=True, reinit=reinit)
        self.reinit = self.opts.reinit
        self._streak = None                                # reinit: the tracks' streaks on the device, per track index
        self.fit, self.icp, self.hypotheses, self.seed = self.opts.tau, self.opts.icp, self.opts.hypotheses, self.opts.seed
        self.spread = hypothesis_spread(dataset_info, self.opts)
        self._calls = 0                                    # the c of the draw keys (seed, c, j)
        self.last_fit = self.last_icp = self.last_choice = self.last_init = self.last_reinit = None
        self.fill_depth = fill_depth
        self.dataset_info = dataset_info
        self.image_size = (dataset_info['resolution'], dataset_info['resolution'])
        if self.image_size[0] != 176:
            raise NotImplementedError('libse3tn is built for the reference resolution of 176 (dataset_info.yml:15)')
        self.object_cloud = None
        if model_path is not None:
            self.object_cloud = object_cloud(model_path)
        if 'object_width' not in dataset_info:
            if self.object_cloud is None:
                raise ValueError("need model_path or dataset_info['object_width']")
            w = compute_obj_max_width(np.asarray(self.object_cloud.points))
            self.object_width = w + dataset_info['boundingbox'] / 100 * w
        else:
            self.object_width = dataset_info['object_width']
        self.mean = images_mean
        self.std = images_std
        cam_cfg = dataset_info['camera']
        self.K = np.array([cam_cfg['focalX'], 0, cam_cfg['centerX'], 0, cam_cfg['focalY'], cam_cfg['centerY'], 0, 0, 1]).reshape(3, 3)

        if isinstance(ckpt_dir, dict):
            checkpoint = ckpt_dir if 'state_dict' in ckpt_dir else {'state_dict': ckpt_dir}
        else:
            checkpoint = torch.load(ckpt_dir, map_location='cpu')
        keep = reinit_keep(self.opts)
        if engine is not None and self.reinit is not None and engine.max_batch < keep:
            raise ValueError('reinit restarts a lost track with init keep=%d candidates, more than the engine\'s max_batch=%d'
                             % (keep, engine.max_batch))
        self.engine = engine if engine is not None else Engine(max_batch=max_batch * max(self.hypotheses, keep))
        self.weight_id = weight_id
        self.precision = precision
        self.model = Se3TrackNet(image_size=self.image_size[0], engine=self.engine, weight_id=weight_id, precision=precision)
        self.model.load_state_dict(checkpoint['state_dict'])
        self.model = self.model.cuda()
        self.model.eval()
        self.engine.set_stats(np.asarray(images_mean), np.asarray(images_std), weight_id)
        U.set_engine(self.engine)

        # Input A.  renderer='cuda' (or nothing, with a .ply model that has normals + colours): the CUDA rasteriser
        # (csrc/render.cu) -- no OpenGL, all tracks in one launch.  Otherwise an object with render_window(ob2cam), or the
        # reference's own OpenGL renderers when they are importable.
        # dataset_info['renderer'] == 'pyrenderer' selects the reference's pyrender producer (predict.py:161-164): the rasteriser's
        # unlit full-camera-image mode followed by crop_bbox; anything else its vispy producer.
        pyr = dataset_info.get('renderer') == 'pyrenderer'
        if renderer == 'cuda' or (renderer is None and model_path is not None and str(model_path).lower().endswith(('.ply', '.obj') if pyr else '.ply')):
            try:
                renderer = CudaRenderer(model_path, self.K, self.engine, self.object_width, mesh_id=weight_id,
                                        mode='pyrender' if pyr else 'vispy', image_hw=(cam_cfg['height'], cam_cfg['width']) if pyr else None)
            except ValueError:
                if renderer == 'cuda':
                    raise
                renderer = None                                    # e.g. a vertices-only ply: fall through to the GL renderers
        self.renderer = renderer if renderer is not None else self._try_reference_renderer(model_path, cam_cfg)
        if not isinstance(self.renderer, CudaRenderer):
            self._check_step_draws(why='it needs the CUDA renderer (renderer="cuda"), not %r' % (self.renderer,))
        self._np_bufs = {}
        self._copy_stream = torch.cuda.Stream(device=self.engine.device)      # _uploads: two staging slots, used alternately
        self._stage_bufs = ({}, {})
        self._stage_done = (torch.cuda.Event(), torch.cuda.Event())
        self._stage_slot = 0
        self.prev_rgb = None
        self.prev_depth = None
        self.frame_cnt = 0
        self.errs = []
        self.trans_normalizer = trans_normalizer
        self.rot_normalizer = rot_normalizer
        self.dataset = TrackDataset('', 'eval', images_mean, images_std, None, None, None, dataset_info,
                                    trans_normalizer=trans_normalizer, rot_normalizer=rot_normalizer,
                                    engine=self.engine, weight_id=weight_id, precision=precision)
        self.dataset._stats_set = True

    # ------------------------------------------------------------------ renderer glue (out-of-scope producer)
    def _try_reference_renderer(self, model_path, cam_cfg):
        """The reference picks pyrender or vispy by dataset_info['renderer'] (predict.py:161-182).
        Both are OpenGL stacks outside this package; use them if the user's environment has them."""
        if model_path is None:
            return None
        try:
            if self.dataset_info.get('renderer') == 'pyrenderer':
                from offscreen_renderer import Renderer            # reference module, if on sys.path
            else:
                from vispy_renderer import VispyRenderer           # reference module, if on sys.path
        except ImportError:
            return None                                            # no OpenGL stack in this environment: rgbA/depthA must be passed in
        # the renderer module IS there: a failure to construct it (no GL context, bad mesh) is the user's to see
        if self.dataset_info.get('renderer') == 'pyrenderer':
            return Renderer([model_path], self.K, cam_cfg['height'], cam_cfg['width'])
        return VispyRenderer(model_path, self.K, H=self.dataset_info['resolution'], W=self.dataset_info['resolution'])

    def render_window(self, ob2cam):
        """rgb u8 (176,176,3), depth u16 mm (176,176) of the model at `ob2cam` inside the crop window
        (reference predict.py:193-215)."""
        r = self.renderer
        if r is None:
            raise RuntimeError('no renderer available: pass rgbA/depthA to on_track, or renderer= to Tracker')
        if hasattr(r, 'render_window'):
            return r.render_window(ob2cam)
        glcam_in_cvcam = np.diag([1.0, -1.0, -1.0, 1.0])
        if hasattr(r, 'update_cam_mat'):                           # vispy-style
            bbox = U.compute_bbox(ob2cam, self.K, self.object_width, scale=(1000, -1000, 1000))
            ob2cam_gl = np.linalg.inv(glcam_in_cvcam).dot(ob2cam)
            r.update_cam_mat(self.K, np.min(bbox[:, 1]), np.max(bbox[:, 1]), np.max(bbox[:, 0]), np.min(bbox[:, 0]))
            return r.render_image(ob2cam_gl)
        bbox = U.compute_bbox(ob2cam, self.K, self.object_width, scale=(1000, 1000, 1000))
        rgb, depth = r.render([ob2cam])
        return U.crop_bbox(rgb, (depth * 1000).astype(np.uint16), bbox, self.image_size)

    def _fused_renderer(self, weight_ids=None, renderer_width=False):
        """The CudaRenderer when the tracking step can render input A itself and draw exactly what rendering it first would,
        else None.  The step draws with the Tracker's engine, camera and widths, and track i draws the model of its weight id.
        A renderer on another engine, with another K, drawing another model without per-track ids, or (renderer_width:
        Tracker.render_window draws at the renderer's own width) with another width renders input A first, as before."""
        r = self.renderer
        if not isinstance(r, CudaRenderer) or r.engine is not self.engine or not np.array_equal(r.K, self.K):
            return None
        if weight_ids is None and r.mesh_id != self.weight_id:
            return None
        if renderer_width and r.object_width != float(self.object_width):
            return None
        return r

    # ------------------------------------------------------------------ a start without a pose
    def initialize(self, depth, mask=None, label=1, box=None, depths=Engine.INIT_BOX_DEPTHS, **init):
        """The start pose of this Tracker's object from its mask or its 2D box and the depth frame (Engine.init_poses /
        Engine.init_boxes), with the Tracker's mesh, width and render mode.  Exactly one of mask and box.  depth: uint16 (H,W)
        mm, numpy or CUDA; mask: a bool (H,W) array (the object's pixels) or a uint8 label image in which the object's pixels
        are `label`; box: a detector's (x0, y0, x1, y1) in frame pixels, floats allowed, rounded outwards (floor x0 / y0, ceil
        x1 / y1) and clipped to the frame (Engine.box_pixels); depths: init_boxes' depth candidates.  init: Engine.init_spec's
        fields.  A Tracker built with fill_depth fills the depth first with the same settings, so the start is scored on the
        depth its steps see.  -> the 4x4 float64 start on_track takes; the kept score row (status, candidate, model, maskc,
        overlap, pairs, inlier, delta_mm) is left in last_init.  A ValueError names the status when there is no start (an
        empty mask or box, too few pixels with depth)."""
        if (mask is None) == (box is None):
            raise ValueError('initialize: give exactly one of mask and box')
        r = self._fused_renderer()
        if r is None:
            raise ValueError('initialize draws the model on the device: it needs the CUDA renderer (renderer="cuda") on this '
                             "Tracker's engine and camera, not %r" % (self.renderer,))
        dev = self.engine.device
        as_dev = lambda a, dt: a.to(dev, dt).contiguous() if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
        depth_d = as_dev(depth, np.uint16 if not torch.is_tensor(depth) else torch.uint16)
        seg, labels, boxes = self._object_pixels('initialize', mask, label, box, *depth_d.shape)
        on, max_depth, extrapolate, blur = Engine.depth_fill_spec(self.fill_depth)
        if on:
            depth_d = self.engine.fill_depth(depth_d, max_depth, extrapolate=bool(extrapolate), blur_type='gaussian' if blur else 'bilateral')
        width = torch.full((1,), float(self.object_width), dtype=torch.float64, device=dev)
        common = dict(weight_ids=None if r.mesh_id == 0 else [r.mesh_id], mode=r.mode, image_hw=r.image_hw, init=init or None)
        if boxes is None:
            poses, rows = self.engine.init_poses(depth_d, as_dev(seg, seg.dtype), self.K, labels, width, **common)
        else:
            poses, rows = self.engine.init_boxes(depth_d, boxes, self.K, width, depths=depths, **common)
        self.last_init = rows[0].cpu().numpy()
        status = int(self.last_init[0])
        if status:
            what, source = ('label %d' % label, 'mask') if boxes is None else ('box %s' % (tuple(int(x) for x in boxes[0]),), 'box')
            raise ValueError('initialize: no start for %s: %s (status %d)' % (what, Engine.init_status(status, source), status))
        return poses[0].cpu().numpy()

    @staticmethod
    def _object_pixels(fn, mask, label, box, H, W):
        """One object's pixels in an H x W frame as on_track_batch's seg, labels and boxes, nothing copied to the device: mask, a
        bool (H,W) mask or an integer label image with labels 0..255 (numpy or a tensor), as a uint8 label image in which the
        object is `label`; box, a detector's (x0, y0, x1, y1) as Engine.box_pixels rounds and clips it; neither, all None."""
        if mask is not None and box is not None:
            raise ValueError('%s: give mask or box, not both' % fn)
        if mask is None:
            return None, None, (None if box is None else Engine.box_pixels(box, H, W)[None])
        m = mask if torch.is_tensor(mask) else np.asarray(mask)
        if torch.is_tensor(m) and m.dtype == torch.bool:
            seg = m.to(torch.uint8) * int(label)
        elif not torch.is_tensor(m) and m.dtype == np.bool_:
            seg = np.where(m, np.uint8(label), np.uint8(0))
        else:
            lo, hi = (int(m.min()), int(m.max())) if (m.numel() if torch.is_tensor(m) else m.size) else (0, 0)
            if lo < 0 or hi > 255:
                raise ValueError('%s: mask must be a bool mask or a uint8 label image (any integer type, labels 0..255), not %s '
                                 'with labels %d..%d' % (fn, m.dtype, lo, hi))
            seg = m.to(torch.uint8) if torch.is_tensor(m) else m.astype(np.uint8, copy=False)
        if tuple(seg.shape) != (H, W):
            raise ValueError('%s: mask %s and depth %s differ in shape' % (fn, tuple(seg.shape), (H, W)))
        return seg, [int(label)], None

    # ------------------------------------------------------------------ the hot path
    def on_track(self, prev_pose, current_rgb, current_depth, gt_A_in_cam=None, gt_B_in_cam=None, debug=False, samples=1,
                 rgbA=None, depthA=None, show=False, mask=None, label=1, box=None):
        """One frame, one object (reference predict.py:217-296) -> new 4x4 float64 pose.  Without rgbA / depthA and with the
        CUDA rasteriser, input A is rendered inside the tracking step itself (se3tn_track_render_host), and refined
        Tracker.iterations times.  mask: with reinit, the object's pixels of this frame, a bool (H,W) array or a label image
        in which they are `label`, as Tracker.initialize takes them; read only when the track is lost.  box: with reinit, instead of mask, the object's
        (x0, y0, x1, y1) box in this frame (Tracker.initialize's rounding): a lost track restarts from it (Engine.init_boxes)."""
        A_in_cam = _as_numpy_pose(prev_pose).copy()
        seg, labels, boxes = self._object_pixels('on_track', mask, label, box, *np.shape(current_depth)[:2])
        kw = dict(seg=seg, labels=labels, boxes=boxes)                 # read by on_track_batch only with reinit
        fused = (rgbA is None or depthA is None) and self._fused_renderer(renderer_width=True) is not None
        if not fused:
            self._check_step_draws(rgbA is not None or depthA is not None)
        if fused:
            out = self.on_track_batch(A_in_cam[None], current_rgb, current_depth, **kw)
        else:
            if rgbA is None or depthA is None:
                rgbA, depthA = self.render_window(A_in_cam)
            out = self.on_track_batch(A_in_cam[None], current_rgb, current_depth,
                                      np.ascontiguousarray(rgbA, dtype=np.uint8)[None],
                                      np.ascontiguousarray(depthA).astype(np.uint16)[None], **kw)
        final_estimate = out[0]
        self.prev_rgb = current_rgb
        self.prev_depth = current_depth
        if show:
            import cv2
            pred_color, _ = self.render_window(final_estimate)
            cv2.imshow('AB', pred_color[..., ::-1])
            cv2.waitKey(1)
        self.frame_cnt += 1
        return final_estimate

    def on_track_batch(self, prev_poses, current_rgb, current_depth, rgbA=None, depthA=None, weight_ids=None, object_width=None,
                       seg=None, labels=None, boxes=None):
        """N independent tracks of ONE frame -> (N,4,4) float64.  rgbA / depthA None: rendered on the device by the CUDA
        rasteriser (needs a CudaRenderer; per-track models follow weight_ids), inside the tracking step when the renderer
        allows it (_fused_renderer).  The types of the inputs pick one of two routes:

        host    numpy frame and poses (ids and widths not tensors), input A numpy or drawn inside the step: one
                Engine.track_host / track_render_host call stages the frame's crop-window rectangle, the poses and input A
                through pinned memory and returns numpy poses (synchronous, like the reference's on_track).
        device  everything else.  CUDA tensors are used as they are; every other input (numpy arrays, pageable or pinned
                CPU tensors) is staged through one double-buffered set (_uploads).  Input A is rendered first when the step
                cannot draw it, and one Engine.track_render / track_batch call is enqueued.  Tensor poses give a CUDA
                tensor and nothing is synchronised; numpy poses give a numpy result.
        A pageable input may be overwritten as soon as the call returns.  A pinned CPU tensor is read asynchronously: it must
        stay unchanged until the current stream has run this call's step.
        seg / labels: with reinit, the frame's uint8 (H,W) label image (numpy or a tensor) and each track's label in it (ints
        in 1..255; None with one track: 1), read only when a track is lost (_reinit).  boxes: instead of seg / labels, each
        track's (x0, y0, x1, y1) box in this frame, ints (n, 4) (Engine.init_boxes).  Without seg or boxes no track is
        restarted."""
        if self.reinit is None:
            return self._track_step(prev_poses, current_rgb, current_depth, rgbA, depthA, weight_ids, object_width)
        n = len(prev_poses)
        labels = [1] if labels is None and n == 1 else labels
        Engine.reinit_source('on_track_batch', n, seg, labels, boxes)
        if n * reinit_keep(self.opts) > self.engine.max_batch:     # checked before the step, which would update the streaks
            raise ValueError('reinit: %d tracks x init keep=%d exceed the engine\'s max_batch=%d'
                             % (n, reinit_keep(self.opts), self.engine.max_batch))
        self.last_reinit = None
        out = self._track_step(prev_poses, current_rgb, current_depth, rgbA, depthA, weight_ids, object_width)
        return self._reinit(out, current_depth, seg, labels, boxes, weight_ids, object_width)

    def reset_reinit(self):
        """Start every track's streak of frames below the fit threshold from 0 (reinit), as at a new sequence."""
        self._streak = None

    def _reinit(self, out, depth, seg, labels, boxes, weight_ids, object_width):
        """Engine.reinit after the step that gave `out` (a CUDA tensor, updated in place, or numpy, uploaded and brought back)
        and last_fit, on the raw frame depth (filled as the step fills it), with the step's meshes, widths and render mode."""
        dev, n = self.engine.device, len(out)
        if self._streak is None or self._streak.numel() != n:
            self._streak = torch.zeros(n, dtype=torch.int32, device=dev)
        on_host = not torch.is_tensor(out)
        poses = torch.from_numpy(np.ascontiguousarray(out)).to(dev) if on_host else out
        rows = self.last_fit if torch.is_tensor(self.last_fit) else torch.from_numpy(np.ascontiguousarray(self.last_fit)).to(dev)
        ow = object_width.to(dev, torch.float64).contiguous() if torch.is_tensor(object_width) else \
            torch.from_numpy(self._widths(object_width, n)).to(dev)
        r = self.renderer
        event = self.engine.reinit(depth, seg, self.K, labels, ow, poses, rows, self._streak, self.opts.tau, self.reinit['below'],
                                   self.reinit['after'], weight_ids=self._weight_ids(weight_ids, n), mode=r.mode, image_hw=r.image_hw,
                                   init=self.reinit['init'], fill_depth=self.fill_depth, boxes=boxes)
        if not on_host:
            self.last_reinit = event
            return out
        self.last_reinit = event.cpu().numpy()
        if not torch.is_tensor(self.last_fit):           # the host route's rows; the device route's were updated in place
            self.last_fit = rows.cpu().numpy()
        return poses.cpu().numpy()

    def _track_step(self, prev_poses, current_rgb, current_depth, rgbA, depthA, weight_ids, object_width):
        """on_track_batch's tracking step, without re-initialisation."""
        render = rgbA is None or depthA is None
        if render and not hasattr(self.renderer, 'render_batch'):
            raise RuntimeError('on_track_batch without rgbA/depthA needs the CUDA renderer (Tracker(renderer="cuda", model_path=*.ply))')
        renderer = self._fused_renderer(weight_ids) if render else None      # None: render input A first, then track
        if renderer is None:
            self._check_step_draws(not render)
        self.last_fit = self.last_icp = self.last_choice = None
        opts, hyp = self.opts, None
        if opts.hypotheses > 1:                       # (c << 32) + j: track j's draw key in this call
            n_tracks = len(prev_poses)
            if n_tracks * opts.hypotheses > self.engine.max_batch:
                raise ValueError('%d tracks x hypotheses=%d exceed the engine\'s max_batch=%d'
                                 % (n_tracks, opts.hypotheses, self.engine.max_batch))
            keys = (np.int64(self._calls) << np.int64(32)) + np.arange(n_tracks, dtype=np.int64)
            hyp = dict(hypotheses=opts.hypotheses, max_translation=self.spread[0], max_rotation_deg=self.spread[1], seed=opts.seed)
        is_np = lambda *xs: all(isinstance(x, np.ndarray) for x in xs)
        if (is_np(current_rgb, current_depth) and (renderer is not None or is_np(rgbA, depthA))
                and not any(torch.is_tensor(x) for x in (prev_poses, weight_ids, object_width))):
            c = lambda a, dt: a if (a.dtype == dt and a.flags['C_CONTIGUOUS']) else np.ascontiguousarray(a).astype(dt, copy=False)
            poses = np.ascontiguousarray(prev_poses, dtype=np.float64).reshape(-1, 4, 4)
            n = len(poses)
            wh = self._weight_ids(weight_ids, n)
            frame, ow = (c(current_rgb, np.uint8), c(current_depth, np.uint16)), self._widths(object_width, n)
            A = () if renderer is not None else (c(rgbA, np.uint8), c(depthA, np.uint16))
            if self._fp8_pending(wh):                 # the inputs go to the device only to calibrate
                with self._uploads(poses, *frame, *(A or (None, None)), ow) as d:
                    self._calibrate_fp8(weight_ids, wh, *d)
            kw = dict(weight_ids=wh, precision=self.precision, fill_depth=self.fill_depth)
            if hyp is not None:
                out, self.last_choice, self.last_fit = self.engine.track_hypotheses_host(
                    *frame, self.K, poses, ow, self.trans_normalizer, self.rot_normalizer, keys, mode=renderer.mode,
                    image_hw=renderer.image_hw, iterations=self.iterations, fit=opts.tau, **hyp, **kw)
                self._calls += 1                      # only a call that ran uses up its c
                return out
            if renderer is not None:
                out = self.engine.track_render_host(*frame, self.K, poses, ow, self.trans_normalizer, self.rot_normalizer,
                                                    mode=renderer.mode, image_hw=renderer.image_hw, iterations=self.iterations,
                                                    fit=opts.tau, icp=opts.icp, **kw)
                if opts.icp is not None:
                    *out, self.last_icp = out
                    out = out[0] if len(out) == 1 else tuple(out)
                if opts.tau:
                    out, self.last_fit = out
                return out
            return self.engine.track_host(*frame, self.K, poses, ow, *A, self.trans_normalizer, self.rot_normalizer, **kw)

        dev = self.engine.device
        n = len(prev_poses)
        wh = self._weight_ids(weight_ids, n)
        if object_width is None:
            ow = self._resident(('ow', n), lambda: self._widths(None, n))
        else:
            ow = object_width if torch.is_tensor(object_width) else self._widths(object_width, n)
        with self._uploads(prev_poses, current_rgb, current_depth, *((None, None) if render else (rgbA, depthA)), ow) as d:
            poses, rgb_d, depth_d, rgbA_d, depthA_d, ow = d
            if self._fp8_pending(wh):
                self._calibrate_fp8(weight_ids, wh, *d)
            wd = None if wh is None else self._resident(('wids', wh.tobytes()), lambda: wh)
            if render and renderer is None:          # a renderer the step cannot stand in for draws input A first
                rgbA_d, depthA_d = self.renderer.render_batch(poses, ow, None if weight_ids is None else wd)
            as_numpy = not torch.is_tensor(prev_poses)
            outs = {}
            if as_numpy:                              # results go back to the host: persistent output buffers keep the graph key stable too
                ob = self._np_bufs.get(('out', n))
                if ob is None:
                    ob = self._np_bufs[('out', n)] = (torch.empty(n, 4, 4, dtype=torch.float64, device=dev),
                                                      torch.empty(n, 3, dtype=torch.float32, device=dev), torch.empty(n, 3, dtype=torch.float32, device=dev))
                outs = dict(out_poses=ob[0], out_trans=ob[1], out_rot=ob[2])
            kw = dict(weight_ids_host=wh, weight_ids_dev=wd, precision=self.precision, fill_depth=self.fill_depth, **outs)
            if hyp is not None:                       # keys, choice and rows in persistent buffers: one graph, frame after frame
                kb = self._np_bufs.get(('hyp', n))
                if kb is None:
                    kb = self._np_bufs[('hyp', n)] = (torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
                                                      torch.empty(n, _lib.FIT_COLS, dtype=torch.int32, device=dev))
                # formed on the device from the call count: no host copy, nothing waits for the previous step
                torch.arange(n, dtype=torch.int64, device=dev, out=kb[0]).add_(self._calls << 32)
                out, self.last_choice, self.last_fit = self.engine.track_hypotheses(
                    rgb_d, depth_d, self.K, poses, ow, self.trans_normalizer, self.rot_normalizer, kb[0], mode=renderer.mode,
                    image_hw=renderer.image_hw, iterations=self.iterations, fit=opts.tau, out_choice=kb[1], out_fit=kb[2], **hyp, **kw)
                self._calls += 1
            elif renderer is not None:                  # input A is drawn inside the step, with the weight ids as mesh ids
                res = self.engine.track_render(rgb_d, depth_d, self.K, poses, ow, self.trans_normalizer, self.rot_normalizer,
                                               mode=renderer.mode, image_hw=renderer.image_hw, iterations=self.iterations,
                                               fit=opts.tau, icp=opts.icp, **kw)
                out = res[0]
                if opts.tau:
                    self.last_fit = res[3]
                if opts.icp is not None:
                    self.last_icp = res[-1]
            else:
                out, _, _ = self.engine.track_batch(rgb_d, depth_d, self.K, poses, ow, rgbA_d, depthA_d,
                                                    self.trans_normalizer, self.rot_normalizer, **kw)
        return out.cpu().numpy() if as_numpy else out

    def _check_step_draws(self, given=False, why=None):
        """A ValueError when iterations > 1, the fit check or ICP need the models drawn inside the tracking step and it cannot
        draw them: why, or input A given (given), or a renderer the step cannot stand in for."""
        if why is None:
            why = 'input A was passed in' if given else 'the renderer cannot draw input A inside the tracking step (_fused_renderer)'
        needs = (['iterations=%d redraws input A at each refined pose' % self.iterations] if self.iterations > 1 else []) + \
                (['fit=%d draws every model at its new pose' % self.opts.tau] if self.opts.tau else []) + \
                (['icp=%r draws every model at its refined pose' % (self.opts.icp,)] if self.opts.icp is not None else [])
        if needs:
            raise ValueError('%s, but %s' % (' and '.join(needs), why))

    def _weight_ids(self, weight_ids, n):
        """The tracks' weight ids as an int32 host array: the Tracker's weight set unless given, None for set 0 (a step
        without ids uses set 0)."""
        if weight_ids is None:
            return np.full(n, self.weight_id, dtype=np.int32) if self.weight_id != 0 else None
        return np.ascontiguousarray(weight_ids.cpu().numpy() if torch.is_tensor(weight_ids) else weight_ids, dtype=np.int32)

    def _fp8_pending(self, wh):
        """'fp8' and some weight set among the tracks' ids (wh as _weight_ids gives them) has no activation scales yet."""
        return self.precision == 'fp8' and any(self.engine.fp8_scales(w) is None for w in set([0] if wh is None else wh.tolist()))

    def _calibrate_fp8(self, weight_ids, wh, poses, rgb, depth, rgbA, depthA, ow):
        """'fp8': the weight sets of this frame's tracks that have no activation scales yet are calibrated on their tracks of
        this frame before the step runs (Engine.calibrate_fp8_tracks), from the device inputs _uploads made: input A as given
        or (rgbA None) drawn by the rasteriser, B cropped at the previous pose from the frame (hole-filled as the step fills
        it).  Sets that have scales are left alone."""
        n = poses.shape[0]
        ids = np.zeros(n, np.int32) if wh is None else wh
        render = None
        if rgbA is None:
            r, dev = self.renderer, self.engine.device
            mesh_ids = (torch.from_numpy(ids).to(dev) if weight_ids is not None
                        else torch.full((n,), r.mesh_id, dtype=torch.int32, device=dev))
            render = dict(mode=r.mode, image_hw=r.image_hw, mesh_ids=mesh_ids)
        self.engine.calibrate_fp8_tracks(rgb, depth, self.K, poses, ow, rgbA, depthA, weight_ids=ids, fill_depth=self.fill_depth,
                                         render=render)

    def _widths(self, object_width, n):
        """The tracks' object widths as a float64 host array: the Tracker's object width unless given."""
        return np.full(n, self.object_width if object_width is None else object_width, dtype=np.float64)

    def _resident(self, key, make):
        """A device copy of the small host array make() returns (weight ids, the default widths), made once per key and kept:
        its stable address keeps the step's CUDA graph, and later calls copy nothing."""
        t = self._np_bufs.get(key)
        if t is None:
            t = self._np_bufs[key] = torch.from_numpy(make()).to(self.engine.device)
        return t

    _UPLOADS = (('poses', torch.float64), ('rgb', torch.uint8), ('depth', torch.uint16), ('rgbA', torch.uint8),
                ('depthA', torch.uint16), ('widths', torch.float64))

    @contextlib.contextmanager
    def _uploads(self, *inputs):
        """The device route's inputs (poses, rgb, depth, rgbA, depthA, widths; None stays None) as device tensors, for the
        with-block to read.  A CUDA tensor is used as it is (converted when its dtype or layout differ).  Any other input -- a
        numpy array (depth coerced to uint16), a pageable or a pinned CPU tensor -- is copied into this call's slot of two
        staging sets, used alternately.  A slot keeps one device buffer per argument, reallocated only when that argument's
        shape changes: the step's CUDA graph is keyed by its device pointers, so stable addresses mean one graph launch per
        frame.  The copies run non_blocking on the copy stream once the kernels that last read the slot are done, so the
        uploads of call k overlap the kernels of call k-1, and the current stream waits for them.  A copy from pageable memory
        has read its source when it returns; a pinned tensor is read asynchronously.  When the block exits, the slot's done
        event is recorded on the current stream after every kernel the block enqueued."""
        dev = self.engine.device
        cur, cs = torch.cuda.current_stream(dev), self._copy_stream
        self._stage_slot ^= 1
        bufs, done = self._stage_bufs[self._stage_slot], self._stage_done[self._stage_slot]
        out, copies = [], []
        for (name, dt), x in zip(self._UPLOADS, inputs):
            if x is None or (torch.is_tensor(x) and x.is_cuda):
                out.append(x if x is None else x.to(dev, dt).contiguous())
                continue
            if not torch.is_tensor(x):
                a = np.ascontiguousarray(x)
                x = torch.from_numpy(a.astype(np.uint16) if dt == torch.uint16 and a.dtype != np.uint16 else a)
            src = x if x.dtype == dt else x.to(dt)
            buf = bufs.get(name)
            if buf is None or buf.shape != src.shape:
                buf = bufs[name] = torch.empty(src.shape, dtype=dt, device=dev)
                cs.wait_stream(cur)                  # a new buffer may reuse memory that kernels queued on cur still use
            copies.append((buf, src))
            out.append(buf)
        if copies:
            cs.wait_event(done)                      # the kernels that last read this slot are done
            with torch.cuda.stream(cs):
                for buf, src in copies:
                    buf.copy_(src, non_blocking=True)
            cur.wait_stream(cs)
        try:
            yield out
        finally:
            if copies:
                done.record(cur)


# ====================================================================================================
# Sequence driver + on-disk formats (SURVEY.md 8f row 3): the reference's predictSequenceYcbInEOAT
# (predict.py:579-623) and __main__ (predict.py:626-672) without the GUI (imshow / waitKey / VideoWriter).
#   <seq>/rgb/*.png, <seq>/depth_filled/*.png (uint16 mm), <seq>/annotated_poses/*.txt (4x4, np.loadtxt)
#   --train_data_path/../dataset_info.yml, --mean_std_path/{mean,std}.npy (train.py:124-125),
#   --ckpt_dir model_best_val.pth.tar = {'epoch', 'state_dict', ...} (problems.py:149-151), --model_path *.ply
#   -> <outdir>/%07d.txt written with np.savetxt (predict.py:611): what eval_ycb.py scores.
# ====================================================================================================
def read_rgb(path):
    """np.array(Image.open(path))[:, :, :3] (predict.py:604)."""
    from PIL import Image
    return np.ascontiguousarray(np.array(Image.open(path))[:, :, :3])


def read_depth(path):
    """cv2.imread(path, IMREAD_UNCHANGED).astype(uint16) (predict.py:606): millimetres."""
    import cv2
    d = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if d is None:
        raise FileNotFoundError(path)
    return d.astype(np.uint16)


def _decode_into(host, name, read, path):
    """A StagingRing job: read(path) (read_rgb or read_depth) into the pinned camera image host[name]."""
    img = read(path)
    dst = host[name]
    if img.shape != tuple(dst.shape):
        raise ValueError('%s: %s, the camera image is %s (dataset_info.yml)' % (path, img.shape, tuple(dst.shape)))
    dst.numpy()[...] = img


# The result videos' frame label: cv2.putText(img, text, (W//2, H-50), FONT_HERSHEY_SIMPLEX, fontScale=1, thickness=4)
# (predict.py:428, 556, 618).  "frame:0" ... "frame:9999999" set pixels in rows H-73 ... H-48 only, so the label is kept as the
# full-width strip of rows [H - LABEL_TOP, H - LABEL_BOTTOM).
LABEL_TOP, LABEL_BOTTOM = 80, 40


def label_strip(text, H, W, out=None):
    """(y0, mask): the pixels of the result videos' label `text` on an H x W frame, as a uint8 (LABEL_TOP - LABEL_BOTTOM, W) mask
    (255 where cv2.putText sets a pixel, 0 elsewhere; LINE_8 draws no anti-aliased edge) of the rows from y0 = H - LABEL_TOP.
    Written into `out` when given.  Engine.draw_tracks takes it as its label."""
    import cv2
    if H < LABEL_TOP:
        raise ValueError('a labelled video frame needs at least %d rows, not %d' % (LABEL_TOP, H))
    y0 = H - LABEL_TOP
    mask = np.zeros((LABEL_TOP - LABEL_BOTTOM, W), dtype=np.uint8) if out is None else out
    mask[...] = 0
    cv2.putText(mask, text, (W // 2, H - 50 - y0), cv2.FONT_HERSHEY_SIMPLEX, fontScale=1, thickness=4, color=255)
    return y0, mask


def _label_into(host, text, H, W):
    """A StagingRing job: the label strip of `text` into the pinned host['label']."""
    label_strip(text, H, W, host['label'].numpy())


def sequence_files(test_data_path):
    """(rgb files, depth files, ground-truth pose files), each sorted (predict.py:584-590)."""
    import glob
    rgb = sorted(glob.glob('{}/rgb/*.png'.format(test_data_path)))
    depth = sorted(glob.glob('{}/depth_filled/*.png'.format(test_data_path)))
    gt = sorted(glob.glob('{}/annotated_poses/*.txt'.format(test_data_path)))
    if not rgb or len(rgb) != len(depth):
        raise FileNotFoundError('need the same number of rgb/*.png and depth_filled/*.png under ' + str(test_data_path))
    if not gt:
        raise FileNotFoundError('need annotated_poses/*.txt (frame 0 initialises the track) under ' + str(test_data_path))
    return rgb, depth, gt


def load_run_config(train_data_path, mean_std_path):
    """dataset_info.yml next to the training data and the channel statistics (predict.py:657-664)."""
    import yaml
    with open(os.path.join(train_data_path, '../dataset_info.yml'), 'r') as ff:
        dataset_info = yaml.safe_load(ff)
    images_mean = np.load(os.path.join(mean_std_path, 'mean.npy'))
    images_std = np.load(os.path.join(mean_std_path, 'std.npy'))
    return dataset_info, images_mean, images_std


def predictSequenceYcbInEOAT(test_data_path, dataset_info, images_mean, images_std, ckpt_dir, model_path, outdir,
                             tracker=None, max_frames=None, **tracker_kwargs):
    """Track one object through a recorded sequence, starting from the first annotated pose, one pose file per frame.
    The reference's normalisers for this data set are 0.03 m / 30 degrees (predict.py:587).  Returns the (N,4,4) poses."""
    rgb_files, depth_files, gt_files = sequence_files(test_data_path)
    if tracker is None:
        tracker = Tracker(dataset_info, images_mean, images_std, ckpt_dir, model_path=model_path, trans_normalizer=0.03,
                          rot_normalizer=30 * np.pi / 180, **tracker_kwargs)
    prev_pose = np.loadtxt(gt_files[0]).copy()
    os.makedirs(outdir, exist_ok=True)
    n = len(rgb_files) if max_frames is None else min(max_frames, len(rgb_files))
    poses = []
    for i in range(n):
        rgb = read_rgb(rgb_files[i])
        depth = read_depth(depth_files[i])
        cur_pose = tracker.on_track(prev_pose.copy(), rgb, depth, gt_A_in_cam=np.eye(4), gt_B_in_cam=np.eye(4), debug=False, samples=1)
        prev_pose = cur_pose.copy()
        np.savetxt(os.path.join(outdir, '%07d.txt' % i), cur_pose)
        poses.append(cur_pose)
    return np.stack(poses)


# ----------------------------------------------------------------------------------------------------
# YCB-Video drivers (reference predict.py:299-575): predictSequenceYcb (one sequence, optional PoseCNN / PoseRBPF
# initialisation and re-initialisation frames, per-sequence ADD-S AUC) and getResultsYcb (every test sequence 0048-0059
# that contains the class; what eval_ycb.py scores).  Headless: no VideoWriter / imshow.  The data-set layout is the
# reference's:  <ycb_dir>/<seq %04d>/{color,depth_filled,seg,pose_gt/<class_id>}/..., <ycb_dir>/image_sets/keyframe.txt,
# <ycb_dir>/YCB_Video_toolbox/results_PoseCNN_RSS2018/%06d.mat (rois, poses_icp), .../PoseRBPF_Results/YCB_results_RGBD/.
# ----------------------------------------------------------------------------------------------------
def quaternion_matrix3(q_wxyz):
    """3x3 rotation of a (w, x, y, z) quaternion -- transformations.quaternion_matrix(q)[:3,:3] (reference predict.py:117)."""
    q = np.array(q_wxyz, dtype=np.float64, copy=True)
    n = np.dot(q, q)
    if n < np.finfo(float).eps * 4.0:
        return np.identity(3)
    q *= np.sqrt(2.0 / n)
    q = np.outer(q, q)
    return np.array([[1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0]],
                     [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0]],
                     [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2]]])


def read_keyframes(ycb_dir):
    with open('{}/image_sets/keyframe.txt'.format(ycb_dir), 'r') as ff:
        return [l.rstrip() for l in ff.readlines()]


def nearest_keyframe(seq_frames, seq_id, start_frame):
    """The keyframe of `seq_id` closest to `start_frame`, searching outwards (reference predict.py:93-107, 485-496)."""
    neighbor = 0
    while neighbor < 100000:
        for cand in (start_frame + neighbor, start_frame - neighbor):
            tmp = '%04d/%06d' % (seq_id, cand)
            if tmp in seq_frames:
                return tmp, seq_frames.index(tmp), cand
        neighbor += 1
    raise ValueError('sequence %04d has no keyframe' % seq_id)


def posecnn_pose(mat_path, class_id):
    """Pose of `class_id` from a PoseCNN result file: rois[:,1] == class id, poses_icp = (qw,qx,qy,qz,x,y,z) (predict.py:111-122)."""
    import scipy.io
    res = scipy.io.loadmat(mat_path)
    idx = np.where(res['rois'][:, 1] == class_id)
    tmp = res['poses_icp'][idx].reshape(-1)
    if tmp.size < 7:
        raise ValueError('class %d not in %s' % (class_id, mat_path))
    pose = np.eye(4)
    pose[:3, :3] = quaternion_matrix3(tmp[:4])
    pose[:3, 3] = tmp[4:7]
    return pose


def use_posecnn_res(class_id, seq_frame_str, ycb_dir, posecnn_dir=None):
    """PoseCNN's estimate at the keyframe nearest to `seq_frame_str` = '%04d/%06d' (reference predict.py:89-123)."""
    seq_frames = read_keyframes(ycb_dir)
    seq_id, start_frame = int(seq_frame_str.split('/')[0]), int(seq_frame_str.split('/')[1])
    _, index, _ = nearest_keyframe(seq_frames, seq_id, start_frame)
    posecnn_dir = posecnn_dir or '{}/YCB_Video_toolbox/results_PoseCNN_RSS2018/'.format(ycb_dir)
    return posecnn_pose(os.path.join(posecnn_dir, '%06d.mat' % index), class_id)


def poserbpf_pose(ycb_dir, class_id, seq_id, seqs):
    """First pose of PoseRBPF's result file for (class, sequence) (reference predict.py:376-390, 498-513): 'x y z qw qx qy qz' after two tokens."""
    import glob
    res_dir = '{}/YCB_Video_toolbox/PoseRBPF_Results/YCB_results_RGBD/'.format(ycb_dir)
    folders = sorted(os.listdir(res_dir))
    cur = res_dir + folders[class_id - 1] + '/' + 'seq_{}/'.format(seqs.index(seq_id) + 1)
    with open(glob.glob(cur + 'Pose*.txt')[0], 'r') as ff:
        pose = ff.readlines()[0].rstrip().split()[2:]
    out = np.eye(4)
    out[:3, 3] = np.array(pose[:3], dtype=np.float64)
    out[:3, :3] = quaternion_matrix3(np.array(pose[3:7], dtype=np.float64))
    return out


def findClassContainedVideosYcb(class_id, data_dir, testset=True):
    """Sequence ids under `data_dir` whose pose_gt/ has a folder for `class_id` (reference Utils.py:108-123; test set = 0048..0059)."""
    import glob, re
    out = []
    for gt_dir in sorted(glob.glob(os.path.join(data_dir, '**/pose_gt'))):
        video_index = int(re.findall(r'/[0-9]{4}/', gt_dir + '/')[0][1:-1])
        if testset and (video_index < 48 or video_index > 59):
            continue
        if class_id in list(map(int, os.listdir(gt_dir))):
            out.append(video_index)
    return out


def _ycb_sequence_files(seq_dir, class_id):
    import glob
    rgb = sorted(glob.glob(os.path.join(seq_dir, 'color/*')))
    depth = sorted(glob.glob(os.path.join(seq_dir, 'depth_filled/*')))
    gt = sorted(glob.glob(os.path.join(seq_dir, 'pose_gt/{}/*'.format(class_id))))
    if not rgb or len(rgb) != len(depth) or len(gt) < len(rgb):
        raise FileNotFoundError('need matching color/, depth_filled/ and pose_gt/%d/ files under %s' % (class_id, seq_dir))
    return rgb, depth, gt


def predictSequenceYcb(ycb_dir, seq_id, class_id, dataset_info, images_mean, images_std, ckpt_dir, model_path, outdir,
                       init='gt', reinit_frames=None, start_frame=0, tracker=None, max_frames=None, **tracker_kwargs):
    """Track `class_id` through YCB-Video sequence `seq_id` (reference predict.py:446-575).  init: 'gt' | 'posecnn' | 'poserbpf'.
    reinit_frames: '%04d/%06d' strings (1-based frame ids, as the reference compares them): the track restarts there from
    PoseCNN's estimate.  Writes <outdir>/%05d.txt and %05dgt.txt and returns (poses (N,4,4), ADD-S AUC in percent)."""
    test_data_path = '{}/%04d'.format(ycb_dir) % seq_id
    rgb_files, depth_files, gt_files = _ycb_sequence_files(test_data_path, class_id)
    gt_poses = [np.loadtxt(f) for f in gt_files]
    reinit_frames = list(reinit_frames or [])
    if tracker is None:
        tracker = Tracker(dataset_info, images_mean, images_std, ckpt_dir, model_path=model_path, **tracker_kwargs)
    if init == 'gt':
        prev_pose = gt_poses[start_frame].copy()
    elif init == 'posecnn':
        seq_frame_str, _, start_frame = nearest_keyframe(read_keyframes(ycb_dir), seq_id, start_frame)
        prev_pose = use_posecnn_res(class_id, seq_frame_str, ycb_dir)
    elif init == 'poserbpf':
        seqs = sorted(findClassContainedVideosYcb(class_id, ycb_dir, testset=True))
        prev_pose = poserbpf_pose(ycb_dir, class_id, seq_id, seqs)
    else:
        raise ValueError('init must be gt, posecnn or poserbpf')
    pred_poses = [prev_pose]
    os.makedirs(outdir, exist_ok=True)
    n = len(rgb_files) if max_frames is None else min(len(rgb_files), start_frame + 1 + max_frames)
    for i in range(start_frame + 1, n):
        rgb = read_rgb(rgb_files[i])
        depth = read_depth(depth_files[i])
        A_in_cam = prev_pose.copy()
        if '%04d/%06d' % (seq_id, i + 1) in reinit_frames:
            A_in_cam = use_posecnn_res(class_id, '%04d/%06d' % (seq_id, i - 1), ycb_dir)
        cur_pose = tracker.on_track(A_in_cam, rgb, depth, gt_A_in_cam=gt_poses[i - 1], gt_B_in_cam=gt_poses[i], debug=False, samples=1)
        prev_pose = cur_pose.copy()
        pred_poses.append(cur_pose)
    pred_poses = np.array(pred_poses)
    for i in range(len(pred_poses)):
        np.savetxt(os.path.join(outdir, '%05d.txt' % i), pred_poses[i])
        np.savetxt(os.path.join(outdir, '%05dgt.txt' % i), gt_poses[start_frame + i])
    adi_auc = None
    if tracker.object_cloud is not None:                           # per-sequence ADD-S AUC (predict.py:566-575) on the device (csrc/metrics.cu)
        eng = tracker.engine
        pts = torch.from_numpy(np.ascontiguousarray(tracker.object_cloud.points)).to(eng.device)
        gts = torch.from_numpy(np.stack(gt_poses[start_frame:start_frame + len(pred_poses)])).to(eng.device)
        _, adi = eng.add_adi(pts, torch.from_numpy(pred_poses).to(eng.device), gts, want_add=False)
        adi_auc = eng.vocap(adi) * 100
    return pred_poses, adi_auc


def _ycb_first_pose(ycb_dir, class_id, seq_id, gt_file0, initialize_method, keyframes_all, seqs):
    """The pose a track of `class_id` starts sequence `seq_id` from (reference predict.py:376-390): the ground truth of its first
    frame, PoseCNN's estimate at the sequence's first key frame, or PoseRBPF's first pose.  seqs: the class's test sequences."""
    if initialize_method == 'posecnn':
        seq_frame = '%04d/%06d' % (seq_id, 1)
        return posecnn_pose('{}/YCB_Video_toolbox/results_PoseCNN_RSS2018/%06d.mat'.format(ycb_dir) % keyframes_all.index(seq_frame), class_id)
    if initialize_method == 'poserbpf':
        return poserbpf_pose(ycb_dir, class_id, seq_id, seqs)
    if initialize_method == 'gt':
        return np.loadtxt(gt_file0)
    raise ValueError('initialize_method must be gt, posecnn or poserbpf')


def getResultsYcb(ycb_dir, class_id, dataset_info, images_mean, images_std, ckpt_dir, model_path, outdir,
                  initialize_method='gt', tracker=None, max_frames=None, **tracker_kwargs):
    """Every YCB-Video TEST sequence (0048..0059) under <ycb_dir>/data_organized/ that contains `class_id`, tracked from its first
    frame; one <outdir>/seq<id>/%07d.txt per frame -- the files eval_ycb.py globs (reference predict.py:299-443).  Returns {seq_id: poses}."""
    import glob, re
    test_data_dir = '{}/data_organized/'.format(ycb_dir)
    os.makedirs(outdir, exist_ok=True)
    if tracker is None:
        tracker = Tracker(dataset_info, images_mean, images_std, ckpt_dir, model_path=model_path, **tracker_kwargs)
    keyframes_all = read_keyframes(ycb_dir) if initialize_method == 'posecnn' else []
    seqs = sorted(findClassContainedVideosYcb(class_id, test_data_dir, testset=True))
    results = {}
    for gt_dir in sorted(glob.glob(test_data_dir + '**/pose_gt')):
        seq_id = int(re.findall(r'/\d{4}/', gt_dir + '/')[0][1:-1])
        if seq_id not in seqs:
            continue
        seq_dir = os.path.join(gt_dir, '..')
        rgb_files, depth_files, gt_files = _ycb_sequence_files(seq_dir, class_id)
        prev_pose = _ycb_first_pose(ycb_dir, class_id, seq_id, gt_files[0], initialize_method, keyframes_all, seqs)
        pred_poses = [prev_pose]
        n = len(rgb_files) if max_frames is None else min(len(rgb_files), 1 + max_frames)
        for i in range(1, n):
            rgb = read_rgb(rgb_files[i])
            depth = read_depth(depth_files[i])
            cur_pose = tracker.on_track(prev_pose, rgb, depth, gt_A_in_cam=None, gt_B_in_cam=np.loadtxt(gt_files[i]), debug=False, samples=1)
            prev_pose = cur_pose.copy()
            pred_poses.append(cur_pose)
        while len(pred_poses) < len(rgb_files) and max_frames is None:      # predict.py:437-440
            pred_poses.append(pred_poses[-1])
        sdir = os.path.join(outdir, 'seq{}'.format(seq_id))
        os.makedirs(sdir, exist_ok=True)
        for i in range(len(pred_poses)):
            np.savetxt(os.path.join(sdir, '%07d.txt' % i), pred_poses[i])
        results[seq_id] = np.array(pred_poses)
    return results


# ----------------------------------------------------------------------------------------------------
# Every class in one pass: the YCB-Video evaluation (the paper's Table I) as one run instead of one getResultsYcb run per class.
# Each test sequence's requested classes are tracked together, one se3tn_track_render step per frame with one weight set and
# mesh per class; each frame is decoded once.  The output tree is what eval_ycb.eval_all scores:
#   <outdir>/<CADmodels folder of the class>/run/seq<id>/%07d.txt
# Per-class configuration is four path templates with {class_id} and {class_name} (the CADmodels/ folder name) placeholders.
# ----------------------------------------------------------------------------------------------------
YCB_ALL_TEMPLATES = ('train_data_path', 'mean_std_path', 'ckpt_dir', 'model_path')
YCB_ALL_RUN = 'run'


def ycb_class_names(ycb_dir):
    """The CADmodels/ folder names in sorted order: class id k is entry k - 1, as eval_ycb.py maps them."""
    d = os.path.join(ycb_dir, 'CADmodels')
    if not os.path.isdir(d):
        raise FileNotFoundError('no CADmodels/ folder under %s: it names the classes' % ycb_dir)
    return sorted(os.listdir(d))


def ycb_classes(ycb_dir, class_ids):
    """[(class id, CADmodels/ folder name)] of class_ids, ascending and without repeats.  An id outside [1, the number of
    CADmodels/ folders] is a ValueError."""
    names = ycb_class_names(ycb_dir)
    out = []
    for c in sorted(set(int(c) for c in class_ids)):
        if not 1 <= c <= len(names):
            raise ValueError('class %d: CADmodels/ under %s has %d classes' % (c, ycb_dir, len(names)))
        out.append((c, names[c - 1]))
    return out


def ycb_all_res_dir(outdir, class_name):
    """Where getResultsYcbAll writes a class's seq<id>/%07d.txt files: eval_ycb.eval_all takes the class folders in sorted order
    as class ids 1, 2, ..., and the first folder inside each as its result folder."""
    return os.path.join(outdir, class_name, YCB_ALL_RUN)


def _expand_templates(config, config_name, **placeholders):
    """The four YCB_ALL_TEMPLATES path templates of config with the given placeholders filled in."""
    out = {}
    for key in YCB_ALL_TEMPLATES:
        if key not in config:
            raise ValueError('%s needs a %r template' % (config_name, key))
        try:
            out[key] = str(config[key]).format(**placeholders)
        except (KeyError, IndexError, ValueError) as e:
            raise ValueError('%s[%r] = %r: the only placeholders are %s (%s)' % (config_name, key, config[key],
                             ' and '.join('{%s}' % p for p in placeholders), e)) from None
    return out


def expand_class_paths(class_config, class_id, class_name):
    """The four path templates of class_config for one class -> {train_data_path, mean_std_path, ckpt_dir, model_path}."""
    return _expand_templates(class_config, 'class_config', class_id=class_id, class_name=class_name)


def _load_run_files(label, paths):
    """dataset_info.yml, mean and std of expanded paths, after checking that every file the run reads exists: a missing one is a
    FileNotFoundError naming `label` and the path.  -> dict of dataset_info, mean, std and the paths."""
    import yaml
    info_path = os.path.join(paths['train_data_path'], '../dataset_info.yml')
    files = [('dataset_info.yml', info_path), ('mean', os.path.join(paths['mean_std_path'], 'mean.npy')),
             ('std', os.path.join(paths['mean_std_path'], 'std.npy')), ('checkpoint', paths['ckpt_dir']), ('mesh', paths['model_path'])]
    for what, path in files:
        if not os.path.isfile(path):
            raise FileNotFoundError('%s: no %s file at %s' % (label, what, path))
    with open(info_path, 'r') as ff:
        info = yaml.safe_load(ff)
    return dict(dataset_info=info, mean=np.load(files[1][1]), std=np.load(files[2][1]), **paths)


def _check_shared(entries, label, short, shared, why):
    """Every entry at the resolution libse3tn is built for, and equal to the first in each (name, getter) of `shared`; otherwise a
    ValueError naming the entry (label(entry)) and the first (short(entry))."""
    first = entries[0]
    for k in entries:
        if k['dataset_info']['resolution'] != 176:
            raise ValueError('%s: resolution %s; libse3tn is built for 176' % (label(k), k['dataset_info']['resolution']))
        for what, get in shared:
            if get(k) != get(first):
                raise ValueError('%s: %s %r differs from %s\'s %r; %s' % (label(k), what, get(k), short(first), get(first), why))


def _camera(k):
    return {key: float(v) for key, v in k['dataset_info']['camera'].items()}


def _pyrender(k):
    return k['dataset_info'].get('renderer') == 'pyrenderer'


def _class_normalizer(class_config, key, class_id, default):
    v = class_config.get(key, default)
    if isinstance(v, dict) and class_id not in v:
        raise ValueError('class_config[%r] has no value for class %d' % (key, class_id))
    return float(v[class_id] if isinstance(v, dict) else v)


# The modes the one-pass YCB-Video driver offers: every mode but 'fp16', which its callers have treated as an unknown name
# since before the mode existed.  The YCBInEOAT driver, the Tracker and the Engine take every mode of engine.PREC.
YCB_ALL_PRECISIONS = ('bf16x3', 'tf32', 'bf16', 'fp8', 'fp32')
# Every mode of engine.PREC, in the order a sweep of the YCBInEOAT driver lists them.
PRECISIONS = ('bf16x3', 'tf32', 'bf16', 'fp16', 'fp8', 'fp32')


def precision_modes(precision, modes):
    """The modes a one-pass driver tracks in -> (modes tuple, sweep).  A single mode name gives ((name,), False) and is checked
    where it always was; 'all' gives (modes, True); a sequence of names gives (those names, True).  In a sweep, a name not in
    `modes`, a name listed twice and an empty sequence are a ValueError."""
    if isinstance(precision, str) and precision != 'all':
        return (precision,), False
    got = tuple(modes) if isinstance(precision, str) else tuple(precision)
    if not got:
        raise ValueError('no precision mode given')
    for m in got:
        if m not in modes:
            raise ValueError('precision %r is not a mode of this driver (one of %s)' % (m, ', '.join(modes)))
    twice = sorted(set(m for m in got if got.count(m) > 1))
    if twice:
        raise ValueError('precision %s listed more than once' % ', '.join(twice))
    return got, True


def sweep_reference(modes):
    """The mode a sweep's drift is measured from: 'fp32' if swept, else 'bf16x3' if swept, else the first mode listed."""
    return 'fp32' if 'fp32' in modes else 'bf16x3' if 'bf16x3' in modes else modes[0]


def precision_outdir(outdir, mode):
    """Where a sweep writes mode `mode`'s output tree: <outdir>/<mode>/, what a single-mode run with that outdir writes."""
    return os.path.join(outdir, mode)


def refine_counts(iterations):
    """The refinement counts a one-pass driver tracks with -> (counts tuple, sweep).  An integer k gives ((k,), False); a sequence
    of them gives (those counts, True).  A count outside [1, 8] (Engine.refine_iterations), a count listed twice and an empty
    sequence are a ValueError."""
    if isinstance(iterations, (list, tuple)):
        got = tuple(_refine_iterations(k) for k in iterations)
        if not got:
            raise ValueError('no iteration count given')
        twice = sorted(set(k for k in got if got.count(k) > 1))
        if twice:
            raise ValueError('iterations %s listed more than once' % ', '.join(map(str, twice)))
        return got, True
    return (_refine_iterations(iterations),), False


def iterations_outdir(outdir, k):
    """Where a sweep of refinement counts writes count k's output tree: <outdir>/iter<k>/, what a run with that k and that outdir
    writes (with <mode>/ below it when precision modes are swept too)."""
    return os.path.join(outdir, 'iter%d' % k)


def checkpoint_outdir(outdir, i):
    """Where a run over several checkpoints writes checkpoint i's output tree: <outdir>/ckpt<i>/, what a run of checkpoint i
    alone with that outdir writes (with iter<k>/ and <mode>/ below it when those are swept too)."""
    return os.path.join(outdir, 'ckpt%d' % i)


# Several checkpoints in one run: checkpoint i's weight set of the class or object of weight id w is w + CKPT_ID_STRIDE * i.  The
# context takes any id >= 0 (its per-id tables grow to the largest); the stride keeps the checkpoints' ids apart, so a run over
# several checkpoints takes base ids below it.
CKPT_ID_STRIDE = 32


def checkpoint_list(ckpts, mean_std_paths, ckpt_name='ckpt_dir', stats_name='mean_std_path'):
    """The checkpoints of a run -> [(checkpoint, mean_std_path)]: ckpts one path (or template) or a list of them, mean_std_paths
    one folder shared by all or one per checkpoint (train.py writes mean / std per training run).  An empty list or entry, a
    checkpoint listed twice and any other number of mean_std_paths are a ValueError naming the argument."""
    ckpts = [ckpts] if isinstance(ckpts, str) else list(ckpts)
    stats = [mean_std_paths] if isinstance(mean_std_paths, str) else list(mean_std_paths)
    if not ckpts or not all(ckpts):
        raise ValueError('%s: an empty checkpoint entry' % ckpt_name)
    if not stats or not all(stats):
        raise ValueError('%s: an empty entry' % stats_name)
    twice = sorted(set(c for c in ckpts if ckpts.count(c) > 1))
    if twice:
        raise ValueError('%s: checkpoint %s listed more than once' % (ckpt_name, ', '.join(twice)))
    if len(stats) not in (1, len(ckpts)):
        raise ValueError('%s: %d entries for %d checkpoints; give one, shared by all, or one per checkpoint'
                         % (stats_name, len(stats), len(ckpts)))
    return list(zip(ckpts, stats * len(ckpts) if len(stats) == 1 else stats))


def checkpoint_configs(config):
    """A one-pass driver's path templates with ckpt_dir (and mean_std_path) as lists -> one config per checkpoint, each with a
    single ckpt_dir and mean_std_path (checkpoint_list's rules).  Plain strings give [config] unchanged."""
    if 'ckpt_dir' not in config or 'mean_std_path' not in config:
        return [config]
    if isinstance(config['ckpt_dir'], str) and isinstance(config['mean_std_path'], str):
        return [config]
    return [dict(config, ckpt_dir=c, mean_std_path=m) for c, m in checkpoint_list(config['ckpt_dir'], config['mean_std_path'])]


def _check_checkpoint_ids(base_ids, ckpts, what):
    """With several checkpoints, every base weight id below CKPT_ID_STRIDE: otherwise a ValueError naming it."""
    for w in base_ids:
        if ckpts > 1 and not 0 <= w < CKPT_ID_STRIDE:
            raise ValueError('%s %d: with %d checkpoints the weight ids are %s id + %d x checkpoint index, so the %s ids stop at %d'
                             % (what, w, ckpts, what, CKPT_ID_STRIDE, what, CKPT_ID_STRIDE - 1))


def _sweep_variants(outdir, modes, sweep, counts, ksweep, ckpts=1):
    """The variants a one-pass driver tracks every frame in -> [(mode, k, output tree)] with one checkpoint, [(mode, k,
    checkpoint index, output tree)] with several: each entry is a variant's key followed by its tree.  With one checkpoint the
    tree has no ckpt<i>/ level."""
    out = []
    for c in range(ckpts):
        root = checkpoint_outdir(outdir, c) if ckpts > 1 else outdir
        for k in counts:
            base = iterations_outdir(root, k) if ksweep else root
            for m in modes:
                out.append((m, k) + ((c,) if ckpts > 1 else ()) + (precision_outdir(base, m) if sweep else base,))
    return out


def _variant_checkpoint(key):
    """The checkpoint index of a variant key: (mode, k) is checkpoint 0 of a one-checkpoint run, (mode, k, i) checkpoint i."""
    return key[2] if len(key) > 2 else 0


def _sweep_results(results, variants, sweep, ksweep):
    """A driver's return value from {variant key: what one variant's run returns}: per checkpoint, that alone for one variant,
    {mode: ...} for a precision sweep, {k: ...} for a sweep of counts, {k: {mode: ...}} for both; {checkpoint index: that}
    with more than one checkpoint."""
    per_c = {}
    for v in variants:
        m, k = v[:2]
        per_c.setdefault(_variant_checkpoint(v[:-1]), {}).setdefault(k, {})[m] = results[v[:-1]]
    for c, per_k in per_c.items():
        per_k = {k: (v if sweep else next(iter(v.values()))) for k, v in per_k.items()}
        per_c[c] = per_k if ksweep else next(iter(per_k.values()))
    return per_c if len(per_c) > 1 else per_c[0]


def ycb_all_classes(ycb_dir, class_ids, class_config, precision='bf16x3'):
    """The checked configuration of every requested class, before anything is loaded onto a device -> list (ascending class id)
    of dicts: class_id, name, the expanded paths, dataset_info, mean, std, trans_normalizer, rot_normalizer.

    class_config: the YCB_ALL_TEMPLATES path templates; optionally trans_normalizer / rot_normalizer (the Tracker's, default
    0.03 m and 5 degrees as getResultsYcb uses them), each a number or a {class_id: number} mapping.  A missing file is a
    FileNotFoundError naming the class and the path.  One step tracks every class of a frame, so the classes must share the
    camera (K and image size), the resolution (176), the render mode, the two normalisers and the precision: a class that differs
    from the first is a ValueError naming it."""
    if precision not in YCB_ALL_PRECISIONS:
        raise ValueError('precision %r is not a mode of the one-pass YCB-Video driver (one of %s)' % (precision, ', '.join(YCB_ALL_PRECISIONS)))
    ids = ycb_classes(ycb_dir, class_ids)
    if not ids:
        raise ValueError('no class ids given')
    classes = []
    for c, name in ids:
        k = _load_run_files('class %d (%s)' % (c, name), expand_class_paths(class_config, c, name))
        classes.append(dict(k, class_id=c, name=name,
                            trans_normalizer=_class_normalizer(class_config, 'trans_normalizer', c, 0.03),
                            rot_normalizer=_class_normalizer(class_config, 'rot_normalizer', c, 5 * np.pi / 180)))
    _check_shared(classes, lambda k: 'class %d (%s)' % (k['class_id'], k['name']), lambda k: 'class %d' % k['class_id'],
                  (('camera', _camera), ('renderer', _pyrender),
                   ('trans_normalizer', lambda k: k['trans_normalizer']), ('rot_normalizer', lambda k: k['rot_normalizer'])),
                  'classes tracked in one step must share it')
    return classes


def ycb_track_sets(ycb_dir, class_ids):
    """{seq_id: [class ids]}, ascending: for every YCB-Video test sequence (0048..0059) under <ycb_dir>/data_organized/, the
    requested classes its pose_gt/ lists -- the sequences a getResultsYcb run of each class visits."""
    data_dir = '{}/data_organized/'.format(ycb_dir)
    sets = {}
    for c in sorted(set(int(c) for c in class_ids)):
        for s in findClassContainedVideosYcb(c, data_dir, testset=True):
            sets.setdefault(s, []).append(c)
    return dict(sorted(sets.items()))


def _one_pass_trackers(entries, precision, max_batch):
    """One Engine of max_batch tracks per step on the current device and {weight id: Tracker} on it for
    [(weight id, label, checked configuration)]: the configuration's files and normalisers, the CUDA renderer.  A ValueError is
    relabelled with the class or object it is about."""
    eng = Engine(max_batch=max_batch)
    trackers = {}
    for wid, label, k in entries:
        try:
            trackers[wid] = Tracker(k['dataset_info'], k['mean'], k['std'], k['ckpt_dir'], model_path=k['model_path'], engine=eng,
                                    weight_id=wid, precision=precision, renderer='cuda',
                                    trans_normalizer=k['trans_normalizer'], rot_normalizer=k['rot_normalizer'])
        except ValueError as e:
            raise ValueError('%s: %s' % (label, e)) from e
    return eng, trackers


# Multi-hypothesis steps in the drivers (Tracker(hypotheses=S) per step): track j of a step draws its starts with a 64-bit key
# that names where it is in the run, so a run keys its draws the same on one GPU or several.
def hypothesis_key(a, b, c):
    """The draw key (a << 40) + (b << 16) + c: (sequence index in the run's sorted list, frame index, track index) in the one-pass
    drivers, (key-frame index, row, 0) in ycbv_recover.  a < 2^23, b < 2^24, c < 2^16."""
    if not (0 <= a < 1 << 23 and 0 <= b < 1 << 24 and 0 <= c < 1 << 16):
        raise ValueError('hypothesis key (%d, %d, %d) out of range' % (a, b, c))
    return (a << 40) + (b << 16) + c


def hypothesis_groups(trackers, wh, opts):
    """The tracks of one step grouped by the spread of their class (hypothesis_spread): [(None or an int64 numpy index array,
    spread)].  One group of all tracks (None) when every class shares one spread; otherwise the step runs once per spread on its
    tracks."""
    spreads = [hypothesis_spread(trackers[int(w)].dataset_info, opts) for w in wh]
    if len(set(spreads)) == 1:
        return [(None, spreads[0])]
    return [(np.asarray([j for j, sp in enumerate(spreads) if sp == g], dtype=np.int64), g) for g in sorted(set(spreads))]


def track_step(eng, trackers, trk, rgb, depth, poses, widths, wh, wd, keys, opts, precision, iterations, outs):
    """One driver step of a variant for n tracks over the device frame (rgb, depth), with trk's camera, normalisers and render
    mode.  Without hypotheses, one Engine.track_render with opts' fit check and ICP.  With S > 1, Engine.track_hypotheses with
    the draw keys `keys` (int64 (n)), once per spread group (hypothesis_groups), the rows of each group landing at their tracks.
    outs: out_poses (n,4,4), out_trans / out_rot (n,3), and as the step has them out_fit (n,6), out_choice (n), out_rounds
    (k,n,4,4) / (k,n,S,4,4), out_hyp_poses (n,S,4,4), out_icp_poses (M,n,4,4).  poses may be out_poses."""
    kw = dict(fit=opts.tau, precision=precision, iterations=iterations, mode=trk.renderer.mode, image_hw=trk.renderer.image_hw)
    if opts.hypotheses == 1:
        eng.track_render(rgb, depth, trk.K, poses, widths, trk.trans_normalizer, trk.rot_normalizer, weight_ids_host=wh,
                         weight_ids_dev=wd, icp=opts.icp, **kw, **outs)
        return
    for idx, (mt, mr) in hypothesis_groups(trackers, wh, opts):
        hyp = dict(kw, max_translation=mt, max_rotation_deg=mr, seed=opts.seed)
        if idx is None:
            eng.track_hypotheses(rgb, depth, trk.K, poses, widths, trk.trans_normalizer, trk.rot_normalizer, keys, opts.hypotheses,
                                 weight_ids_host=wh, weight_ids_dev=wd, **hyp, **outs)
            continue
        di = torch.from_numpy(idx).to(eng.device)
        sub = {k: (v.index_select(1, di) if k == 'out_rounds' else v.index_select(0, di)).contiguous() for k, v in outs.items()}
        eng.track_hypotheses(rgb, depth, trk.K, poses.index_select(0, di).contiguous(), widths.index_select(0, di).contiguous(),
                             trk.trans_normalizer, trk.rot_normalizer, keys.index_select(0, di).contiguous(), opts.hypotheses,
                             weight_ids_host=wh[idx], weight_ids_dev=wd.index_select(0, di).contiguous(), **hyp, **sub)
        for k, v in sub.items():
            outs[k].index_copy_(1 if k == 'out_rounds' else 0, di, v)


def _track_sequences(eng, trackers, sequences, variants, depth, workers, video, opts, seq_index):
    """The one-pass drivers' tracking loop.  sequences: [(rgb files, depth files, weight ids (tuple), initial poses (n,4,4))], the
    files those of the frames to track; trackers: {weight id: Tracker} on eng, sharing camera, normalisers and render mode;
    variants: what every frame is tracked in (a tuple) as _sweep_variants keys them, (mode, k) or (mode, k, c): precision mode, k
    refinement rounds per step (Engine.track_render's iterations) and the weight sets of checkpoint c (ids + CKPT_ID_STRIDE * c).
    Yields each sequence's ({variant: (frames, n, 4, 4) numpy poses}, the poses after each frame, and its fit rows or None) as
    soon as the sequence ends.

    Every frame is one se3tn_track_render step per variant (track_step) for the sequence's n tracks, all reading the same device
    frame: the frames of all sequences decode ahead, across sequence boundaries, through one StagingRing of `depth` sets (`workers`
    threads) into its one device frame, so a frame is decoded once whatever the number of variants.  The steps' other device arguments are
    kept: the ids and widths per distinct weight-id tuple, and per (variant, n) the pose tensor that variant's steps update in place
    and their outputs.  So in each variant every step after a track set's first replays that variant's CUDA graph, across
    sequences too ('fp32' steps are never captured).  Each checkpoint steps in the sequence's n, as a run of it alone does, so
    every variant keeps that run's bits.  With 'fp8' among the modes, each weight set is calibrated on the first frame of the first
    sequence that tracks it, before that frame's steps, at the sequence's initial poses.  After each step the
    variant's poses are copied into its device history, which comes back to the host once per sequence.

    video: None, or (label order, [(paths, labels)] per sequence): paths holds one mp4 path per track, labels one text per frame.
    Then each frame's decode jobs also render its label strip into the ring, and after each step Engine.draw_tracks draws every
    track's Tracker.object_cloud points at its new pose over the device frame (the point sets uploaded once, as one table), and a
    VideoSink of `depth` sets writes the half-size frames; every video is complete when the generator is exhausted or closed.
    Videos are drawn for one variant only.

    opts: step_options' value for every step.  With opts.fit, each sequence's fit rows are {variant: (frames, n, 6) int32 numpy
    rows}, row t the fit of the step that wrote pose t.  With ICP the poses and fit rows are those after ICP.  With S > 1
    hypotheses the poses and fit rows are the kept hypotheses', and track j of frame t of sequence k draws with
    hypothesis_key(seq_index[k], t, j): seq_index is each sequence's index in the run's sorted list, so a share of the sequences
    on one GPU draws what the whole run draws.

    opts.reinit (re-initialisation of lost tracks): each sequence is then a 5-tuple whose last entry is the label-image file of
    every tracked frame, decoded through the same ring (its 'seg' field).  After each variant's step, Engine.reinit runs on that
    variant's poses and fit rows, in place, before the history copy: the labels are the class ids, the meshes the weight ids, and
    every (variant, sequence) has its own streaks, zero at the sequence's start.  The yield then has a third entry, {variant:
    (frames, n) int32 event codes}, and the fit rows are those after the restarts (None unless opts.fit)."""
    if video is not None and len(variants) != 1:
        raise ValueError('result videos are drawn for one variant, not %d' % len(variants))
    fp8 = {}                                               # checkpoint index -> its first fp8 variant
    for v in variants:
        if v[0] == 'fp8':
            fp8.setdefault(_variant_checkpoint(v), v)
    if not sequences:
        return
    dev = eng.device
    cam = trackers[sequences[0][2][0]].dataset_info['camera']
    H, W = int(cam['height']), int(cam['width'])
    spec = {'rgb': ((H, W, 3), torch.uint8), 'depth': ((H, W), torch.uint16)}
    if video is not None:
        spec['label'] = ((LABEL_TOP - LABEL_BOTTOM, W), torch.uint8)
    reinit = opts.reinit
    if reinit is not None:
        spec['seg'] = ((H, W), torch.uint8)
    ring = StagingRing(spec, depth, dev)
    frames = []
    for k, (rgb_files, depth_files) in enumerate(s[:2] for s in sequences):
        for t, (r, d) in enumerate(zip(rgb_files, depth_files)):
            jobs = [(_decode_into, 'rgb', read_rgb, r), (_decode_into, 'depth', read_depth, d)]
            if reinit is not None:
                jobs.append((_decode_into, 'seg', read_seg, sequences[k][4][t]))
            if video is not None:
                jobs.append((_label_into, video[1][k][1][t], H, W))
            frames.append(jobs)
    with contextlib.ExitStack() as stack:
        if video is not None:
            wids = sorted(set(w for s in sequences for w in s[2]))
            set_of = {w: j for j, w in enumerate(wids)}
            clouds = [np.asarray(trackers[w].object_cloud.points, dtype=np.float64).reshape(-1, 3) for w in wids]
            offsets = np.cumsum([0] + [len(p) for p in clouds]).astype(np.int32)
            table = torch.from_numpy(np.ascontiguousarray(np.concatenate(clouds))).to(dev)
            sink = stack.enter_context(contextlib.closing(VideoSink((max(len(s[2]) for s in sequences), H // 2, W // 2, 3), depth, dev)))
        uploads = stack.enter_context(contextlib.closing(ring.uploads(frames, workers)))
        by_ids, by_n = {}, {}
        for k, (rgb_files, _, ids, init) in enumerate(s[:4] for s in sequences):
            n = len(ids)
            for c in _checkpoints(variants):
                if (ids, c) not in by_ids:
                    wh = np.asarray(ids, dtype=np.int32) + CKPT_ID_STRIDE * c
                    by_ids[ids, c] = (wh, torch.from_numpy(wh).to(dev),
                                      torch.tensor([trackers[int(w)].object_width for w in wh], dtype=torch.float64, device=dev))
            for v in variants:
                if (v, n) not in by_n:
                    outs = dict(out_poses=torch.empty((n, 4, 4), dtype=torch.float64, device=dev),
                                out_trans=torch.empty((n, 3), dtype=torch.float32, device=dev),
                                out_rot=torch.empty((n, 3), dtype=torch.float32, device=dev))
                    keys = None
                    if opts.hypotheses > 1:                # the draw keys, choices and kept rows, at fixed addresses
                        keys = torch.empty(n, dtype=torch.int64, device=dev)
                        outs.update(out_choice=torch.empty(n, dtype=torch.int32, device=dev),
                                    out_fit=torch.empty((n, 6), dtype=torch.int32, device=dev))
                    by_n[v, n] = (outs, keys, None if video is None else torch.empty((n, H // 2, W // 2, 3), dtype=torch.uint8, device=dev))
                by_n[v, n][0]['out_poses'].copy_(torch.from_numpy(init))
            history = {v: torch.empty((len(rgb_files), n, 4, 4), dtype=torch.float64, device=dev) for v in variants}
            fit_rows = {v: torch.empty((len(rgb_files), n, 6), dtype=torch.int32, device=dev) for v in variants} \
                if opts.fit or reinit is not None else None
            if reinit is not None:                          # per variant: the streaks from 0, the event codes of every frame
                streaks = {v: torch.zeros(n, dtype=torch.int32, device=dev) for v in variants}
                events = {v: torch.empty((len(rgb_files), n), dtype=torch.int32, device=dev) for v in variants}
                labels = np.asarray(ids, dtype=np.int32)
            trk = trackers[ids[0]]
            track_set = None if video is None else np.asarray([set_of[w] for w in ids], dtype=np.int32)
            for t in range(len(rgb_files)):
                next(uploads)
                for c, v in (fp8.items() if t == 0 else ()):   # each set calibrated on the first frame of its first sequence
                    wh, wd, widths = by_ids[ids, c]
                    eng.calibrate_fp8_tracks(ring.dev['rgb'], ring.dev['depth'], trk.K, by_n[v, n][0]['out_poses'], widths, weight_ids=wh,
                                             render=dict(mode=trk.renderer.mode, image_hw=trk.renderer.image_hw, mesh_ids=wd))
                for v in variants:
                    wh, wd, widths = by_ids[ids, _variant_checkpoint(v)]
                    outs, keys, drawn = by_n[v, n]
                    poses = outs['out_poses']
                    if keys is not None:
                        keys.copy_(torch.arange(n, dtype=torch.int64, device=dev) + hypothesis_key(seq_index[k], t, 0))
                    track_step(eng, trackers, trk, ring.dev['rgb'], ring.dev['depth'], poses, widths, wh, wd, keys, opts, v[0], v[1],
                               dict(outs, out_fit=fit_rows[v][t]) if fit_rows else outs)
                    if reinit is not None:
                        events[v][t].copy_(eng.reinit(ring.dev['depth'], ring.dev['seg'], trk.K, labels, widths, poses, fit_rows[v][t],
                                                      streaks[v], opts.tau, reinit['below'], reinit['after'], weight_ids=wh,
                                                      mode=trk.renderer.mode, image_hw=trk.renderer.image_hw, init=reinit['init']))
                    history[v][t].copy_(poses)
                if video is not None:
                    eng.draw_tracks(ring.dev['rgb'], trk.K, poses, table, offsets, track_set,
                                    label=(H - LABEL_TOP, ring.dev['label']), label_order=video[0], out=drawn)
                    sink.put(drawn, video[1][k][0], last=t == len(rgb_files) - 1)
            res = ({v: h.cpu().numpy() for v, h in history.items()},
                   None if not opts.fit else {v: r.cpu().numpy() for v, r in fit_rows.items()})
            yield res if reinit is None else res + ({v: e.cpu().numpy() for v, e in events.items()},)


# ----------------------------------------------------------------------------------------------------
# The one-pass drivers on several GPUs (gpus=N): whole sequences are shared out over N ranks, one spawned process per GPU, each
# running _track_sequences on its share with its own Engine and Trackers and writing its sequences' files.  A sequence keeps its
# tracks, so every step has the n of the single-GPU run and the same bits (the trunk's split-K latency mode for n <= 4 and its
# throughput mode beyond are chosen by n).  The one state that passes between sequences is each weight set's fp8 calibration:
# every rank calibrates a set on the frame a single-GPU run uses, the first frame of the set's first sequence in run order.
# ----------------------------------------------------------------------------------------------------
def check_gpus(gpus):
    """The one-pass drivers' gpus argument -> int.  Below 1 is a ValueError; so is more than torch.cuda.device_count(), checked
    only for more than one, so gpus=1 asks nothing of the device."""
    if isinstance(gpus, bool) or int(gpus) != gpus:
        raise ValueError('gpus must be an integer, not %r' % (gpus,))
    gpus = int(gpus)
    if gpus < 1:
        raise ValueError('gpus must be at least 1, not %d' % gpus)
    if gpus > 1 and gpus > torch.cuda.device_count():
        raise ValueError('gpus=%d, but %d CUDA devices are visible' % (gpus, torch.cuda.device_count()))
    return gpus


def assign_ranks(costs, gpus):
    """Sequences onto ranks, greedy longest first: sequence i (cost costs[i], its frame count) goes to the rank with the least
    cost so far (among equals the one with the fewest sequences, then the lowest), the sequences taken by descending cost and then
    in order.  -> one ascending list of sequence indices per rank, min(gpus, len(costs)) ranks, none empty, each sequence on
    exactly one."""
    n = min(int(gpus), len(costs))
    loads, ranks = [0] * n, [[] for _ in range(n)]
    for i in sorted(range(len(costs)), key=lambda i: (-costs[i], i)):
        r = min(range(n), key=lambda r: (loads[r], len(ranks[r]), r))
        ranks[r].append(i)
        loads[r] += costs[i]
    return [sorted(r) for r in ranks]


def borrowed_calibrations(track_sets, mine):
    """Where a rank that tracks sequences `mine` (indices into track_sets, each sequence's weight ids in run order) calibrates the
    fp8 scales of weight sets it cannot calibrate itself -> {sequence index: [track indices]}.  A single-GPU run calibrates each set
    on the first frame of the first sequence that tracks it, at that sequence's initial poses (_track_sequences).  When that
    sequence is the rank's, its own loop does the same; for each other set the rank tracks, the entry names that sequence and the
    tracks of the sets whose first sequence it is."""
    first = {}
    for k, ids in enumerate(track_sets):
        for w in ids:
            first.setdefault(w, k)
    own = set(mine)
    needed = set(w for k in mine for w in track_sets[k])
    out = {}
    for w in sorted(needed):
        if first[w] not in own:
            out.setdefault(first[w], set()).add(w)
    return {k: [j for j, w in enumerate(track_sets[k]) if w in ws] for k, ws in sorted(out.items())}


def _rank_devices(n):
    """The CUDA device of each of n ranks: rank r runs on cuda:r of the visible devices."""
    return list(range(n))


def _checkpoints(variants):
    """The checkpoint indices of a run's variant keys, ascending."""
    return sorted(set(_variant_checkpoint(v) for v in variants))


def _checkpoint_sequences(sequences, c):
    """sequences with every track's weight id moved to checkpoint c's set."""
    return sequences if c == 0 else [(s[0], s[1], tuple(w + CKPT_ID_STRIDE * c for w in s[2])) + tuple(s[3:]) for s in sequences]


def _calibrate_borrowed(eng, trackers, sequences, borrowed):
    """The fp8 calibrations borrowed_calibrations names, in sequence order: each sequence's first frame decoded and calibrated at
    the initial poses of the named tracks, as _track_sequences calibrates it (Engine.calibrate_fp8_tracks, input A drawn by the
    rasteriser).  Calibration takes per-tensor maxima of each set's own tracks, so it gives the single-GPU run's scales."""
    for k, tracks in borrowed.items():
        rgb_files, depth_files, ids, init = sequences[k][:4]
        wh = np.asarray([ids[j] for j in tracks], dtype=np.int32)
        trk, dev = trackers[int(wh[0])], eng.device
        wd = torch.from_numpy(wh).to(dev)
        widths = torch.tensor([trackers[int(w)].object_width for w in wh], dtype=torch.float64, device=dev)
        poses = torch.from_numpy(np.ascontiguousarray(init[tracks])).to(dev)
        rgb = torch.from_numpy(read_rgb(rgb_files[0])).to(dev)
        depth = torch.from_numpy(read_depth(depth_files[0])).to(dev)
        eng.calibrate_fp8_tracks(rgb, depth, trk.K, poses, widths, weight_ids=wh,
                                 render=dict(mode=trk.renderer.mode, image_hw=trk.renderer.image_hw, mesh_ids=wd))


def _track_share(entries, precision, max_batch, sequences, mine, borrowed, variants, depth, workers, video, writes, opts):
    """One process's share of a one-pass run, sequences[k] for k in mine: the Engine and Trackers of `entries`
    (_one_pass_trackers), the fp8 calibrations borrowed from other shares (_calibrate_borrowed), then _track_sequences over the
    share with writes[k] (fn, *args) called as fn(*args, tracked) on sequence k's (poses, fit rows or None).  video: None, or
    (label order, [(paths, labels)] per sequence, folders to make once the trackers exist).  opts: _track_sequences' opts (the
    Engine holds max_batch x S tracks per step, and max_batch x init keep with re-initialisation).  -> (Engine, {k: what writes[k] returned})."""
    eng, trackers = _one_pass_trackers(entries, precision, max_batch * max(opts.hypotheses, reinit_keep(opts)))
    for c in _checkpoints(variants):                    # every checkpoint's sets, each on its own single-GPU frame
        _calibrate_borrowed(eng, trackers, _checkpoint_sequences(sequences, c), borrowed)
    drawn = None
    if video is not None:
        for d in video[2]:
            os.makedirs(d, exist_ok=True)
        drawn = (video[0], [video[1][k] for k in mine])
    out = {}
    for tracked, k in zip(_track_sequences(eng, trackers, [sequences[k] for k in mine], variants, depth, workers, drawn, opts,
                                           list(mine)), mine):
        fn, *args = writes[k]
        out[k] = fn(*args, tracked)
    return eng, out


def _rank_main(conn, rank, device, entries, precision, max_batch, sequences, mine, borrowed, variants, depth, workers, video,
               writes, opts):
    """Rank `rank` of a multi-GPU one-pass run, in its own process on cuda:`device`: _track_share with the weight sets of its
    sequences.  Sends ('ok', {k: what writes[k] returned}, {weight id: fp8 scales or None}) or ('error', traceback text) through
    conn."""
    import traceback
    try:
        wids = _rank_weight_ids(sequences, mine, variants)
        torch.cuda.set_device(device)
        eng, out = _track_share([e for e in entries if e[0] in wids], precision, max_batch, sequences, mine, borrowed, variants,
                                depth, workers, video, writes, opts)
        conn.send(('ok', out, {w: eng.fp8_scales(w) for w in sorted(wids)}))
    except BaseException:
        conn.send(('error', traceback.format_exc()))
    finally:
        conn.close()


def _rank_weight_ids(sequences, mine, variants):
    """The weight sets a rank tracking sequences `mine` loads: every checkpoint's set of each of their tracks."""
    return set(w + CKPT_ID_STRIDE * c for k in mine for w in sequences[k][2] for c in _checkpoints(variants))


def _agree_fp8_scales(per_rank):
    """The ranks' {weight id: fp8 scales or None} -> one such dict.  Ranks that both have scales for a set have the same ones:
    otherwise a RuntimeError, since the poses would depend on how the sequences were shared out."""
    out = {}
    for r, scales in enumerate(per_rank):
        for w, s in scales.items():
            if s is None:
                continue
            if w in out and not np.array_equal(out[w][1], s):
                raise RuntimeError('ranks %d and %d calibrated weight set %d differently: %s, %s' % (out[w][0], r, w, out[w][1], s))
            out.setdefault(w, (r, s))
    return {w: s for w, (_, s) in sorted(out.items())}


def _track_on_ranks(gpus, entries, precision, max_batch, sequences, variants, depth, workers, video, writes, opts):
    """_track_share over `sequences` on min(gpus, len(sequences)) GPUs, with writes[k] applied to sequence k's poses on its
    rank (_rank_main) -> [what writes[k] returned], in sequence order.  Sequences are shared out by assign_ranks on their
    frame counts; rank r runs as a spawned process on _rank_devices()[r].  A rank that raises or dies is a RuntimeError naming it,
    with its traceback; then, as on any other exit (KeyboardInterrupt included), every rank still running is terminated, and every
    rank is joined before this returns or raises."""
    import multiprocessing as mp
    from multiprocessing.connection import wait
    plan = assign_ranks([len(s[0]) for s in sequences], gpus)
    fp8 = any(v[0] == 'fp8' for v in variants)
    track_sets = [s[2] for s in sequences]
    devices = _rank_devices(len(plan))
    if len(_checkpoints(variants)) > 1:
        for r, mine in enumerate(plan):
            check_weight_sets_fit(len(_rank_weight_ids(sequences, mine, variants)), devices[r], 'weight sets (checkpoints x classes)')
    ctx = mp.get_context('spawn')
    procs, conns, done = [], [], False
    try:
        for r, mine in enumerate(plan):
            recv, send = ctx.Pipe(duplex=False)
            conns.append(recv)
            borrowed = borrowed_calibrations(track_sets, mine) if fp8 else {}
            p = ctx.Process(target=_rank_main, name='one-pass rank %d' % r, daemon=True,
                            args=(send, r, devices[r], entries, precision, max_batch, sequences, mine, borrowed, variants, depth,
                                  workers, video, writes, opts))
            try:
                p.start()
            finally:
                send.close()                       # the child's end: once the child exits, recv sees EOF
            procs.append(p)
        results, scales, pending = {}, {}, dict(enumerate(conns))
        while pending:
            ready = wait(list(pending.values()) + [procs[r].sentinel for r in pending])
            for r in [r for r, c in pending.items() if c in ready or procs[r].sentinel in ready]:
                try:
                    msg = pending[r].recv() if pending[r].poll() else None
                except EOFError:
                    msg = None
                if msg is None:
                    procs[r].join(5)
                    raise RuntimeError('rank %d (cuda:%d) exited with code %s before sending its results'
                                       % (r, devices[r], procs[r].exitcode))
                if msg[0] == 'error':
                    raise RuntimeError('rank %d (cuda:%d) failed:\n%s' % (r, devices[r], msg[1]))
                results.update(msg[1])
                scales[r] = msg[2]
                del pending[r]
        _agree_fp8_scales([scales[r] for r in range(len(plan))])
        done = True
    finally:
        for p in procs:
            if not done and p.is_alive():
                p.terminate()
        for p in procs:
            p.join(60)
            if p.is_alive():
                p.kill()
                p.join()
        for c in conns:
            c.close()
    return [results[k] for k in range(len(sequences))]


# The fit check in the one-pass drivers: FIT_FILE beside each sequence's pose files.  Not a .txt (eval_ycb globs **/*.txt under a
# tree) and never at a tree's root (eval_ycbineoat takes every root entry for a video folder).
FIT_FILE = 'fit.npy'
# --score's fit table: a frame whose ADD-S is at least this far from the annotation counts as lost (a fixed bound, not an option)
FIT_LOST_ADDS = 0.02
# Re-initialisation in the YCB-Video one-pass driver: REINIT_FILE beside each sequence's pose files, the event code of every
# pose file's step (include/se3tn.h: 0 not below, 1 below, 2 restarted, 3 no start, 4 rejected), row 0 (the start pose) -1
REINIT_FILE = 'reinit.npy'


def write_fit_rows(folder, rows):
    """<folder>/FIT_FILE: the fit rows of a sequence as int32 (frames, 6)."""
    os.makedirs(folder, exist_ok=True)
    np.save(os.path.join(folder, FIT_FILE), np.ascontiguousarray(rows, dtype=np.int32))


# What a one-pass driver's shared front hands its back: the GPU count, the first mode (the Trackers' precision, which
# ycb_all_classes / ycbineoat_objects check), the variants (_sweep_variants), whether modes and counts are swept, the
# checkpoints' configurations and the steps' options (step_options).
_OnePass = collections.namedtuple('_OnePass', 'gpus precision variants sweep ksweep configs opts')


def _one_pass_front(outdir, gpus, precision, modes, video, iterations, config, **step):
    """The checks both one-pass drivers make first, in this order, before anything is read: gpus (check_gpus), the precision
    modes among `modes` (precision_modes), one mode with video, the refinement counts (refine_counts), one count with video, the
    checkpoints of config's ckpt_dir / mean_std_path lists (checkpoint_configs), one checkpoint with video, then the steps'
    fit, hypotheses and ICP (step_options of `step`).  -> _OnePass."""
    gpus = check_gpus(gpus)
    modes, sweep = precision_modes(precision, modes)
    if video and len(modes) > 1:
        raise ValueError('video=True draws the result videos of one precision mode, not of %d' % len(modes))
    counts, ksweep = refine_counts(iterations)
    if video and len(counts) > 1:
        raise ValueError('video=True draws the result videos of one iteration count, not of %d' % len(counts))
    configs = checkpoint_configs(config)
    if video and len(configs) > 1:
        raise ValueError('video=True draws the result videos of one checkpoint, not of %d' % len(configs))
    return _OnePass(gpus, modes[0], _sweep_variants(outdir, modes, sweep, counts, ksweep, len(configs)), sweep, ksweep, configs,
                    step_options(**step))


def _one_pass_back(run, entries, max_batch, sequences, depth, workers, video, writes, collect):
    """The shared end of both one-pass drivers: `sequences` tracked in every variant of run (an _OnePass) with run.opts, in this
    process (_track_share over all of them, every entry loaded) or shared out over run.gpus ranks (_track_on_ranks), writes[k]
    applied to sequence k's (poses, fit rows or None).  Every entry's hypothesis spread is checked first (hypothesis_spread), and
    with several checkpoints a run whose weight sets do not fit in free device memory is refused (check_weight_sets_fit; per rank
    on several GPUs).  -> the driver's return value: _sweep_results of {variant: collect(written, variant)}, written being [what
    writes[k] returned] in sequence order."""
    for _, label, k in entries:
        hypothesis_spread(k['dataset_info'], run.opts, label)
    keys = tuple(v[:-1] for v in run.variants)
    if run.gpus == 1 and len(run.configs) > 1:
        check_weight_sets_fit(len(entries), what='weight sets (checkpoints x classes)')
    if run.gpus == 1:
        _, out = _track_share(entries, run.precision, max_batch, sequences, range(len(sequences)), {}, keys, depth, workers, video,
                              writes, run.opts)
        written = [out[k] for k in range(len(sequences))]
    else:
        written = _track_on_ranks(run.gpus, entries, run.precision, max_batch, sequences, keys, depth, workers, video, writes,
                                  run.opts)
    return _sweep_results({key: collect(written, key) for key in keys}, run.variants, run.sweep, run.ksweep)


def _ckpt_label(i, run):
    """' checkpoint <i>' in the labels of a run over several checkpoints, '' with one."""
    return ' checkpoint %d' % i if len(run.configs) > 1 else ''


def _write_ycb_all_sequence(dirs, seq_id, cls, init, tracked):
    """One test sequence's files of a getResultsYcbAll run: for each variant (dirs: {variant: {class id: result folder}}) and
    class, <folder>/seq<id>/%07d.txt, row 0 the start pose.  tracked: (poses, fit rows or None[, event codes]); with rows, each
    seq<id>/ also gets FIT_FILE, one row per pose file, row 0 (the start pose, not tracked) all -1; with event codes (a run with
    re-initialisation), REINIT_FILE, int32 (pose files,), row 0 -1.  -> {variant: (frames, n, 4, 4) poses}."""
    poses, rows = tracked[:2]
    events = tracked[2] if len(tracked) > 2 else None
    out = {}
    for v, folder in dirs.items():
        pred_poses = np.concatenate([init[None], poses[v]])      # row 0: the start pose, as in getResultsYcb
        for j, c in enumerate(cls):
            sdir = os.path.join(folder[c], 'seq{}'.format(seq_id))
            os.makedirs(sdir, exist_ok=True)
            for i in range(len(pred_poses)):
                np.savetxt(os.path.join(sdir, '%07d.txt' % i), pred_poses[i, j])
            if rows is not None:
                write_fit_rows(sdir, np.concatenate([np.full((1, 6), -1, np.int32), rows[v][:, j]]))
            if events is not None:
                np.save(os.path.join(sdir, REINIT_FILE), np.concatenate([[-1], events[v][:, j]]).astype(np.int32))
        out[v] = pred_poses
    return out


# ----------------------------------------------------------------------------------------------------
# Starts from the segmentation masks (Engine.init_poses): the one-pass YCB-Video driver's --init mask and --mode ycbv_init.  The
# label of class c in a YCB-Video seg/ image is c itself.
# ----------------------------------------------------------------------------------------------------
def read_seg(path):
    """A YCB-Video label image (seg/%06d-label.png) -> uint8 (H, W)."""
    import cv2
    s = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if s is None:
        raise FileNotFoundError(path)
    return np.ascontiguousarray(s if s.ndim == 2 else s[:, :, 0], dtype=np.uint8)


def ycb_label_file(color_file):
    """The seg/ label image of a YCB-Video frame: <seq>/seg/%06d-label.png beside <seq>/color/%06d-color.png."""
    seq_dir = os.path.dirname(os.path.dirname(color_file))
    return os.path.join(seq_dir, 'seg', os.path.basename(color_file).split('-')[0] + '-label.png')


def class_width(k):
    """The object width a Tracker of checked configuration k draws with (Tracker.__init__'s rule), in mm."""
    info = k['dataset_info']
    if 'object_width' in info:
        return float(info['object_width'])
    w = compute_obj_max_width(np.asarray(object_cloud(k['model_path']).points))
    return float(w + info['boundingbox'] / 100 * w)


class MaskStarts:
    """One Engine holding each class's CUDA-renderer mesh under its class id, for init calls of up to n_max classes of one frame
    (max_batch n_max x keep).  classes: checked configurations (class_id, model_path, dataset_info), sharing camera and render
    mode; init: Engine.init_spec's argument."""
    def __init__(self, classes, n_max, init=None):
        from .mesh_io import load_mesh
        self.init = init
        self.spec = Engine.init_spec(init)
        self.eng = Engine(max_batch=max(1, n_max * self.spec.keep))
        self.width = {}
        for k in classes:
            self.eng.set_mesh(load_mesh(k['model_path']), k['class_id'])
            self.width[k['class_id']] = class_width(k)
        cam = classes[0]['dataset_info']['camera']
        self.K = np.array([[cam['focalX'], 0, cam['centerX']], [0, cam['focalY'], cam['centerY']], [0, 0, 1]], dtype=np.float64)
        self.render = dict(mode='pyrender', image_hw=(int(cam['height']), int(cam['width']))) if _pyrender(classes[0]) else \
            dict(mode='vispy', image_hw=None)

    def __call__(self, depth, seg, cls, box=False, depths=None, out=None):
        """One init call for the classes cls (labels = ids = class ids) of one frame (uint16 depth, uint8 seg, numpy or CUDA) ->
        (poses (n, 4, 4), rows (n, INIT_COLS)) CUDA tensors, and out filled: Engine.init_poses, or with box Engine.init_boxes
        (D = depths, None: Engine.INIT_BOX_DEPTHS) on each class's tight box in seg (label_boxes: what a perfect detector
        gives; no pixels, an empty box and status 1)."""
        dev = self.eng.device
        as_dev = lambda a: a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        ids = np.asarray(cls, dtype=np.int32)
        widths = torch.tensor([self.width[int(c)] for c in cls], dtype=torch.float64, device=dev)
        kw = dict(weight_ids=ids, init=self.init, out=out, **self.render)
        if box:
            boxes = label_boxes(seg.cpu().numpy() if torch.is_tensor(seg) else seg, cls)
            return self.eng.init_boxes(as_dev(depth), boxes, self.K, widths, depths=Engine.INIT_BOX_DEPTHS if depths is None else depths, **kw)
        return self.eng.init_poses(as_dev(depth), as_dev(seg), self.K, ids, widths, **kw)

    def close(self):
        self.eng.close()


def label_boxes(seg, labels):
    """The tight half-open box (min u, min v, max u + 1, max v + 1) of each label's pixels in a uint8 label image, (0, 0, 0, 0)
    for a label without pixels -> int32 (n, 4)."""
    seg = np.asarray(seg)
    out = np.zeros((len(labels), 4), np.int32)
    for j, c in enumerate(labels):
        m = seg == int(c)
        rows, cols = np.flatnonzero(m.any(axis=1)), np.flatnonzero(m.any(axis=0))
        if len(rows):
            out[j] = (cols[0], rows[0], cols[-1] + 1, rows[-1] + 1)
    return out


def _mask_start_refusal(seq, c, name, status, source='mask'):
    return ValueError('sequence %04d, class %d (%s): no start from its %s in the first frame: %s (status %d)'
                      % (seq, c, name, source, Engine.init_status(status, source), int(status)))


def getResultsYcbAll(ycb_dir, class_ids, class_config, outdir, initialize_method='gt', precision='bf16x3', max_frames=None,
                     video=False, iterations=1, gpus=1, fit=None, hypotheses=1, seed=0, icp=0, icp_tau=None, init=None, reinit=None,
                     depths=None):
    """getResultsYcb for every class of `class_ids` in one pass -> {class_id: {seq_id: poses}}, and the files each per-class run
    writes, under <outdir>/<class folder>/run/ (see ycb_all_classes for class_config and the refusals).

    precision: one mode of YCB_ALL_PRECISIONS, or a sweep: a sequence of them or 'all' (all five).  'fp16' is refused here, alone
    or in a sequence, while getResultsYcbInEOAT takes it.  A sweep tracks every frame in every mode (one step per mode, each frame
    decoded once, every weight set loaded once) and returns {mode: what a run in that mode returns}; mode m writes its tree under
    <outdir>/<m>/, file for file what a run in mode m with that outdir writes.  score_precisions scores it.  Unknown or repeated
    modes, an empty sequence, and video=True with more than one mode are a ValueError before anything is loaded.

    One Engine holds every class's weights, statistics and CUDA-renderer mesh under weight id = class id.  For each test sequence,
    the tracks are its requested classes in ascending order, each started as getResultsYcb starts it, and every frame after the
    first is one se3tn_track_render step for all of them (_track_sequences: each frame decoded once, two frames ahead).

    video: also write the result video a per-class run writes next to its seq<id>/ (predict.py:403, 424-435): <outdir>/<class
    folder>/run/seq<id>.mp4, one half-size frame per tracked frame (none for the start pose), the class's model points drawn at
    their tracked pose over the frame, under the label 'frame:<i+1>' of frame i.  The drawing runs on the device.

    iterations: k, the refinement rounds of every step (Engine.track_render; 1, today's step, writes what a run without the
    argument writes), or a sweep: a sequence of counts.  A sweep of counts tracks every frame once per (mode, k) and returns
    {k: what a run with that k returns}; count k writes its tree under <outdir>/iter<k>/ (with <mode>/ below it when modes are
    swept too), file for file what a run with that k and mode writes.  score_iterations scores it.  Counts outside [1, 8], repeated
    counts, an empty sequence, and video=True with more than one variant are a ValueError before anything is loaded.

    gpus: the number of GPUs, one process each (1: this process alone).  With N > 1 the test sequences are shared out whole over
    min(N, sequences) spawned ranks on cuda:0 .. cuda:N-1 (assign_ranks, on frame counts); each rank loads the weight sets of its
    sequences, tracks them as above and writes their files and videos, every file the one a single-GPU run writes.  The return
    value equals the single-GPU run's, bit for bit and in the same order, and so do the files; each fp8 set is calibrated on the
    frame a single-GPU run calibrates it on (borrowed_calibrations).  gpus below 1 or above torch.cuda.device_count() is a
    ValueError before anything is loaded, as is every other refusal; a rank that fails is a RuntimeError with its traceback,
    raised after every rank has stopped (_track_on_ranks).

    class_config['ckpt_dir'] (and 'mean_std_path') may be lists of templates, one per checkpoint (checkpoint_configs): every
    frame is then tracked once per (checkpoint, mode, k), checkpoint i's sets under weight id class id + 32 i, its tree under
    <outdir>/ckpt<i>/ file for file what a run of it alone writes, and the return value is {i: what that run returns}.
    score_checkpoints scores it.  video=True takes one checkpoint; weight sets beyond the device's free memory are refused.

    fit: tau in mm turns on every step's fit check (Engine.track_render's fit): each class's seq<id>/ of every tree also gets
    FIT_FILE, int32 (pose files, 6), row i the fit of the step that wrote pose i, row 0 -1.  The pose files and the return value
    are what the run without it gives.  score_fit reads it.

    hypotheses: S in [1, 32].  S > 1 tracks every step from S start hypotheses per track around its previous pose, spread by its
    class's dataset_info max_translation / max_rotation, and keeps the one that fits the frame best (Tracker(hypotheses=S),
    _track_sequences' hyp); the pose files hold the kept poses and FIT_FILE, with fit, the kept rows.  Track j of frame t of
    sequence k (the run's sorted list) draws with key hypothesis_key(k, t, j) and `seed`, on one GPU or several.  S = 1 is the
    plain run, file for file.

    icp: M iterations of ICP after every step's last round (Engine.track_render's icp), at the gate icp_tau mm
    (Engine.ICP_TAU_DEFAULT when None); the pose files hold the refined poses and FIT_FILE, with fit, the fit after ICP.  0 is the
    plain run, file for file; several GPUs write the one-GPU trees.  Refused with hypotheses > 1 (step_options).

    initialize_method='mask': each sequence's tracks start from one Engine.init_poses call on its first frame (depth_filled and
    seg/ label image; each class's label is its class id; init: Engine.init_spec's argument), made in this process before any
    tracking, so several GPUs write the one-GPU trees.  A class the call finds no start for (an empty mask, too few pixels with
    depth) is a ValueError naming the sequence and the class.  init without 'mask' or 'box' is a ValueError.

    initialize_method='box': as 'mask', with one Engine.init_boxes call (depths: its D, None the default) whose boxes are each
    class's tight box in that label image (label_boxes), a perfect detector's boxes; a class without pixels has an empty box
    and no start.  depths without 'box' is a ValueError.

    reinit: None off, or {'below': f, 'after': L, 'init': Engine.init_spec's argument} (reinit_options): after every step, the
    tracks whose inlier fraction stayed below f for L frames in a row are restarted from that frame's seg/%06d-label.png (the
    label of class c is c) by Engine.reinit, and a start replaces the tracked pose only when it fits the frame better.  The pose
    files, FIT_FILE and the video hold the poses after the restarts; each class's seq<id>/ also gets REINIT_FILE, the event code
    of every pose file (row 0 -1).  Every variant, checkpoint and sequence has its own streaks, zero at the sequence's start.
    It turns the fit check on at FIT_TAU_DEFAULT when fit is not given; the Engine then holds n_max x init keep tracks (the
    steps' split-K regime depends on n alone, so their bits do not move).  Every tracked frame's label image must exist: a
    missing one is a FileNotFoundError before anything is loaded.  Several GPUs write the one-GPU trees."""
    if init is not None and initialize_method not in ('mask', 'box'):
        raise ValueError("init options need initialize_method='mask' or 'box', not %r" % (initialize_method,))
    if depths is not None and initialize_method != 'box':
        raise ValueError("depths needs initialize_method='box', not %r" % (initialize_method,))
    if initialize_method in ('mask', 'box'):
        Engine.init_spec(init)
    if initialize_method == 'box':
        Engine.depths_spec(Engine.INIT_BOX_DEPTHS if depths is None else depths)
    run = _one_pass_front(outdir, gpus, precision, YCB_ALL_PRECISIONS, video, iterations, class_config, fit=fit,
                          hypotheses=hypotheses, seed=seed, icp=icp, icp_tau=icp_tau, reinit=reinit)
    if initialize_method not in ('gt', 'posecnn', 'poserbpf', 'mask', 'box'):
        raise ValueError('initialize_method must be gt, posecnn, poserbpf, mask or box')
    _check_checkpoint_ids([c for c, _ in ycb_classes(ycb_dir, class_ids)], len(run.configs), 'class')
    per_ckpt = [ycb_all_classes(ycb_dir, class_ids, cfg, run.precision) for cfg in run.configs]
    classes = per_ckpt[0]
    track_sets = ycb_track_sets(ycb_dir, [k['class_id'] for k in classes])
    data_dir = '{}/data_organized/'.format(ycb_dir)
    keyframes_all = read_keyframes(ycb_dir) if initialize_method == 'posecnn' else []
    sequences = []
    if run.opts.reinit is not None:                       # every tracked frame's label image, before anything is loaded
        for seq_id, cls in track_sets.items():
            rgb_files = _ycb_sequence_files(os.path.join(data_dir, '%04d' % seq_id), cls[0])[0]
            nf = len(rgb_files) if max_frames is None else min(len(rgb_files), 1 + max_frames)
            missing = [p for p in (ycb_label_file(r) for r in rgb_files[1:nf]) if not os.path.isfile(p)]
            if missing:
                raise FileNotFoundError('reinit: %d tracked frames of sequence %04d have no label image, the first %s'
                                        % (len(missing), seq_id, missing[0]))
    starts = MaskStarts(classes, max([len(v) for v in track_sets.values()] + [1]), init) if initialize_method in ('mask', 'box') else None
    try:
        for seq_id, cls in track_sets.items():
            files = {c: _ycb_sequence_files(os.path.join(data_dir, '%04d' % seq_id), c) for c in cls}
            rgb_files, depth_files, _ = files[cls[0]]
            nf = len(rgb_files) if max_frames is None else min(len(rgb_files), 1 + max_frames)
            if starts is not None:
                import glob
                segs = sorted(glob.glob(os.path.join(data_dir, '%04d' % seq_id, 'seg', '*')))
                if not segs:
                    raise FileNotFoundError('--init %s: no seg/ label image under %s' % (initialize_method, os.path.join(data_dir, '%04d' % seq_id)))
                P, rows = starts(read_depth(depth_files[0]), read_seg(segs[0]), cls, initialize_method == 'box', depths)
                P, rows = P.cpu().numpy(), rows.cpu().numpy()
                for j, c in enumerate(cls):
                    if rows[j, 0]:
                        raise _mask_start_refusal(seq_id, c, [k['name'] for k in classes if k['class_id'] == c][0], rows[j, 0],
                                                  initialize_method)
                init_poses = P
            else:
                init_poses = np.stack([_ycb_first_pose(ycb_dir, c, seq_id, files[c][2][0], initialize_method, keyframes_all,
                                                       sorted(findClassContainedVideosYcb(c, data_dir, testset=True)))
                                       for c in cls]).astype(np.float64)
            sequences.append((rgb_files[1:nf], depth_files[1:nf], tuple(cls), init_poses)
                             + (() if run.opts.reinit is None else ([ycb_label_file(r) for r in rgb_files[1:nf]],)))
    finally:
        if starts is not None:
            starts.close()
    entries = [(k['class_id'] + CKPT_ID_STRIDE * i, 'class %d (%s)' % (k['class_id'], k['name']) + _ckpt_label(i, run), k)
               for i, cl in enumerate(per_ckpt) for k in cl]
    max_batch = max([len(v) for v in track_sets.values()] + [1])
    name_of = {k['class_id']: k['name'] for k in classes}
    drawn = None
    if video:
        tree = run.variants[0][-1]
        drawn = ('under', [([os.path.join(ycb_all_res_dir(tree, name_of[c]), 'seq%d.mp4' % seq_id) for c in cls],
                            ['frame:%d' % (i + 1) for i in range(1, 1 + len(s[0]))]) for (seq_id, cls), s in zip(track_sets.items(), sequences)],
                 [ycb_all_res_dir(tree, c) for c in name_of.values()])
    dirs = {v[:-1]: {c: ycb_all_res_dir(v[-1], name) for c, name in name_of.items()} for v in run.variants}
    writes = [(_write_ycb_all_sequence, dirs, seq_id, tuple(cls), s[3]) for (seq_id, cls), s in zip(track_sets.items(), sequences)]

    def collect(written, key):
        out = {c: {} for c in name_of}
        for pred_poses, (seq_id, cls) in zip(written, track_sets.items()):
            for j, c in enumerate(cls):
                out[c][seq_id] = pred_poses[key][:, j]
        return out
    return _one_pass_back(run, entries, max_batch, sequences, 2, 2, drawn, writes, collect)


# ----------------------------------------------------------------------------------------------------
# Every YCBInEOAT video in one pass: the paper's Table II as one run instead of one predictSequenceYcbInEOAT run per video.  One
# Engine holds each object's weights, statistics and mesh; each frame is one n = 1 se3tn_track_render step, decoded ahead by a
# thread pool.  The output tree is what eval_ycbineoat.eval_all scores:  <outdir>/<video>/%07d.txt
# Per-object configuration is the four YCB_ALL_TEMPLATES path templates with {object} (a name of eval_ycbineoat.OBJECTS) and,
# with ycb_dir, {class_name} (the CADmodels/ folder of the object) placeholders.
# ----------------------------------------------------------------------------------------------------
YCBINEOAT_TRANS_NORMALIZER, YCBINEOAT_ROT_NORMALIZER = 0.03, 30 * np.pi / 180       # predict.py:586-587


def ycbineoat_videos(root):
    """[(video folder name, object)], sorted by name: every folder under root with rgb/, depth_filled/ and annotated_poses/
    (.tar.gz entries skipped).  A video folder that names no object is a ValueError naming it."""
    from .eval_ycbineoat import OBJECTS, video_object
    videos = []
    for name in sorted(os.listdir(root)):
        d = os.path.join(root, name)
        if '.tar.gz' in name or not all(os.path.isdir(os.path.join(d, sub)) for sub in ('rgb', 'depth_filled', 'annotated_poses')):
            continue
        obj = video_object(name)
        if obj is None:
            raise ValueError('video folder %s names none of the objects %s' % (d, OBJECTS))
        videos.append((name, obj))
    return videos


def ycbineoat_class_name(ycb_dir, obj):
    """The CADmodels/ folder of an object: the first, in sorted order, whose name contains it."""
    for name in ycb_class_names(ycb_dir):
        if obj in name:
            return name
    raise FileNotFoundError('object %s: no CADmodels/ folder under %s contains its name' % (obj, ycb_dir))


def expand_object_paths(object_config, obj, class_name=None):
    """The four path templates of object_config for one object -> {train_data_path, mean_std_path, ckpt_dir, model_path}."""
    ph = dict(object=obj) if class_name is None else dict(object=obj, class_name=class_name)
    return _expand_templates(object_config, 'object_config', **ph)


def ycbineoat_objects(objects, object_config, ycb_dir=None, precision='bf16x3'):
    """The checked configuration of each object, before anything is loaded onto a device -> {object: dict of the expanded paths,
    dataset_info, mean, std}.  A missing file is a FileNotFoundError naming the object and the path.  The frames of all videos go
    through one set of buffers, so the objects must share the camera and the render mode."""
    from .engine import PREC
    if precision not in PREC:
        raise ValueError('unknown precision %r (one of %s)' % (precision, ', '.join(PREC)))
    out = {}
    for obj in objects:
        cname = ycbineoat_class_name(ycb_dir, obj) if ycb_dir else None
        out[obj] = dict(_load_run_files('object %s' % obj, expand_object_paths(object_config, obj, cname)), object=obj)
    if out:
        _check_shared(list(out.values()), lambda k: 'object %s' % k['object'], lambda k: 'object %s' % k['object'],
                      (('camera', _camera), ('renderer', _pyrender)), 'all videos are tracked through one set of frame buffers')
    return out


def write_video_poses(outdir, video, poses):
    """<outdir>/<video>/%07d.txt, one np.savetxt pose per frame: what eval_ycbineoat.eval_all reads with res_dir = outdir + '/'."""
    vdir = os.path.join(outdir, video)
    os.makedirs(vdir, exist_ok=True)
    for i in range(len(poses)):
        np.savetxt(os.path.join(vdir, '%07d.txt' % i), poses[i])


def _write_ycbineoat_video(roots, video, tracked):
    """One video's files of a getResultsYcbInEOAT run: write_video_poses under each variant's tree (roots: {variant: tree}).
    tracked: (poses, fit rows or None); with rows, <tree>/<video>/ also gets FIT_FILE, one row per pose file (every frame is
    tracked).  -> {variant: (frames, 4, 4) poses}."""
    poses, rows = tracked
    out = {}
    for key, root in roots.items():
        out[key] = poses[key][:, 0]
        write_video_poses(root, video, out[key])
        if rows is not None:
            write_fit_rows(os.path.join(root, video), rows[key][:, 0])
    return out


def getResultsYcbInEOAT(ycbineoat_dir, object_config, outdir, precision='bf16x3', max_frames=None, decode_ahead=4, ycb_dir=None,
                        video=False, iterations=1, gpus=1, fit=None, hypotheses=1, seed=0, icp=0, icp_tau=None):
    """predictSequenceYcbInEOAT for every video under ycbineoat_dir in one pass -> {video: (frames,4,4) poses}, and
    <outdir>/<video>/%07d.txt for each frame, which eval_ycbineoat.eval_all scores with res_dir = outdir + '/'.

    Videos and objects as ycbineoat_videos and ycbineoat_objects find and check them.  One Engine holds each object's weights,
    statistics and CUDA-renderer mesh once, under one weight id per object.  Each video starts from its annotated_poses[0] and is
    tracked from frame 0 with the reference's normalisers (0.03 m, 30 degrees), one n = 1 se3tn_track_render step per frame, so
    every step after an object's first replays its CUDA graph (_track_sequences).  A thread pool decodes up to decode_ahead
    frames ahead, across video boundaries, into a ring of that many pinned staging sets.

    video: also write <outdir>/<video>.mp4, a headless stand-in for the window predictSequenceYcbInEOAT shows (predict.py:612-624;
    the reference itself writes no file there): per frame i, the object's model points drawn at the tracked pose over the frame
    with the label 'frame:<i>' over them, at half size.  The drawing runs on the device.  eval_ycbineoat lists the .mp4 files
    among the result folders and finds no pose file in them, so the scores are unchanged.

    precision: one mode of engine.PREC, or a sweep: a sequence of them or 'all' (all six, PRECISIONS).  Unlike getResultsYcbAll,
    which refuses 'fp16', every mode is taken here.  A sweep tracks every frame in every mode (one step per mode, each frame
    decoded once, every weight set loaded once) and returns {mode: what a run in that mode returns}; mode m writes its tree under
    <outdir>/<m>/, file for file what a run in mode m with that outdir writes.  score_precisions scores it.  Unknown or repeated
    modes, an empty sequence, and video=True with more than one mode are a ValueError before anything is loaded.

    iterations: k refinement rounds per step, or a sweep of counts, as in getResultsYcbAll: count k of a sweep writes under
    <outdir>/iter<k>/ (then <mode>/ when modes are swept too).

    gpus: the number of GPUs, as in getResultsYcbAll: whole videos shared out over min(gpus, videos) ranks, each decoding
    decode_ahead frames ahead of its own steps and writing its videos' files; the return value and the files equal the
    single-GPU run's.

    object_config['ckpt_dir'] (and 'mean_std_path') may be lists of templates, one per checkpoint, as in getResultsYcbAll:
    checkpoint i's sets under weight id object index + 32 i, its tree under <outdir>/ckpt<i>/.

    fit: as in getResultsYcbAll; <tree>/<video>/FIT_FILE has one row per pose file, frame 0 included (it is tracked).
    hypotheses, seed: as in getResultsYcbAll, sequence k being the k-th video of the sorted list.
    icp, icp_tau: as in getResultsYcbAll."""
    from .eval_ycbineoat import OBJECTS
    run = _one_pass_front(outdir, gpus, precision, PRECISIONS, video, iterations, object_config, fit=fit, hypotheses=hypotheses,
                          seed=seed, icp=icp, icp_tau=icp_tau)
    decode_ahead = int(decode_ahead)
    if decode_ahead < 1:
        raise ValueError('decode_ahead must be at least 1')
    videos = ycbineoat_videos(ycbineoat_dir)
    files = {v: sequence_files(os.path.join(ycbineoat_dir, v)) for v, _ in videos}
    used = [o for o in OBJECTS if any(o == ob for _, ob in videos)]
    _check_checkpoint_ids([OBJECTS.index(o) for o in used], len(run.configs), 'object')
    entries = [(OBJECTS.index(o) + CKPT_ID_STRIDE * i, 'object %s' % o + _ckpt_label(i, run),
                dict(k, trans_normalizer=YCBINEOAT_TRANS_NORMALIZER, rot_normalizer=YCBINEOAT_ROT_NORMALIZER))
               for i, cfg in enumerate(run.configs) for o, k in ycbineoat_objects(used, cfg, ycb_dir, run.precision).items()]
    sequences = {}
    for v, obj in videos:
        rgb_files, depth_files, gt_files = files[v]
        nf = len(rgb_files) if max_frames is None else min(max_frames, len(rgb_files))
        if nf > 0:
            sequences[v] = (rgb_files[:nf], depth_files[:nf], (OBJECTS.index(obj),), np.loadtxt(gt_files[0]).reshape(1, 4, 4))
    drawn = None
    if video:
        tree = run.variants[0][-1]
        drawn = ('over', [([os.path.join(tree, v + '.mp4')], ['frame:%d' % i for i in range(len(s[0]))]) for v, s in sequences.items()],
                 [tree])
    trees = {v[:-1]: v[-1] for v in run.variants}
    writes = [(_write_ycbineoat_video, trees, v) for v in sequences]
    return _one_pass_back(run, entries, 1, list(sequences.values()), decode_ahead, 2 * decode_ahead, drawn, writes,
                          lambda written, key: {v: w[key] for v, w in zip(sequences, written)})


# ----------------------------------------------------------------------------------------------------
# Pose recovery from perturbed starts on the YCB-Video key frames (--mode ycbv_recover): the perturbed poses `produce_train_pair_data
# --mode ycbv` keeps (ProducerPurturb.generate: "sample various purturbation around for evaluating the mean error") become track
# starts on their own key frame, K refinement rounds run in one tracking step, and every round's pose is scored against the
# annotation: translation / rotation error, ADD, ADD-S and their VOCap AUCs, per class and pooled.
# ----------------------------------------------------------------------------------------------------
RECOVER_GPUS_REFUSAL = ('ycbv_recover runs on one GPU: the perturbations of a key frame are drawn after every earlier frame\'s '
                        'visibility check, so the frames cannot be shared out')


def recover_front(precision='bf16x3', iterations=1, gpus=1):
    """The argument checks of recoverYcbKeyframes, before anything is read -> (modes, K).  precision: a mode of YCB_ALL_PRECISIONS,
    'all' or a list of them ('fp16' refused, as in ycbv_all); iterations: one K in [1, 8]; gpus: 1 (RECOVER_GPUS_REFUSAL).  Every
    refusal is a ValueError."""
    if gpus != 1:
        raise ValueError(RECOVER_GPUS_REFUSAL)
    modes, _ = precision_modes(precision, YCB_ALL_PRECISIONS)
    if modes[0] not in YCB_ALL_PRECISIONS:
        raise ValueError('precision %r is not a mode of ycbv_recover (one of %s)' % (modes[0], ', '.join(YCB_ALL_PRECISIONS)))
    if isinstance(iterations, (list, tuple)) or isinstance(iterations, bool):
        raise ValueError('ycbv_recover takes one iteration count K (every round 1..K is scored), not %r' % (iterations,))
    return modes, _refine_iterations(iterations)


def pair_mesh_base(class_ids, ckpts):
    """The mesh id of class 0's producer mesh in a ycbv_recover run: CKPT_ID_STRIDE x ckpts, above the weight ids c + 32 i of every
    checkpoint i < ckpts, under which the tracking meshes live.  A producer mesh id base + c that is also a weight id is a
    ValueError."""
    base = CKPT_ID_STRIDE * int(ckpts)
    weights = {int(c) + CKPT_ID_STRIDE * i for c in class_ids for i in range(int(ckpts))}
    clash = sorted(base + int(c) for c in class_ids if base + int(c) in weights)
    if clash:
        raise ValueError('producer mesh ids %s (%d + class id) are also weight ids of the tracking meshes; class ids must stay below %d'
                         % (', '.join(map(str, clash)), base, CKPT_ID_STRIDE))
    return base


def pair_model_template(class_config):
    """The producers' mesh template: class_config['pair_model_path'], else model_path with .ply -> .obj, as ProducerPurturb picks
    it (produce_train_pair_data.py:76)."""
    return class_config.get('pair_model_path') or str(class_config['model_path']).replace('.ply', '.obj')


def pose_errors_np(pred, gt):
    """se3tn_pose_errors_sets' translation error (mm) and rotation angle (degrees) in numpy fp64: pred, gt (n, 4, 4) -> (n, 2)."""
    pred = np.asarray(pred, np.float64).reshape(-1, 4, 4)
    gt = np.asarray(gt, np.float64).reshape(-1, 4, 4)
    d = pred[:, :3, 3] - gt[:, :3, 3]
    trans = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]) * 1000.0
    tr = np.zeros(len(pred))
    for i in range(3):
        for j in range(3):
            tr = tr + pred[:, i, j] * gt[:, i, j]
    rot = np.degrees(np.arccos(np.clip((tr - 1.0) / 2.0, -1.0, 1.0)))
    return np.stack([trans, rot], 1)


def _recover_summary(errors, add_auc, adds_auc):
    """One table row's values from (rows, 4) errors (mm, degrees, ADD, ADD-S) and the two AUCs; None values with no row."""
    n = int(errors.shape[0])
    if n == 0:
        return dict(rows=0, add_auc=None, adds_auc=None, rot_mean=None, rot_median=None, trans_mean=None, trans_median=None)
    return dict(rows=n, add_auc=float(add_auc), adds_auc=float(adds_auc), rot_mean=float(np.mean(errors[:, 1])),
                rot_median=float(np.median(errors[:, 1])), trans_mean=float(np.mean(errors[:, 0])), trans_median=float(np.median(errors[:, 0])))


def recoverYcbKeyframes(ycb_dir, class_ids, class_config, num_sample=10, seed=0, precision='bf16x3', iterations=1, max_frames=None,
                        decode_ahead=4, workers=None, gpus=1, hypotheses=1, icp=0, icp_tau=None):
    """Pose recovery from perturbed starts on the YCB-Video key frames, every class in one pass.

    The frame loop is `produce_train_pair_data --mode ycbv`'s own (ycbv_pair_steps, random / np.random seeded with `seed`): the same
    visibility check, draws, centre test and pair step, so a class's kept rows are the pairs that mode writes with this seed and
    num_sample, in its order, with its A_in_cam / B_in_cam, and the RNG ends in the same state.  The producers draw the mesh of
    class_config['pair_model_path'] (default model_path with .ply -> .obj, pair_model_template) under mesh ids pair_mesh_base(...)
    + class id; the tracks draw model_path under their weight ids.

    Each frame's rows (the samples inside the image, classes in order) are n tracks of one se3tn_track_render step (round_poses) per
    variant, started at their A_in_cam on the ring's device frame, with their class's weight set, statistics, mesh and
    Tracker.object_width, refined K times; a row whose segB count is below 100 (the writer drops it) is tracked but not scored:
    the counts stay on the device as the keep mask of se3tn_pose_errors_sets.  After the last frame every round r = 0 (the start)
    .. K of every row is scored against B_in_cam in one launch per round and variant, against the tracking mesh's points
    (Tracker.object_cloud), and se3tn_vocap_sets gives the per-class and pooled ADD / ADD-S AUCs.

    class_config: the ycbv_all templates (YCB_ALL_TEMPLATES, optional normalisers), refused as ycb_all_classes refuses them;
    ckpt_dir / mean_std_path may be lists (checkpoint i's set of class c is weight id c + 32 i).  precision: one mode, 'all' or a
    list (recover_front); iterations: one K in 1..8; gpus: 1.  Every frame is decoded and cut once, then stepped once per
    (checkpoint, mode); fp8 calibrates each set on its own rows of the first frame that has any (Engine.calibrate_fp8_tracks).
    Each variant's numbers are those of a run with that checkpoint and mode alone.  max_frames: the first key frames only.

    -> {variant: {class id: dict, ..., 'all': dict}}, variant (mode, K) with one checkpoint, (mode, K, checkpoint index) with several.
    Each dict: rows, A_in_cam / B_in_cam (rows, 4, 4), poses (K, rows, 4, 4) after each round, errors (K + 1, rows, 4) (translation
    mm, rotation degrees, ADD m, ADD-S m; index 0 the start), and summary: K + 1 dicts of _recover_summary (AUCs in [0, 1]).

    hypotheses: S in [1, 32].  S > 1 makes every row's step track S hypotheses around its A_in_cam (track_step: the spread of
    its class's dataset_info, the fit check at step_options' tau, row j of key frame f keyed hypothesis_key(f, j, 0) and `seed`).
    poses / errors / summary are then hypothesis 0's rounds (an n x S-track step's), and each dict also has 'selected' (the fit's
    choice) and 'best' (per row the hypothesis with the lowest ADD-S against B_in_cam, the bound any selection rule can reach),
    each a dict of poses (rows, 4, 4), errors (rows, 4), summary (one _recover_summary), and 'choice' (rows,) for 'selected'
    and 'best', all at round K.

    icp: M > 0 refines every row with M ICP iterations after round K in the same step (Engine.track_render's icp, gate icp_tau mm,
    Engine.ICP_TAU_DEFAULT when None; refused with hypotheses > 1).  poses / errors / summary then run on past round K: entries
    K + 1 .. K + M are the poses after ICP iterations 1 .. M (out_icp_poses), and each dict has 'icp': M.  Rounds 0 .. K are
    those of the run without it, bit for bit."""
    from . import _lib
    from .produce_train_pair_data import ycbv_producers, ycbv_pair_steps, ycbv_keyframe_jobs
    modes, K = recover_front(precision, iterations, gpus)
    opts = step_options(hypotheses=hypotheses, seed=seed, icp=icp, icp_tau=icp_tau)
    S, M = opts.hypotheses, 0 if opts.icp is None else _engine.Engine.icp_spec(opts.icp).iterations
    configs = checkpoint_configs(class_config)
    ids = [c for c, _ in ycb_classes(ycb_dir, class_ids)]
    if not ids:
        raise ValueError('no class ids given')
    _check_checkpoint_ids(ids, len(configs), 'class')
    base = pair_mesh_base(ids, len(configs))
    per_ckpt = [ycb_all_classes(ycb_dir, ids, cfg, modes[0]) for cfg in configs]
    pair_tpl = dict(train_data_path=class_config['train_data_path'], model_path=pair_model_template(class_config))
    entries = [(k['class_id'] + CKPT_ID_STRIDE * i, 'class %d (%s)' % (k['class_id'], k['name']) + (' checkpoint %d' % i if len(configs) > 1 else ''), k)
               for i, cl in enumerate(per_ckpt) for k in cl]
    if len(configs) > 1:
        check_weight_sets_fit(len(entries), what='weight sets (checkpoints x classes)')
    for _, label, k in entries:
        hypothesis_spread(k['dataset_info'], opts, label)
    eng, trackers = _one_pass_trackers(entries, modes[0], max(1, len(ids) * int(num_sample)) * S)
    _, producers = ycbv_producers(ycb_dir, ids, pair_tpl, eng, workers, mesh_base=base)
    variants = [(m, K) + ((i,) if len(configs) > 1 else ()) for i in range(len(configs)) for m in modes]
    dev = eng.device
    set_of = {c: j for j, c in enumerate(ids)}
    random.seed(seed); np.random.seed(seed)
    jobs = ycbv_keyframe_jobs(ycb_dir, ids)
    if max_frames is not None:
        jobs = jobs[:int(max_frames)]
    trk = trackers[entries[0][0]]
    render = dict(mode=trk.renderer.mode, image_hw=trk.renderer.image_hw)
    starts, counts, row_set, row_B, rounds = [], [], [], [], {v: [] for v in variants}
    picked = {v: ([], [], []) for v in variants} if S > 1 else None     # per variant: selected poses, choices, every hypothesis
    by_n, by_cls = {}, {}
    for f, (owners, chunks, (rgb, depth)) in enumerate(ycbv_pair_steps(eng, producers, jobs, num_sample, decode_ahead, workers, on_device=True,
                                                        with_frame=True)):
        cls = tuple(c for c, _, inside, _ in owners for _ in inside)
        n = len(cls)
        if n not in by_n:                                  # per n: the start poses, draw keys and each variant's outputs, at fixed addresses
            outs = {}
            for v in variants:
                o = dict(out_poses=torch.empty((n, 4, 4), dtype=torch.float64, device=dev),
                         out_trans=torch.empty((n, 3), dtype=torch.float32, device=dev),
                         out_rot=torch.empty((n, 3), dtype=torch.float32, device=dev))
                if S > 1:                                  # every hypothesis after each round; hypothesis 0's rounds are scored
                    o.update(out_choice=torch.empty(n, dtype=torch.int32, device=dev), out_fit=torch.empty((n, 6), dtype=torch.int32, device=dev),
                             out_hyp_poses=torch.empty((n, S, 4, 4), dtype=torch.float64, device=dev),
                             out_rounds=torch.empty((K, n, S, 4, 4), dtype=torch.float64, device=dev))
                    scored = o['out_rounds'][:, :, 0]
                else:                                      # the network's rounds, then (with icp) the poses after each ICP iteration
                    scored = torch.empty((K + M, n, 4, 4), dtype=torch.float64, device=dev)
                    o.update(out_rounds=scored[:K], **({'out_icp_poses': scored[K:]} if M else {}))
                outs[v] = (o, scored)
            by_n[n] = (torch.empty((n, 4, 4), dtype=torch.float64, device=dev), outs,
                       torch.empty(n, dtype=torch.int64, device=dev) if S > 1 else None)
        start, outs, keys = by_n[n]
        start.copy_(torch.cat([r['A_in_cam'] for _, r in chunks]))
        counts.append(torch.cat([r['count'] for _, r in chunks]))
        starts.append(start.clone())
        row_set += [set_of[c] for c in cls]
        row_B += [B for c, B, inside, _ in owners for _ in inside]
        for v in variants:
            i = _variant_checkpoint(v)
            if (cls, i) not in by_cls:
                wh = np.asarray(cls, dtype=np.int32) + CKPT_ID_STRIDE * i
                by_cls[cls, i] = (wh, torch.from_numpy(wh).to(dev),
                                  torch.tensor([trackers[int(w)].object_width for w in wh], dtype=torch.float64, device=dev))
            wh, wd, widths = by_cls[cls, i]
            if v[0] == 'fp8':                              # sets without scales: calibrated on their own rows of this frame
                eng.calibrate_fp8_tracks(rgb, depth, trk.K, start, widths, weight_ids=wh, render=dict(render, mesh_ids=wd))
            o, scored = outs[v]
            if keys is not None:
                keys.copy_(torch.arange(n, dtype=torch.int64, device=dev) * (1 << 16) + hypothesis_key(f, 0, 0))
            track_step(eng, trackers, trk, rgb, depth, start, widths, wh, wd, keys, opts, v[0], K, o)
            rounds[v].append(scored.clone())
            if picked is not None:
                for acc, t in zip(picked[v], (o['out_poses'], o['out_choice'], o['out_hyp_poses'])):
                    acc.append(t.clone())
    out = _score_recovery(eng, trackers, ids, variants, K + M, starts, counts, row_set, row_B, rounds, _lib.PAIR_MIN_SEG, picked)
    if M:
        for res in out.values():
            for d in res.values():
                d['icp'] = M
    return out


def _score_recovery(eng, trackers, ids, variants, K, starts, counts, row_set, row_B, rounds, min_seg, picked=None):
    """recoverYcbKeyframes' scoring, after the last frame: every round of every row in one se3tn_pose_errors_sets launch per round
    and variant (rows whose count is below min_seg masked), one read-back, then se3tn_vocap_sets per round and metric.  picked:
    None, or per variant the hypothesis steps' (selected poses, choices, every hypothesis's poses) per frame: the selected rows
    and every hypothesis are scored the same way, and 'best' takes per row the hypothesis of lowest ADD-S."""
    dev = eng.device
    N = len(row_set)
    S = len(ids)
    clouds = [np.asarray(trackers[c].object_cloud.points, dtype=np.float64).reshape(-1, 3) for c in ids]
    offsets = np.cumsum([0] + [len(p) for p in clouds]).astype(np.int32)
    table = torch.from_numpy(np.ascontiguousarray(np.concatenate(clouds))).to(dev)
    pose_set = np.asarray(row_set, dtype=np.int32)
    if N:
        A = torch.cat(starts)
        B = torch.from_numpy(np.ascontiguousarray(np.stack(row_B), dtype=np.float64)).to(dev)
        keep = (torch.cat(counts) >= min_seg).to(torch.uint8)
        err0, kept_set = eng.pose_errors_sets(table, pose_set, A, B, offsets, keep)
        per_v = {v: torch.cat(rounds[v], 1) for v in variants}
        errs = {v: torch.stack([err0] + [eng.pose_errors_sets(table, pose_set, per_v[v][r], B, offsets, keep)[0] for r in range(K)])
                for v in variants}
        kept = (kept_set >= 0).cpu().numpy()
    else:
        kept = np.zeros(0, bool)
    kidx = torch.from_numpy(np.flatnonzero(kept)).to(dev)
    kset = pose_set[kept]
    A_h = A.index_select(0, kidx).cpu().numpy() if N else np.zeros((0, 4, 4))
    B_h = B.index_select(0, kidx).cpu().numpy() if N else np.zeros((0, 4, 4))
    out = {}
    for v in variants:
        E = errs[v].index_select(1, kidx) if N else torch.zeros((K + 1, 0, 4), dtype=torch.float64, device=dev)
        P = per_v[v].index_select(1, kidx).cpu().numpy() if N else np.zeros((K, 0, 4, 4))
        aucs = [(eng.vocap_sets(E[r, :, 2].contiguous(), kset, S), eng.vocap_sets(E[r, :, 3].contiguous(), kset, S)) for r in range(K + 1)]
        Eh = E.cpu().numpy()
        extra = {}
        if picked is not None:
            extra = _score_hypotheses(eng, table, pose_set, offsets, B if N else None, keep if N else None, picked[v], kidx, kset, S)
        res = {}
        for j, c in enumerate(ids + ['all']):
            rows = np.flatnonzero(kset == j) if c != 'all' else np.arange(len(kset))
            res[c] = dict(rows=len(rows), A_in_cam=A_h[rows], B_in_cam=B_h[rows], poses=P[:, rows], errors=Eh[:, rows],
                          summary=[_recover_summary(Eh[r, rows], aucs[r][0][j], aucs[r][1][j]) for r in range(K + 1)])
            for name, (Pk, Ek, ch, ap) in extra.items():
                res[c][name] = dict(poses=Pk[rows], errors=Ek[rows], choice=ch[rows],
                                    summary=_recover_summary(Ek[rows], ap[0][j], ap[1][j]))
        out[v] = res
    return out


def _score_hypotheses(eng, table, pose_set, offsets, B, keep, picked, kidx, kset, n_sets):
    """recoverYcbKeyframes' two hypothesis rows for one variant: {'selected' | 'best': (poses, errors (rows, 4), choice,
    (ADD AUCs, ADD-S AUCs))} over the kept rows, 'best' being per row the hypothesis of lowest ADD-S (the first on a tie)."""
    if B is None:
        z = (np.zeros((0, 4, 4)), np.zeros((0, 4)), np.zeros(0, np.int32), ([0.0] * (n_sets + 1), [0.0] * (n_sets + 1)))
        return {'selected': z, 'best': z}
    sel, choice, every = (torch.cat(x) for x in picked)
    S = every.shape[1]
    E_sel = eng.pose_errors_sets(table, pose_set, sel, B, offsets, keep)[0]
    E_all = eng.pose_errors_sets(table, np.repeat(pose_set, S), every.reshape(-1, 4, 4).contiguous(), B.repeat_interleave(S, 0),
                                 offsets, keep.repeat_interleave(S, 0))[0].reshape(-1, S, 4)
    best = torch.nan_to_num(E_all[:, :, 3], nan=float('inf')).argmin(1)
    rows = torch.arange(len(best), device=best.device)
    E_best, P_best = E_all[rows, best], every[rows, best]
    out = {}
    for name, E, P, ch in (('selected', E_sel, sel, choice.long()), ('best', E_best, P_best, best)):
        E = E.index_select(0, kidx)
        ap = (eng.vocap_sets(E[:, 2].contiguous(), kset, n_sets), eng.vocap_sets(E[:, 3].contiguous(), kset, n_sets))
        out[name] = (P.index_select(0, kidx).cpu().numpy(), E.cpu().numpy(), ch.index_select(0, kidx).cpu().numpy(), ap)
    return out


def init_classes(ycb_dir, class_ids, class_config):
    """--mode ycbv_init's classes: [dict class_id, name, dataset_info, model_path] from class_config's train_data_path (its
    ../dataset_info.yml) and model_path templates; no checkpoint is read.  A missing file is a FileNotFoundError naming the class;
    classes must share the camera and the render mode (one init call per frame draws all of them)."""
    import yaml
    classes = []
    for c, name in ycb_classes(ycb_dir, class_ids):
        label = 'class %d (%s)' % (c, name)
        paths = {}
        for key in ('train_data_path', 'model_path'):
            if key not in class_config:
                raise ValueError('class_config needs a %r template' % key)
            paths[key] = str(class_config[key]).format(class_id=c, class_name=name)
        info_path = os.path.join(paths['train_data_path'], '../dataset_info.yml')
        for what, path in (('dataset_info.yml', info_path), ('mesh', paths['model_path'])):
            if not os.path.isfile(path):
                raise FileNotFoundError('%s: no %s file at %s' % (label, what, path))
        with open(info_path, 'r') as ff:
            classes.append(dict(class_id=c, name=name, dataset_info=yaml.safe_load(ff), model_path=paths['model_path']))
    if not classes:
        raise ValueError('no class ids given')
    _check_shared(classes, lambda k: 'class %d (%s)' % (k['class_id'], k['name']), lambda k: 'class %d' % k['class_id'],
                  (('camera', _camera), ('renderer', _pyrender)), 'classes started in one call must share it')
    return classes


INIT_ROWS = ('grid', 'icp', 'best of K')


def initYcbKeyframes(ycb_dir, class_ids, class_config, init=None, max_frames=None, box=False, depths=None):
    """Starts from the masks scored on the YCB-Video key frames: no checkpoint, no tracking.  The frames are the key frames of
    ycbv_recover's loop (produce_train_pair_data.ycbv_keyframe_jobs: every key frame with an annotated requested class), each
    with its depth_filled and seg/ images; each is one Engine.init_poses call (MaskStarts) for all its annotated classes, label =
    class id.  Every row is scored against its pose_gt with se3tn_pose_errors_sets against the class's model points
    (object_cloud), and se3tn_vocap_sets gives the per-class and pooled ADD / ADD-S AUCs.  Rows: 'grid' the top grid candidate,
    'icp' the returned pose, 'best of K' per row the kept candidate (after ICP when init has it) of lowest ADD-S, which bounds
    any final choice.  A row whose call reports status != 0 is counted as failed and not scored.  max_frames: the first key
    frames only.  box: each call is Engine.init_boxes (MaskStarts with box, D = depths, None the default) with each class's
    tight box in the key frame's label image, a perfect detector's boxes; a class without pixels gets an empty box and counts
    as failed.  depths without box is a ValueError.

    -> {class id: dict, ..., 'all': dict}; each dict: rows (scored), failed, gt (rows, 4, 4), and per row name of INIT_ROWS a
    dict of poses (rows, 4, 4), errors (rows, 4) (translation mm, rotation degrees, ADD m, ADD-S m) and summary
    (_recover_summary)."""
    from .produce_train_pair_data import ycbv_keyframe_jobs
    spec = Engine.init_spec(init)
    if depths is not None and not box:
        raise ValueError('initYcbKeyframes: depths needs box=True')
    if box:
        Engine.depths_spec(Engine.INIT_BOX_DEPTHS if depths is None else depths)
    classes = init_classes(ycb_dir, class_ids, class_config)
    ids = [k['class_id'] for k in classes]
    jobs = ycbv_keyframe_jobs(ycb_dir, ids)
    if max_frames is not None:
        jobs = jobs[:int(max_frames)]
    starts = MaskStarts(classes, len(ids), init)
    try:
        eng, dev, Kk = starts.eng, starts.eng.device, spec.keep
        set_of = {c: j for j, c in enumerate(ids)}
        row_set, gts, status, grid, final, cands = [], [], [], [], [], []
        for rgb_path, depth_path, seg_path, rows in jobs:
            cls = [c for c, _ in rows]
            n = len(cls)
            out = dict(kept_poses=torch.empty((n, Kk, 4, 4), dtype=torch.float64, device=dev))
            if spec.icp:
                out['icp_poses'] = torch.empty((n, Kk, 4, 4), dtype=torch.float64, device=dev)
            P, R = starts(read_depth(depth_path), read_seg(seg_path), cls, box, depths, out=out)
            row_set += [set_of[c] for c in cls]
            gts += [B for _, B in rows]
            status.append(R[:, 0].clone())
            grid.append(out['kept_poses'][:, 0].clone())
            final.append(P.clone())
            cands.append((out['icp_poses'] if spec.icp else out['kept_poses']).clone())
        N = len(row_set)
        clouds = [np.asarray(object_cloud(k['model_path']).points, dtype=np.float64).reshape(-1, 3) for k in classes]
        offsets = np.cumsum([0] + [len(p) for p in clouds]).astype(np.int32)
        table = torch.from_numpy(np.ascontiguousarray(np.concatenate(clouds))).to(dev)
        pose_set = np.asarray(row_set, dtype=np.int32)
        ok = (torch.cat(status) == 0) if N else torch.zeros(0, dtype=torch.bool, device=dev)
        kidx = torch.nonzero(ok).reshape(-1)
        kset = pose_set[ok.cpu().numpy()]
        B = torch.from_numpy(np.ascontiguousarray(np.stack(gts), dtype=np.float64)).to(dev) if N else None
        keep = ok.to(torch.uint8)
        scored = {}
        if N:
            for name, Pn in (('grid', torch.cat(grid)), ('icp', torch.cat(final))):
                scored[name] = (Pn, eng.pose_errors_sets(table, pose_set, Pn, B, offsets, keep)[0])
            every = torch.cat(cands)
            E_all = eng.pose_errors_sets(table, np.repeat(pose_set, Kk), every.reshape(-1, 4, 4).contiguous(), B.repeat_interleave(Kk, 0),
                                         offsets, keep.repeat_interleave(Kk, 0))[0].reshape(-1, Kk, 4)
            best = torch.nan_to_num(E_all[:, :, 3], nan=float('inf')).argmin(1)
            r = torch.arange(N, device=dev)
            scored['best of K'] = (every[r, best], E_all[r, best])
        res = {}
        for name in INIT_ROWS:
            if N:
                Pn, En = (x.index_select(0, kidx) for x in scored[name])
                ap = (eng.vocap_sets(En[:, 2].contiguous(), kset, len(ids)), eng.vocap_sets(En[:, 3].contiguous(), kset, len(ids)))
                Pn, En = Pn.cpu().numpy(), En.cpu().numpy()
            else:
                Pn, En, ap = np.zeros((0, 4, 4)), np.zeros((0, 4)), ([0.0] * (len(ids) + 1),) * 2
            for j, c in enumerate(ids + ['all']):
                sel = np.flatnonzero(kset == j) if c != 'all' else np.arange(len(kset))
                d = res.setdefault(c, dict(rows=len(sel), gt=(B.index_select(0, kidx).cpu().numpy()[sel] if N else np.zeros((0, 4, 4)))))
                d[name] = dict(poses=Pn[sel], errors=En[sel], summary=_recover_summary(En[sel], ap[0][j], ap[1][j]))
        failed = (~ok).cpu().numpy()
        for j, c in enumerate(ids + ['all']):
            res[c]['failed'] = int((failed & (pose_set == j)).sum()) if c != 'all' else int(failed.sum())
        return res
    finally:
        starts.close()


def print_init_tables(results, names):
    """initYcbKeyframes' tables: one per class (names: {class id: label}), then the pooled one, in the columns of
    print_recover_tables plus the failed rows; AUCs in percent, errors in degrees and mm."""
    head = '%-10s %6s %6s %8s %8s %9s %9s %9s %9s' % ('start', 'rows', 'failed', 'ADD', 'ADD-S', 'rot mean', 'rot med', 'trans mean',
                                                    'trans med')
    for c, d in results.items():
        label = 'all classes' if c == 'all' else 'class %d (%s)' % (c, names.get(c, c))
        print('%s: %d rows scored, %d failed; AUCs in percent (VOCap, 0.1 m), rotation in degrees, translation in mm'
              % (label, d['rows'], d['failed']))
        print(head)
        for name in INIT_ROWS:
            s = d[name]['summary']
            if s['rows'] == 0:
                print('%-10s %6d %6d' % (name, 0, d['failed']))
                continue
            print('%-10s %6d %6d %8.3f %8.3f %9.4g %9.4g %9.4g %9.4g' % (name, s['rows'], d['failed'], 100 * s['add_auc'], 100 * s['adds_auc'],
                                                                        s['rot_mean'], s['rot_median'], s['trans_mean'], s['trans_median']))


def print_recover_tables(results, names):
    """recoverYcbKeyframes' tables: one per class (names: {class id: label}), then the pooled one; a row per (checkpoint, mode,
    round), round 0 (the perturbed start, the same in every variant) printed once.  AUCs in percent, errors in degrees and mm."""
    variants = list(results)
    first = results[variants[0]]
    head = '%-5s %-8s %5s %6s %8s %8s %9s %9s %9s %9s' % ('ckpt', 'mode', 'round', 'rows', 'ADD', 'ADD-S', 'rot mean', 'rot med',
                                                       'trans mean', 'trans med')

    def line(ckpt, mode, r, s):
        if s['rows'] == 0:
            return '%-5s %-8s %5s %6d' % (ckpt, mode, r, 0)
        return '%-5s %-8s %5s %6d %8.3f %8.3f %9.4g %9.4g %9.4g %9.4g' % (ckpt, mode, r, s['rows'], 100 * s['add_auc'], 100 * s['adds_auc'],
                                                                       s['rot_mean'], s['rot_median'], s['trans_mean'], s['trans_median'])
    for c in first:
        label = 'all classes' if c == 'all' else 'class %d (%s)' % (c, names.get(c, c))
        print('%s: %d rows; AUCs in percent (VOCap, 0.1 m), rotation in degrees, translation in mm' % (label, first[c]['rows']))
        print(head)
        print(line('-', 'start', 0, first[c]['summary'][0]))
        for v in variants:
            s = results[v][c]['summary']
            K = len(s) - 1 - results[v][c].get('icp', 0)                 # rows past round K: 'icp 1' .. 'icp M'
            for r in range(1, len(s)):
                print(line(str(_variant_checkpoint(v)), v[0], r if r <= K else 'icp %d' % (r - K), s[r]))
            for name, label in (('selected', 'selected'), ('best', 'best of S')):
                if name in results[v][c]:
                    print(line(str(_variant_checkpoint(v)), v[0], len(s) - 1, results[v][c][name]['summary']) + '  ' + label)


def score_precisions(results, outdir, ycb_dir, config, YCBInEOAT_dir=None):
    """What each mode of a precision sweep scores, and how far it drifts from the reference mode.  results: what getResultsYcbAll
    (YCBInEOAT_dir None) or getResultsYcbInEOAT returned for a sweep, {mode: ...}; outdir, ycb_dir and config (the path
    templates) those of the run.  -> (reference mode, {mode: {'add', 'adds', 'add_max', 'add_mean', 'adds_max', 'adds_mean'}}).

    add / adds: the ADD and ADD-S AUCs (percent) of the mode's tree <outdir>/<mode>/ from the existing scorers, whose lines are
    printed under a 'precision <mode>' header: eval_ycbineoat.eval_all; for YCB-Video eval_ycb.eval_all when all 21 classes were
    tracked, else eval_ycb.eval_one_class per class, with the errors of all classes pooled through eval_ycb.VOCap.
    add_* / adds_*: ADD and ADD-S between every pose the mode returned and the reference mode's pose of the same track and frame,
    max and mean in mm, on each class's or object's Tracker.object_cloud points; one add_adi_sets launch per mode.  No ground
    truth is involved, so it also shows where modes part ways on frames without annotations.  The reference is
    sweep_reference(modes), whose own row is 0."""
    modes = list(results)
    ref = sweep_reference(modes)
    return ref, _score_variants(results, {m: precision_outdir(outdir, m) for m in modes}, ref, 'precision %s', ycb_dir, config,
                                YCBInEOAT_dir)


def score_iterations(results, outdir, ycb_dir, config, YCBInEOAT_dir=None, precision='bf16x3'):
    """score_precisions for a sweep of refinement counts: results what getResultsYcbAll / getResultsYcbInEOAT returned for
    iterations=[k1, k2, ...] with this precision (a mode, or the modes of a precision sweep).  One row per variant, labelled by its
    tree under outdir: 'iter<k>', or 'iter<k>/<mode>' when modes were swept too, each with its AUCs and its drift from the k = 1
    tree of the sweep's reference mode (sweep_reference; the smallest k swept when 1 is not).  -> (reference label, rows)."""
    sweep = precision_modes(precision, PRECISIONS)[1]
    modes = list(next(iter(results.values()))) if sweep else [precision]
    label = lambda k, m: os.path.relpath(precision_outdir(iterations_outdir(outdir, k), m) if sweep else iterations_outdir(outdir, k), outdir)
    flat = {label(k, m): (res[m] if sweep else res) for k, res in results.items() for m in modes}
    ref = label(1 if 1 in results else min(results), sweep_reference(modes))
    return ref, _score_variants(flat, {v: os.path.join(outdir, v) for v in flat}, ref, 'variant %s', ycb_dir, config, YCBInEOAT_dir)


def score_checkpoints(results, outdir, ycb_dir, config, YCBInEOAT_dir=None, precision='bf16x3', iterations=1):
    """score_precisions for a run over several checkpoints: results what getResultsYcbAll / getResultsYcbInEOAT returned,
    {checkpoint index: ...}, for this precision (a mode or a sweep) and iterations (a count or a sweep); config the run's
    templates (ckpt_dir / mean_std_path lists).  One row per variant, labelled by its tree under outdir ('ckpt<i>', then
    '/iter<k>' and '/<mode>' when those were swept), each with its AUCs and its drift from checkpoint 0 in the sweep's reference
    mode (sweep_reference) and k (1, or the smallest swept).  -> (reference label, rows)."""
    sweep = precision_modes(precision, PRECISIONS)[1]
    counts, ksweep = refine_counts(iterations)
    one = results[0][counts[0]] if ksweep else results[0]
    modes = tuple(one) if sweep else (precision,)
    variants = _sweep_variants(outdir, modes, sweep, counts, ksweep, len(results))
    flat, roots = {}, {}
    for m, k, c, tree in variants:
        label = os.path.relpath(tree, outdir)
        r = results[c][k] if ksweep else results[c]
        flat[label], roots[label] = (r[m] if sweep else r), tree
    k0 = 1 if 1 in counts else min(counts)
    ref = next(os.path.relpath(t, outdir) for m, k, c, t in variants if c == 0 and m == sweep_reference(modes) and k == k0)
    return ref, _score_variants(flat, roots, ref, 'variant %s', ycb_dir, checkpoint_configs(config)[0], YCBInEOAT_dir)


def best_checkpoints(rows):
    """{variant below ckpt<i>/ ('' when only checkpoints vary): (checkpoint index, its ADD-S AUC)}, the checkpoint with the highest
    ADD-S AUC among the rows of score_checkpoints, the first listed among equals."""
    from .problems import best_checkpoint
    groups = {}
    for label, r in rows.items():
        head, _, sub = label.partition('/')
        groups.setdefault(sub, []).append((int(head[len('ckpt'):]), r['adds']))
    out = {}
    for sub, got in groups.items():
        b = best_checkpoint([-a for _, a in got])
        out[sub] = got[b]
    return out


def print_best_checkpoints(rows, ckpts):
    """After score_checkpoints' table: one line per mode (and k) naming the checkpoint with the highest ADD-S AUC."""
    ckpts = [ckpts] if isinstance(ckpts, str) else list(ckpts)
    for sub, (i, adds) in best_checkpoints(rows).items():
        print('best%s: checkpoint %d (%s), ADD-S %.4f' % (' ' + sub if sub else '', i, ckpts[i], adds))


def _score_variants(results, roots, ref, header, ycb_dir, config, YCBInEOAT_dir):
    """The rows of score_precisions / score_iterations: results {label: what one variant's run returned}, roots {label: its tree},
    ref the label drift is measured from; each variant's scorer lines are printed under header % label."""
    import argparse
    from .eval_ycbineoat import eval_all, video_object
    modes = list(results)
    if YCBInEOAT_dir is None:
        names = ycb_class_names(ycb_dir)
        keys = [(c, s) for c in sorted(results[ref]) for s in sorted(results[ref][c])]
        poses_of = lambda m, key: results[m][key[0]][key[1]]
        model_of = {key: expand_class_paths(config, key[0], names[key[0] - 1])['model_path'] for key in keys}
    else:
        keys = sorted(results[ref])
        poses_of = lambda m, key: results[m][key]
        model_of = {v: expand_object_paths(config, video_object(v), ycbineoat_class_name(ycb_dir, video_object(v)) if ycb_dir else None)
                    ['model_path'] for v in keys}
    paths = sorted(set(model_of.values()))
    clouds = [object_cloud(p).points for p in paths]
    pose_set = np.concatenate([np.full(len(poses_of(ref, k)), paths.index(model_of[k]), dtype=np.int32) for k in keys])
    eng = U._eng()
    stacked = lambda m: torch.from_numpy(np.ascontiguousarray(np.concatenate([poses_of(m, k) for k in keys]).reshape(-1, 4, 4),
                                                              dtype=np.float64)).to(eng.device)
    ref_poses = stacked(ref)
    rows = {}
    for m in modes:
        print(header % m)
        root = roots[m]
        if YCBInEOAT_dir is None:
            adds, add = _score_ycb_tree(ycb_dir, root, sorted(results[m]))
        else:
            _, adds, add, _ = eval_all(argparse.Namespace(YCBInEOAT_dir=YCBInEOAT_dir, ycb_dir=ycb_dir, res_dir=root + '/'))
        d_add, d_adds = (d.cpu().numpy() * 1000 for d in eng.add_adi_sets(clouds, pose_set, stacked(m), ref_poses))
        rows[m] = dict(add=add, adds=adds, add_max=float(d_add.max()), add_mean=float(d_add.mean()),
                       adds_max=float(d_adds.max()), adds_mean=float(d_adds.mean()))
    return rows


def _score_ycb_tree(ycb_dir, root, class_ids):
    """eval_ycb's lines for a getResultsYcbAll tree under root -> (ADD-S AUC, ADD AUC) in percent: eval_all when the tree holds
    all 21 classes (it pools exactly those), else eval_one_class per class, the errors of all of them pooled through VOCap."""
    import argparse
    from . import eval_ycb
    names = ycb_class_names(ycb_dir)
    if list(class_ids) == list(range(1, 22)) and len(names) == 21:
        adi_auc, add_auc, _ = eval_ycb.eval_all(argparse.Namespace(ycb_dir=ycb_dir, res_root=root))
        return adi_auc, add_auc
    errs = [eval_ycb.eval_one_class(argparse.Namespace(ycb_dir=ycb_dir, class_id=c, res_dir=ycb_all_res_dir(root, names[c - 1]) + '/'))
            for c in class_ids]
    return (eval_ycb.VOCap(np.concatenate([e[0] for e in errs])) * 100, eval_ycb.VOCap(np.concatenate([e[1] for e in errs])) * 100)


def roc_auc(score, positive):
    """Area under the ROC curve of `score` as a detector of `positive` (bool): the chance that a random positive scores above a
    random negative, ties counting half.  NaN without positives or without negatives."""
    score, positive = np.asarray(score, np.float64), np.asarray(positive, bool)
    npos, nneg = int(positive.sum()), int((~positive).sum())
    if npos == 0 or nneg == 0:
        return float('nan')
    _, inv, counts = np.unique(score, return_inverse=True, return_counts=True)
    ranks = (np.cumsum(counts) - (counts - 1) / 2.0)[inv]          # 1-based ranks, ties averaged
    return float((ranks[positive].sum() - npos * (npos + 1) / 2.0) / (npos * nneg))


def _fit_frames(root, ycb_dir, YCBInEOAT_dir=None, class_ids=None):
    """The frames the tree's scorer scores that a step tracked, from the pose files and each folder's FIT_FILE -> (ADD-S in m,
    fit rows (frames, 6)).  YCB-Video (class_ids): eval_ycb.eval_one_class's key frames of every class; YCBInEOAT: every frame
    eval_ycbineoat.eval_all scores.  ADD-S is computed as those scorers compute it, on the same points and annotations."""
    import glob
    from . import eval_ycb, eval_ycbineoat
    eng = U._eng()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.stack(a).reshape(-1, 4, 4), dtype=np.float64)).to(eng.device)
    adds, rows = [], []

    def add(points, preds, gts, fit):
        if preds:
            adds.append(eng.add_adi(torch.from_numpy(np.ascontiguousarray(points)).to(eng.device), t(preds), t(gts))[1].cpu().numpy())
            rows.append(np.stack(fit))
    if YCBInEOAT_dir is None:
        names = ycb_class_names(ycb_dir)
        model_files = sorted(glob.glob('{}/CADmodels/**/points.xyz'.format(ycb_dir), recursive=True))
        with open('{}/YCB_Video_toolbox/keyframe.txt'.format(ycb_dir)) as ff:
            keyframes = set(line.rstrip() for line in ff.readlines())
        for c in class_ids:
            res_dir = ycb_all_res_dir(root, names[c - 1]) + '/'
            preds, gts, fit, loaded = [], [], [], {}
            for pose_file in sorted(glob.glob(res_dir + '**/*.txt', recursive=True)):
                seq_dir = os.path.dirname(pose_file)
                seq_id = int(pose_file.replace(res_dir, '').split('/')[0].replace('seq', ''))
                i = int(os.path.basename(pose_file).split('.')[0])
                if '%04d/%06d' % (seq_id, i + 1) not in keyframes:
                    continue
                r = loaded.setdefault(seq_dir, np.load(os.path.join(seq_dir, FIT_FILE)))[i]
                if (r == -1).all():                      # the start pose: no step tracked it
                    continue
                preds.append(np.loadtxt(pose_file)); fit.append(r)
                gts.append(np.loadtxt('{}/data_organized/%04d/pose_gt/{}/%06d.txt'.format(ycb_dir, c) % (seq_id, i + 1)))
            add(eval_ycb._read_points(model_files[c - 1]), preds, gts, fit)
    else:
        models = eval_ycbineoat.model_points(ycb_dir)
        for folder in sorted(os.listdir(root)):
            d = os.path.join(root, folder)
            if not os.path.isfile(os.path.join(d, FIT_FILE)):
                continue
            r = np.load(os.path.join(d, FIT_FILE))
            pred_files = sorted(glob.glob(d + '/*.txt'))
            gt_files = sorted(glob.glob(os.path.join(YCBInEOAT_dir, folder, 'annotated_poses', '*.txt')))
            add(models[eval_ycbineoat.video_object(folder)], [np.loadtxt(f) for f in pred_files],
                [np.loadtxt(f) for f in gt_files[:len(pred_files)]], list(r[:len(pred_files)]))
    if not adds:
        return np.zeros(0), np.zeros((0, 6), np.int32)
    return np.concatenate(adds), np.concatenate(rows)


def score_fit(root, ycb_dir, YCBInEOAT_dir=None, class_ids=None):
    """How well the fit check flags lost frames in one variant's tree (a run with fit): over the frames _fit_frames finds, a frame
    is lost when its ADD-S is at least FIT_LOST_ADDS (2 cm).  -> {'frames', 'lost' (share), 'inlier_lost' / 'inlier_kept' (mean
    inlier fraction of the lost frames / of the rest, NaN for none), 'auc' (ROC AUC of 1 - inlier fraction as a detector of
    the lost frames)}."""
    adds, rows = _fit_frames(root, ycb_dir, YCBInEOAT_dir, class_ids)
    lost = adds >= FIT_LOST_ADDS
    inl = fit_fractions(rows)['inlier']
    mean = lambda a: float(a.mean()) if len(a) else float('nan')
    return dict(frames=int(len(adds)), lost=mean(lost.astype(np.float64)), inlier_lost=mean(inl[lost]), inlier_kept=mean(inl[~lost]),
                auc=roc_auc(1.0 - inl, lost))


def score_reinit(root, ycb_dir, class_ids):
    """What re-initialisation did in one variant's tree of a YCB-Video run with reinit, from each seq<id>/'s REINIT_FILE ->
    {'tracked' frames (pose files a step wrote, over every class), 'below' (event != 0), 'attempts' (events 2, 3 and 4: every
    frame has its mask here, so these are the lost frames),
    'restarted', 'rejected', 'failed' (no start), 'restarts_near' (the share of restarted poses within FIT_LOST_ADDS ADD-S of
    the annotation, on the class's points.xyz as eval_ycb reads them; NaN without restarts)}."""
    import glob
    from . import eval_ycb
    eng = U._eng()
    names = ycb_class_names(ycb_dir)
    model_files = sorted(glob.glob('{}/CADmodels/**/points.xyz'.format(ycb_dir), recursive=True))
    ev, near = [], []
    for c in class_ids:
        restarted, gts = [], []
        for f in sorted(glob.glob(os.path.join(ycb_all_res_dir(root, names[c - 1]), 'seq*', REINIT_FILE))):
            e = np.load(f)[1:]
            ev.append(e)
            seq_id = int(os.path.basename(os.path.dirname(f))[3:])
            for i in np.nonzero(e == _lib.REINIT_RESTARTED)[0] + 1:
                restarted.append(np.loadtxt(os.path.join(os.path.dirname(f), '%07d.txt' % i)))
                gts.append(np.loadtxt('{}/data_organized/%04d/pose_gt/{}/%06d.txt'.format(ycb_dir, c) % (seq_id, i + 1)))
        if restarted:
            t = lambda a: torch.from_numpy(np.ascontiguousarray(np.stack(a), dtype=np.float64)).to(eng.device)
            pts = torch.from_numpy(np.ascontiguousarray(eval_ycb._read_points(model_files[c - 1]))).to(eng.device)
            near.append(eng.add_adi(pts, t(restarted), t(gts))[1].cpu().numpy() < FIT_LOST_ADDS)
    e = np.concatenate(ev) if ev else np.zeros(0, np.int32)
    near = np.concatenate(near) if near else np.zeros(0, bool)
    count = lambda *codes: int(np.isin(e, codes).sum())
    return dict(tracked=int(len(e)), below=int((e != 0).sum()), attempts=count(2, 3, 4), restarted=count(2), rejected=count(4),
                failed=count(3), restarts_near=float(near.mean()) if len(near) else float('nan'))


def print_reinit_table(rows):
    """--score's table for a run with --reinit_below: one row per variant tree of score_reinit's result."""
    print('re-initialisation: restarts near = the share of restarted poses within %g cm ADD-S of the annotation' % (FIT_LOST_ADDS * 100))
    print('%-16s %8s %8s %8s %9s %8s %8s %14s' % ('variant', 'tracked', 'below', 'attempts', 'restarted', 'rejected', 'failed',
                                                 'restarts near'))
    for label, r in rows.items():
        print('%-16s %8d %8d %8d %9d %8d %8d %14.4f' % (label, r['tracked'], r['below'], r['attempts'], r['restarted'], r['rejected'],
                                                      r['failed'], r['restarts_near']))


def print_fit_table(rows):
    """--score's table for a run with --fit: one row per variant tree of score_fit's result."""
    print('fit check: frames with ADD-S >= %g cm count as lost; inlier fraction = inlier / model pixels' % (FIT_LOST_ADDS * 100))
    print('%-16s %8s %8s %12s %12s %8s' % ('variant', 'frames', 'lost', 'inlier lost', 'inlier kept', 'ROC AUC'))
    for label, r in rows.items():
        print('%-16s %8d %8.4f %12.4f %12.4f %8.4f' % (label, r['frames'], r['lost'], r['inlier_lost'], r['inlier_kept'], r['auc']))


def print_precision_table(ref, rows, sweep='precision sweep', column='mode'):
    """The table --score prints after a sweep's per-mode scores: one row per mode of score_precisions' result (per variant of
    score_iterations' with sweep='iteration sweep', column='variant')."""
    print('%s: AUCs in percent; drift from %s in mm (ADD / ADD-S to its pose of the same track and frame)' % (sweep, ref))
    print('%-8s %9s %9s %11s %11s %11s %11s' % (column, 'ADD', 'ADD-S', 'ADD max', 'ADD mean', 'ADD-S max', 'ADD-S mean'))
    for m, r in rows.items():
        print('%-8s %9.4f %9.4f %11.4g %11.4g %11.4g %11.4g' % (m, r['add'], r['adds'], r['add_max'], r['add_mean'], r['adds_max'],
                                                               r['adds_mean']))


def main(argv=None):
    import argparse
    parser = argparse.ArgumentParser(description='headless se(3)-TrackNet sequence tracking on libse3tn (flags of the reference predict.py:626-641)')
    parser.add_argument('--mode', default='ycbv', help='ycbv (one YCB-Video sequence) / ycbineoat / ycbv_all (every class of --class_ids '
                        'through every YCB-Video test sequence in one pass) / ycbineoat_all (every video under --YCBInEOAT_dir in one '
                        'pass) / ycbv_recover (score refinement from the perturbed starts of the YCB-Video key frames, every class of '
                        '--class_ids in one pass; nothing is written) / ycbv_init (score the starts Engine.init_poses finds from the masks of '
                        'the YCB-Video key frames; no checkpoint) / anything else: every YCB-Video test sequence of the class')
    parser.add_argument('--seq_id', default=None, type=int)
    parser.add_argument('--ycb_dir', default=None)
    parser.add_argument('--YCBInEOAT_dir', default=None)
    parser.add_argument('--train_data_path', required=True, help='dataset_info.yml is read from <train_data_path>/../')
    parser.add_argument('--class_id', default=-1, type=int, help='class id in YCB Video')
    parser.add_argument('--class_ids', default=None, help='ycbv_all: comma-separated class ids, or all')
    parser.add_argument('--model_path', type=str, required=True, help='path to mesh (.ply with normals and vertex colours for the CUDA renderer)')
    parser.add_argument('--ckpt_dir', type=str, default=None, help='required by every mode but ycbv_init')
    parser.add_argument('--mean_std_path', type=str, default=None, help='required by every mode but ycbv_init')
    parser.add_argument('--outdir', type=str, default=None, help='required by every mode but ycbv_recover')
    parser.add_argument('--pair_model_path', default=None, help='ycbv_recover: path template of the mesh the perturbed pairs are '
                        'cut with (default --model_path with .ply -> .obj, as ProducerPurturb picks it)')
    parser.add_argument('--num_sample', type=int, default=10, help='ycbv_recover: perturbations drawn per annotated class and key frame')
    parser.add_argument('--seed', type=int, default=0, help='ycbv_recover: seed of random and np.random before the first draw, and '
                        'of the hypotheses\' draws; ycbv_all / ycbineoat_all: seed of the hypotheses\' draws')
    parser.add_argument('--hypotheses', type=int, default=None, help='ycbv_all / ycbineoat_all / ycbv_recover: track every step from S '
                        'start hypotheses per track (1..32, default 1) and keep the one whose model fits the frame best')
    parser.add_argument('--reinit_frames', type=str, default=None, help='comma-separated %%04d/%%06d frames to re-initialise from PoseCNN')
    parser.add_argument('--init', default='gt', help='gt / posecnn / poserbpf (the reference hard-codes gt); ycbv_all also mask: '
                        'each sequence starts from Engine.init_poses on its first frame\'s depth and seg/ label image; ycbv_all and '
                        'ycbv_init also box: Engine.init_boxes with each class\'s tight box in that label image')
    parser.add_argument('--init_depths', type=int, default=None, help='--init box: depth candidates D along each box\'s ray (1..%d, '
                        'default %d)' % (_engine.Engine.MAX_INIT_DEPTHS, _engine.Engine.INIT_BOX_DEPTHS))
    parser.add_argument('--init_viewpoints', type=int, default=None, help='--init mask / ycbv_init: grid viewpoints V (default %d)'
                        % _engine.Engine.INIT_DEFAULTS['viewpoints'])
    parser.add_argument('--init_inplane', type=int, default=None, help='--init mask / ycbv_init: in-plane angles R (default %d)'
                        % _engine.Engine.INIT_DEFAULTS['inplane'])
    parser.add_argument('--init_keep', type=int, default=None, help='--init mask / ycbv_init: candidates kept K (default %d)'
                        % _engine.Engine.INIT_DEFAULTS['keep'])
    parser.add_argument('--init_icp', type=int, default=None, help='--init mask / ycbv_init: ICP iterations on the kept candidates '
                        '(0: none; default %d)' % _engine.Engine.INIT_DEFAULTS['icp'])
    parser.add_argument('--reinit_below', type=float, default=None, help='ycbv_all: re-initialise a track from its frame\'s seg/ '
                        'label image when its fit check\'s inlier fraction stays below F (0..1, three decimals) for --reinit_after '
                        'frames; the --init_* options set the restart.  Each sequence folder gets reinit.npy, and --score adds its table.  '
                        'Defaults are guesses: choose F with --fit --score')
    parser.add_argument('--reinit_after', type=int, default=None, help='with --reinit_below: the frames in a row below F that make a '
                        'track lost (1..1000, default %d)' % _engine.Engine.REINIT_DEFAULTS['after'])
    parser.add_argument('--max_frames', type=int, default=None)
    parser.add_argument('--score', action='store_true', help='ycbv_all / ycbineoat_all: score the output with eval_ycb / '
                        'eval_ycbineoat and print its lines')
    parser.add_argument('--decode_ahead', type=int, default=4, help='ycbineoat_all: frames decoded ahead of the tracking step')
    parser.add_argument('--video', action='store_true', help='ycbv_all / ycbineoat_all: also write the result videos, each track\'s '
                        'model points drawn over its frames on the device (<class folder>/run/seq<id>.mp4 / <video>.mp4)')
    parser.add_argument('--precision', default=None, help='MODE|all|MODE,MODE,...: the precision mode (default bf16x3).  ycbv_all / '
                        'ycbineoat_all also take a comma-separated list of modes or all: every frame is tracked in each mode, mode m '
                        'written under <outdir>/<m>/, and --score prints each mode\'s scores and a table of their AUCs and drift')
    parser.add_argument('--iterations', default=None, help='K|K1,K2,...: refine every track K times per frame in one tracking step '
                        '(1..8, default 1).  ycbv_all / ycbineoat_all also take a comma-separated list: every frame is tracked with '
                        'each K, K\'s tree written under <outdir>/iter<K>/, and --score adds a table of each variant\'s AUCs and drift '
                        'from K = 1')
    parser.add_argument('--fit', type=int, default=None, help='ycbv_all / ycbineoat_all: check every step\'s fit, tau in mm '
                        '(1..1000): each sequence folder gets fit.npy beside its pose files, and --score adds the fit table')
    parser.add_argument('--icp', type=int, default=None, help='ycbv_all / ycbineoat_all / ycbv_recover: refine every track with M '
                        'iterations of point-to-plane ICP against the depth after the last round (0..16, default 0: off); '
                        'ycbv_recover adds rows icp 1 .. icp M after round K')
    parser.add_argument('--icp_tau', type=int, default=None, help='with --icp: the association gate in mm (1..1000, default %d, a '
                        'starting guess)' % _engine.Engine.ICP_TAU_DEFAULT)
    parser.add_argument('--gpus', type=int, default=None, help='ycbv_all / ycbineoat_all: share the sequences out over N GPUs, '
                        'one process each (default 1); every file is the one a one-GPU run writes')
    args = parser.parse_args(argv)
    cli_reinit(args)
    init = cli_init(args)
    if args.mode == 'ycbv_init':
        return _main_init(args, init)
    missing = [f for f in ('--ckpt_dir', '--mean_std_path') if getattr(args, f[2:]) is None]
    if missing:
        parser.error('the following arguments are required: %s' % ', '.join(missing))
    if args.fit is not None:
        if args.mode not in ('ycbv_all', 'ycbineoat_all'):
            raise SystemExit('--fit needs --mode ycbv_all or ycbineoat_all; --mode %s does not check the fit' % args.mode)
        try:
            step_options(fit=args.fit)
        except ValueError as e:
            raise SystemExit('--fit %d: %s' % (args.fit, e))
    if args.hypotheses is not None:
        if args.hypotheses != 1 and args.mode not in ('ycbv_all', 'ycbineoat_all', 'ycbv_recover'):
            raise SystemExit('--hypotheses %d needs --mode ycbv_all, ycbineoat_all or ycbv_recover; --mode %s tracks one start per '
                             'track' % (args.hypotheses, args.mode))
        try:
            step_options(hypotheses=args.hypotheses)
        except ValueError:
            raise SystemExit('--hypotheses %d: must be in [1, %d]' % (args.hypotheses, _lib.MAX_HYPOTHESES))
    if args.icp is not None or args.icp_tau is not None:
        if args.mode not in ('ycbv_all', 'ycbineoat_all', 'ycbv_recover'):
            raise SystemExit('--icp / --icp_tau need --mode ycbv_all, ycbineoat_all or ycbv_recover; --mode %s does not refine '
                             'with ICP' % args.mode)
        try:
            step_options(hypotheses=args.hypotheses or 1, icp=args.icp, icp_tau=args.icp_tau)
        except ValueError as e:
            raise SystemExit('--icp %s --icp_tau %s: %s' % (args.icp, args.icp_tau, e))
    if args.mode == 'ycbv_recover':
        return _main_recover(args)
    if args.outdir is None:
        parser.error('the following arguments are required: --outdir')
    if args.gpus is not None and args.gpus < 1:
        raise SystemExit('--gpus %d: the number of GPUs is at least 1' % args.gpus)
    if args.gpus is not None and args.gpus > 1 and args.mode not in ('ycbv_all', 'ycbineoat_all'):
        raise SystemExit('--gpus %d needs --mode ycbv_all or ycbineoat_all' % args.gpus)
    precision = cli_precision(args.precision, args.mode)
    iterations = cli_iterations(args.iterations, args.mode)
    if args.mode in ('ycbv_all', 'ycbineoat_all'):
        return _main_one_pass(args, precision, iterations)
    prec_kw = dict({} if precision is None else {'precision': precision}, **({} if iterations is None else {'iterations': iterations}))
    dataset_info, images_mean, images_std = load_run_config(args.train_data_path, args.mean_std_path)
    if args.mode == 'ycbineoat':
        if not args.YCBInEOAT_dir:
            raise SystemExit('--mode ycbineoat needs --YCBInEOAT_dir')
        poses = predictSequenceYcbInEOAT(args.YCBInEOAT_dir, dataset_info, images_mean, images_std, args.ckpt_dir, args.model_path,
                                         args.outdir, max_frames=args.max_frames, **prec_kw)
        print('wrote %d poses to %s' % (len(poses), args.outdir))
        return
    if not args.ycb_dir:
        raise SystemExit('--mode %s needs --ycb_dir' % args.mode)
    if args.mode == 'ycbv':
        if args.seq_id is None:
            raise SystemExit('--mode ycbv needs --seq_id')
        class_id = args.class_id if args.class_id is not None and args.class_id >= 0 else 4      # predict.py:450-452
        reinit = args.reinit_frames.split(',') if args.reinit_frames else None
        poses, auc = predictSequenceYcb(args.ycb_dir, args.seq_id, class_id, dataset_info, images_mean, images_std, args.ckpt_dir,
                                        args.model_path, args.outdir, init=args.init, reinit_frames=reinit, max_frames=args.max_frames,
                                        **prec_kw)
        print('reinit_frames {}, adi_auc {}'.format(reinit or '', auc))
        return
    res = getResultsYcb(args.ycb_dir, args.class_id, dataset_info, images_mean, images_std, args.ckpt_dir, args.model_path, args.outdir,
                        initialize_method=args.init, max_frames=args.max_frames, **prec_kw)
    print('tracked class %d through sequences %s -> %s' % (args.class_id, sorted(res), args.outdir))


def cli_precision(text, mode):
    """--precision of `mode` -> None (not given: the drivers' default, bf16x3), a mode name, or for ycbv_all / ycbineoat_all a
    list of names or 'all' (a sweep).  A name that is no mode, and a list or 'all' with any other mode, are a SystemExit; so is a
    sweep its driver refuses (unknown or repeated modes, an empty list, 'fp16' with ycbv_all)."""
    if text is None:
        return None
    if text != 'all' and ',' not in text:
        if text not in PRECISIONS:
            raise SystemExit('--precision %s: not a precision mode (one of %s)' % (text, ', '.join(PRECISIONS)))
        return text
    if mode not in ('ycbv_all', 'ycbineoat_all', 'ycbv_recover'):
        raise SystemExit('--precision %s: a list of modes or all needs --mode ycbv_all or ycbineoat_all, or ycbv_recover' % text)
    precision = 'all' if text == 'all' else [m.strip() for m in text.split(',')]
    try:
        precision_modes(precision, YCB_ALL_PRECISIONS if mode in ('ycbv_all', 'ycbv_recover') else PRECISIONS)
    except ValueError as e:
        raise SystemExit('--precision %s: %s' % (text, e))
    return precision


def cli_iterations(text, mode):
    """--iterations of `mode` -> None (not given: one round per step), a count, or for ycbv_all / ycbineoat_all a list of counts
    (a sweep).  A count outside [1, 8] or not an integer, and a list with any other mode, are a SystemExit; so is a list its
    driver refuses (repeated counts, an empty entry)."""
    if text is None:
        return None
    try:
        if ',' not in text:
            return _refine_iterations(int(text))
        if mode not in ('ycbv_all', 'ycbineoat_all'):
            raise SystemExit('--iterations %s: a list of counts needs --mode ycbv_all or ycbineoat_all' % text)
        counts = [int(k) for k in text.split(',')]
        refine_counts(counts)
    except ValueError as e:
        raise SystemExit('--iterations %s: %s' % (text, e))
    return counts


def cli_recover(args):
    """--mode ycbv_recover's arguments -> (class ids, class_config, keyword arguments of recoverYcbKeyframes); every refusal
    recover_front makes, a missing argument and an unreadable --class_ids are a SystemExit, before anything is read but the
    CADmodels/ names."""
    if not args.ycb_dir or not args.class_ids:
        raise SystemExit('--mode ycbv_recover needs --ycb_dir and --class_ids')
    if args.gpus is not None and args.gpus != 1:
        raise SystemExit('--gpus %d: %s' % (args.gpus, RECOVER_GPUS_REFUSAL))
    precision = cli_precision(args.precision, args.mode)
    iterations = cli_iterations(args.iterations, args.mode)
    try:
        recover_front(precision or 'bf16x3', iterations or 1)
    except ValueError as e:
        raise SystemExit('--precision / --iterations: %s' % e)
    config = {key: getattr(args, key) for key in YCB_ALL_TEMPLATES}
    if args.pair_model_path:
        config['pair_model_path'] = args.pair_model_path
    for key in ('ckpt_dir', 'mean_std_path'):
        if ',' in config[key]:
            config[key] = config[key].split(',')
    try:
        checkpoint_configs(config)
    except ValueError as e:
        raise SystemExit('--ckpt_dir / --mean_std_path: %s' % e)
    if args.class_ids == 'all':
        class_ids = list(range(1, len(ycb_class_names(args.ycb_dir)) + 1))
    else:
        try:
            class_ids = sorted(set(int(c) for c in args.class_ids.split(',')))
        except ValueError:
            raise SystemExit('--class_ids must be comma-separated integers or all, not %r' % args.class_ids)
    try:
        pair_mesh_base(class_ids, len(checkpoint_configs(config)))
    except ValueError as e:
        raise SystemExit('--class_ids: %s' % e)
    kw = dict(num_sample=args.num_sample, seed=args.seed, precision=precision or 'bf16x3', iterations=iterations or 1,
              max_frames=args.max_frames)
    if getattr(args, 'hypotheses', None) is not None:
        kw['hypotheses'] = args.hypotheses
    for key in ('icp', 'icp_tau'):
        if getattr(args, key, None) is not None:
            kw[key] = getattr(args, key)
    return class_ids, config, kw


def cli_init(args):
    """The start-from-mask options of the command line -> Engine.init_spec's dict (None: the defaults), also left in
    args.init_spec.  --init mask needs --mode ycbv_all; the --init_* options need --init mask or --mode ycbv_init; the other
    modes refuse --init mask and them; --reinit_below (ycbv_all) also takes them, for its restarts; a value init_spec refuses is
    a SystemExit."""
    flags = {'viewpoints': args.init_viewpoints, 'inplane': args.init_inplane, 'keep': args.init_keep, 'icp': args.init_icp}
    given = {k: v for k, v in flags.items() if v is not None}
    depths = getattr(args, 'init_depths', None)
    if args.init == 'box' and args.mode not in ('ycbv_all', 'ycbv_init'):
        raise SystemExit('--init box needs --mode ycbv_all or ycbv_init, not --mode %s' % args.mode)
    if depths is not None and args.init != 'box':
        raise SystemExit('--init_depths needs --init box')
    if args.init == 'box' and args.reinit_below is not None:
        raise SystemExit('--init box with --reinit_below: restarts inside the one-pass driver come from masks only')
    if depths is not None:
        try:
            _engine.Engine.depths_spec(depths)
        except ValueError as e:
            raise SystemExit('--init_depths: %s' % e)
    if args.init == 'mask' and args.mode != 'ycbv_all':
        raise SystemExit('--init mask needs --mode ycbv_all; --mode %s does not start from masks (--mode ycbv_init scores the '
                         'starts on the key frames)' % args.mode)
    if given and args.mode != 'ycbv_init' and args.init not in ('mask', 'box') and args.reinit_below is None:
        raise SystemExit('%s need --init mask (with --mode ycbv_all), --reinit_below or --mode ycbv_init'
                         % ', '.join('--init_' + k for k in given))
    spec = given or None
    try:
        _engine.Engine.init_spec(spec)
    except ValueError as e:
        raise SystemExit('--init_*: %s' % e)
    args.init_spec = spec
    return spec


def cli_reinit(args):
    """The re-initialisation options of the command line, checked before anything else: --reinit_below needs --mode ycbv_all
    (the other modes' layouts have no per-frame masks, or they do not track a sequence), --reinit_after needs --reinit_below,
    and values reinit_options refuses are a SystemExit."""
    if args.reinit_after is not None and args.reinit_below is None:
        raise SystemExit('--reinit_after needs --reinit_below')
    if args.reinit_below is None:
        return
    if args.mode != 'ycbv_all':
        raise SystemExit('--reinit_below needs --mode ycbv_all; --mode %s does not re-initialise tracks from per-frame masks' % args.mode)
    try:
        reinit_options({'below': args.reinit_below, 'after': _engine.Engine.REINIT_DEFAULTS['after'] if args.reinit_after is None
                        else args.reinit_after})
    except ValueError as e:
        raise SystemExit('--reinit_below / --reinit_after: %s' % e)


def _main_init(args, init):
    """--mode ycbv_init: initYcbKeyframes, then its tables (print_init_tables).  Needs --ycb_dir, --class_ids, --train_data_path
    and --model_path; takes no checkpoint, and refuses the tracking options."""
    if not args.ycb_dir or not args.class_ids:
        raise SystemExit('--mode ycbv_init needs --ycb_dir and --class_ids')
    tracking = [f for f, v in (('--outdir', args.outdir), ('--precision', args.precision), ('--iterations', args.iterations),
                               ('--fit', args.fit), ('--hypotheses', args.hypotheses), ('--icp', args.icp), ('--icp_tau', args.icp_tau),
                               ('--gpus', args.gpus), ('--video', args.video or None), ('--score', args.score or None)) if v is not None]
    if tracking:
        raise SystemExit('%s: --mode ycbv_init scores starts, it does not track (--init_icp sets its ICP)' % ', '.join(tracking))
    if args.class_ids == 'all':
        class_ids = list(range(1, len(ycb_class_names(args.ycb_dir)) + 1))
    else:
        try:
            class_ids = sorted(set(int(c) for c in args.class_ids.split(',')))
        except ValueError:
            raise SystemExit('--class_ids must be comma-separated integers or all, not %r' % args.class_ids)
    config = dict(train_data_path=args.train_data_path, model_path=args.model_path)
    try:
        box = dict(box=True, depths=getattr(args, 'init_depths', None)) if args.init == 'box' else {}
        res = initYcbKeyframes(args.ycb_dir, class_ids, config, init=init, max_frames=args.max_frames, **box)
    except ValueError as e:
        raise SystemExit(str(e))
    names = ycb_class_names(args.ycb_dir)
    spec = _engine.Engine.init_spec(init)
    print('ycbv_init: V %d, R %d, K %d, ICP %d, %s%s' % (spec.viewpoints, spec.inplane, spec.keep, spec.icp.contents.iterations if spec.icp else 0,
                                                         torch.cuda.get_device_name(torch.cuda.current_device()),
                                                         ', boxes from the labels, D %d' % (getattr(args, 'init_depths', None) or _engine.Engine.INIT_BOX_DEPTHS)
                                                         if args.init == 'box' else ''))
    print_init_tables(res, {c: names[c - 1] for c in class_ids})
    return res


def _main_recover(args):
    """--mode ycbv_recover: recoverYcbKeyframes, then its tables (print_recover_tables)."""
    class_ids, config, kw = cli_recover(args)
    try:
        res = recoverYcbKeyframes(args.ycb_dir, class_ids, config, **kw)
    except ValueError as e:
        raise SystemExit(str(e))
    names = ycb_class_names(args.ycb_dir)
    print('ycbv_recover: num_sample %d, seed %d, K = %d, %s' % (kw['num_sample'], kw['seed'], kw['iterations'],
                                                               torch.cuda.get_device_name(torch.cuda.current_device())))
    print_recover_tables(res, {c: names[c - 1] for c in class_ids})
    return res


def _main_one_pass(args, precision=None, iterations=None):
    """--mode ycbv_all / ycbineoat_all: --train_data_path, --mean_std_path, --ckpt_dir and --model_path are the per-class /
    per-object path templates.  --video, --precision, --gpus and --iterations are passed to the driver only when given, so a run
    without them makes the same call."""
    import argparse
    ycbv = args.mode == 'ycbv_all'
    if ycbv and (not args.ycb_dir or not args.class_ids):
        raise SystemExit('--mode ycbv_all needs --ycb_dir and --class_ids')
    if not ycbv and not args.YCBInEOAT_dir:
        raise SystemExit('--mode ycbineoat_all needs --YCBInEOAT_dir')
    if not ycbv and args.score and not args.ycb_dir:
        raise SystemExit('--score needs --ycb_dir (the model points eval_ycbineoat reads)')
    config = {key: getattr(args, key) for key in YCB_ALL_TEMPLATES}
    for key in ('ckpt_dir', 'mean_std_path'):                   # template lists: one pass over several checkpoints
        if ',' in config[key]:
            config[key] = config[key].split(',')
    try:
        ckpts = len(checkpoint_configs(config))
    except ValueError as e:
        raise SystemExit('--%s: %s' % ('ckpt_dir / --mean_std_path', e))
    kw = {key: v for key, v in (('video', args.video or None), ('precision', precision), ('gpus', args.gpus),
                                ('iterations', iterations), ('fit', getattr(args, 'fit', None)),
                                ('hypotheses', getattr(args, 'hypotheses', None)), ('icp', getattr(args, 'icp', None)),
                                ('icp_tau', getattr(args, 'icp_tau', None))) if v is not None}
    if 'hypotheses' in kw:
        kw['seed'] = args.seed
    if ycbv:
        if args.class_ids == 'all':
            class_ids = list(range(1, len(ycb_class_names(args.ycb_dir)) + 1))
        else:
            try:
                class_ids = sorted(set(int(c) for c in args.class_ids.split(',')))
            except ValueError:
                raise SystemExit('--class_ids must be comma-separated integers or all, not %r' % args.class_ids)
        if args.init in ('mask', 'box'):
            kw['init'] = getattr(args, 'init_spec', None)
        if args.init == 'box' and getattr(args, 'init_depths', None) is not None:
            kw['depths'] = args.init_depths
        if args.reinit_below is not None:
            kw['reinit'] = dict(below=args.reinit_below, init=getattr(args, 'init_spec', None),
                                **({} if args.reinit_after is None else {'after': args.reinit_after}))
        res = getResultsYcbAll(args.ycb_dir, class_ids, config, args.outdir, initialize_method=args.init, max_frames=args.max_frames, **kw)
        outdir, eoat = args.outdir, {}
    else:
        res = getResultsYcbInEOAT(args.YCBInEOAT_dir, config, args.outdir, max_frames=args.max_frames, decode_ahead=args.decode_ahead,
                                  ycb_dir=args.ycb_dir, **kw)
        outdir, eoat = args.outdir.rstrip('/'), dict(YCBInEOAT_dir=args.YCBInEOAT_dir)
    sweep = precision is not None and precision_modes(precision, PRECISIONS)[1]
    one = res[0] if ckpts > 1 else res
    one = next(iter(one.values()), {}) if isinstance(iterations, list) else one      # the printout lists the first variant's run
    one = next(iter(one.values()), {}) if sweep else one
    if ycbv:
        for c in sorted(one):
            print('tracked class %d through sequences %s' % (c, sorted(one[c])))
    else:
        for v in one:
            print('tracked %s: %d frames' % (v, len(one[v])))
    print('-> %s' % args.outdir)
    if args.score and ckpts > 1:
        ref, rows = score_checkpoints(res, outdir, args.ycb_dir, config, precision=precision or 'bf16x3',
                                      iterations=iterations or 1, **eoat)
        print_precision_table(ref, rows, sweep='checkpoint sweep', column='variant')
        print_best_checkpoints(rows, config['ckpt_dir'])
    elif args.score and isinstance(iterations, list):
        print_precision_table(*score_iterations(res, outdir, args.ycb_dir, config, precision=precision or 'bf16x3', **eoat),
                              sweep='iteration sweep', column='variant')
    elif args.score and sweep:
        print_precision_table(*score_precisions(res, outdir, args.ycb_dir, config, **eoat))
    elif args.score and ycbv:
        _score_ycb_tree(args.ycb_dir, outdir, class_ids)
    elif args.score:
        from . import eval_ycbineoat
        eval_ycbineoat.eval_all(argparse.Namespace(YCBInEOAT_dir=args.YCBInEOAT_dir, ycb_dir=args.ycb_dir, res_dir=outdir + '/'))
    if args.score and getattr(args, 'fit', None):
        modes, msweep = precision_modes(precision or 'bf16x3', YCB_ALL_PRECISIONS if ycbv else PRECISIONS)
        counts, ksweep = refine_counts(iterations or 1)
        trees = [v[-1] for v in _sweep_variants(outdir, modes, msweep, counts, ksweep, ckpts)]
        print_fit_table({os.path.relpath(tr, outdir): score_fit(tr, args.ycb_dir, args.YCBInEOAT_dir if not ycbv else None,
                                                                 class_ids if ycbv else None) for tr in trees})
    if args.score and ycbv and args.reinit_below is not None:
        modes, msweep = precision_modes(precision or 'bf16x3', YCB_ALL_PRECISIONS)
        counts, ksweep = refine_counts(iterations or 1)
        trees = [v[-1] for v in _sweep_variants(outdir, modes, msweep, counts, ksweep, ckpts)]
        print_reinit_table({os.path.relpath(tr, outdir): score_reinit(tr, args.ycb_dir, class_ids) for tr in trees})
    return res


if __name__ == '__main__':
    main()
