"""Engine: one libse3tn context bound to one CUDA device, driven with torch tensors.

PyTorch is used here for device-memory ownership, the current stream and (in dist.py)
torch.distributed -- all arithmetic happens inside libse3tn.so.  There is no CPU or eager
fallback: without a CUDA device and the built library every call raises.
"""
import ctypes as C
import decimal
import math
import numpy as np
import torch

from . import _lib
from .weights import pack_state_dict

PREC = {'tf32': _lib.PREC_TF32, 'fp32': _lib.PREC_FP32, 'bf16x3': _lib.PREC_BF16X3, 'bf16': _lib.PREC_BF16, 'fp8': _lib.PREC_FP8,
        'fp16': _lib.PREC_FP16}
IMAGE_SIZE = 176
LABEL_ORDER = {'under': _lib.LABEL_UNDER_POINTS, 'over': _lib.LABEL_OVER_POINTS}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _hptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else C.c_void_p(0)


def _track_arrays(ptr, **fields):
    """An se3tn_track_arrays by reference: the given CUDA tensors (ptr=_ptr) or numpy arrays (ptr=_hptr); None and absent fields
    are NULL."""
    return C.byref(_lib.TrackArrays(**{k: ptr(v).value for k, v in fields.items()}))


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def check_weight_sets_fit(n_sets, device=None, what='weight sets'):
    """A ValueError, with the numbers, unless n_sets weight sets (se3tn_weight_set_bytes each: every storage format a set is
    kept in) fit in the free memory of CUDA device `device` (default: the current one).  Called before any set is loaded."""
    each = int(_lib.load().se3tn_weight_set_bytes())
    dev = torch.cuda.current_device() if device is None else int(device)
    free = int(torch.cuda.mem_get_info(dev)[0])
    if n_sets * each > free:
        raise ValueError('%d %s need %.2f GB of device memory (%.1f MB each, in every storage format), but cuda:%d has %.2f GB free'
                         % (n_sets, what, n_sets * each / 1e9, each / 1e6, dev, free / 1e9))
    return each


class Engine:
    def __init__(self, max_batch=64, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError('se3tn Engine needs a CUDA device (sm_90a); there is no CPU fallback')
        self.lib = _lib.load()
        self.device = torch.device('cuda', torch.cuda.current_device() if device is None else
                                   (device.index if isinstance(device, torch.device) else int(device)))
        self.max_batch = int(max_batch)
        nbytes = self.lib.se3tn_workspace_bytes(self.max_batch)
        # caller-owned workspace: a torch allocation, so torch's allocator accounts for it
        self._workspace = torch.empty(nbytes + 1024, dtype=torch.uint8, device=self.device)
        base = self._workspace.data_ptr()
        aligned = (base + 1023) // 1024 * 1024
        ctx = C.c_void_p()
        with torch.cuda.device(self.device):
            rc = self.lib.se3tn_create(self.device.index, self.max_batch, C.c_void_p(aligned), C.byref(ctx))
        _lib.check(rc, None)
        self._ctx = ctx
        self._weight_ids = set()
        self._stats = {}                  # weight id -> the (dtype, mean, std) bytes last set on the context

    def close(self):
        if getattr(self, '_ctx', None):
            torch.cuda.synchronize(self.device)
            self.lib.se3tn_destroy(self._ctx)
            self._ctx = None
            self._fit_rows = None
            self._icp_rows = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ parameters
    def load_state_dict(self, state_dict, weight_id=0):
        blob = pack_state_dict(state_dict)
        _lib.check(self.lib.se3tn_load_weights(self._ctx, int(weight_id), blob.ctypes.data_as(C.c_void_p), blob.size), self._ctx)
        self._weight_ids.add(int(weight_id))

    def set_stats(self, mean, std, weight_id=0):
        """A weight set's channel statistics.  New values drop the context's captured steps (se3tn_set_stats), so the values a
        set already has are not set again: a validation pass or a Tracker that restates them keeps every step's CUDA graph."""
        mean = np.ascontiguousarray(mean); std = np.ascontiguousarray(std)
        if mean.shape != (8,) or std.shape != (8,):
            raise ValueError('mean/std must be 8-vectors (A channels then B channels)')
        f64 = (mean.dtype == np.float64) or (std.dtype == np.float64)
        dt = np.float64 if f64 else np.float32
        mean = mean.astype(dt); std = std.astype(dt)
        key = (bool(f64), mean.tobytes(), std.tobytes())
        if self._stats.get(int(weight_id)) == key:
            return
        _lib.check(self.lib.se3tn_set_stats(self._ctx, int(weight_id), mean.ctypes.data_as(C.c_void_p),
                                            std.ctypes.data_as(C.c_void_p), int(f64)), self._ctx)
        self._stats[int(weight_id)] = key

    def calibrate_fp8(self, A, B, weight_id=0):
        """The 'fp8' mode's activation scales of a weight set from normalised pairs A, B (float32 (n,4,176,176) CUDA tensors,
        n <= max_batch): the set's bf16x3 forward on them, max|x| of every e4m3 tensor, s = 2^ceil(log2(max|x| * H / 448)).
        -> the scales (float32 (8,), the se3tn.h order).  Synchronises the device."""
        self._check_img(A); self._check_img(B)
        n = A.shape[0]
        if B.shape[0] != n:
            raise ValueError('A and B batch sizes differ')
        _lib.check(self.lib.se3tn_calibrate_fp8(self._ctx, int(weight_id), _ptr(A), _ptr(B), n, _stream(self.device)), self._ctx)
        return self.fp8_scales(weight_id)

    def calibrate_fp8_missing(self, A, B, weight_ids=None):
        """The one place where the 'fp8' mode picks calibration pairs from data (Tracker, problems and the one-pass drivers
        come through here): every weight set among the pairs' ids (weight_ids: host int array, None = all set 0) that has
        no activation scales yet is calibrated on its own pairs of the normalised A, B (CUDA tensors).  Sets that have
        scales keep them.  -> the ids calibrated."""
        ids = np.zeros(A.shape[0], np.int32) if weight_ids is None else np.asarray(weight_ids, dtype=np.int32)
        done = []
        for w in sorted(set(ids.tolist())):
            if self.fp8_scales(w) is not None:
                continue
            idx = torch.from_numpy(np.flatnonzero(ids == w)[:self.max_batch]).to(self.device)
            self.calibrate_fp8(A.index_select(0, idx), B.index_select(0, idx), weight_id=w)
            done.append(w)
        return done

    def calibrate_fp8_tracks(self, frame_rgb, frame_depth, K, poses, object_width, rgbA=None, depthA=None, weight_ids=None,
                             fill_depth=None, render=None):
        """calibrate_fp8_missing on the pairs a tracking step of these tracks would form (all CUDA tensors, as track_batch
        takes them): input A as given, or drawn by the rasteriser when render = dict(mode, image_hw, mesh_ids); B cropped
        from the frame (hole-filled first with fill_depth) at the previous pose.  Nothing runs when every set has scales."""
        n = poses.shape[0]
        ids = np.zeros(n, np.int32) if weight_ids is None else np.asarray(weight_ids, dtype=np.int32)
        if all(self.fp8_scales(w) is not None for w in set(ids.tolist())):
            return []
        wd = torch.from_numpy(np.ascontiguousarray(ids)).to(self.device)
        if rgbA is None or depthA is None:
            rgbA, depthA = self.render(K, poses, object_width, mesh_ids=render['mesh_ids'], mode=render['mode'],
                                       image_hw=render['image_hw'])
        on, max_depth, extrapolate, blur = self.depth_fill_spec(fill_depth)
        if on:
            frame_depth = self.fill_depth(frame_depth, max_depth=max_depth, extrapolate=bool(extrapolate),
                                          blur_type='gaussian' if blur else 'bilateral')
        A, B, _, _ = self.preprocess(frame_rgb, frame_depth, K, poses, object_width, rgbA, depthA, weight_ids=wd, want_tensors=True)
        return self.calibrate_fp8_missing(A, B, ids)

    def calibrate_fp8_pairs(self, rgbA, depthA, rgbB, depthB, A_in_cam, weight_ids=None):
        """calibrate_fp8_missing on validation pairs as eval_pairs takes them (CUDA tensors)."""
        n = A_in_cam.shape[0]
        ids = np.zeros(n, np.int32) if weight_ids is None else np.asarray(weight_ids, dtype=np.int32)
        if all(self.fp8_scales(w) is not None for w in set(ids.tolist())):
            return []
        wd = torch.from_numpy(np.ascontiguousarray(ids)).to(self.device)
        A, B = self.normalize(rgbA, depthA, rgbB, depthB, A_in_cam, weight_ids=wd, want_tensors=True)
        return self.calibrate_fp8_missing(A, B, ids)

    def fp8_scales(self, weight_id=0):
        """The 'fp8' activation scales of a weight set (float32 (8,)), or None when it has none."""
        out = np.zeros(_lib.FP8_SCALES, dtype=np.float32)
        rc = self.lib.se3tn_get_fp8_scales(self._ctx, int(weight_id), out.ctypes.data_as(C.c_void_p), out.size)
        if rc == _lib.ERR_STATE:
            return None
        _lib.check(rc, self._ctx)
        return out

    def set_fp8_scales(self, scales, weight_id=0):
        """Saved 'fp8' activation scales (8 powers of two, e.g. from fp8_scales) for a weight set."""
        s = np.ascontiguousarray(scales, dtype=np.float32)
        if s.shape != (_lib.FP8_SCALES,):
            raise ValueError('fp8 scales must be a %d-vector' % _lib.FP8_SCALES)
        _lib.check(self.lib.se3tn_set_fp8_scales(self._ctx, int(weight_id), s.ctypes.data_as(C.c_void_p), s.size), self._ctx)

    # ------------------------------------------------------------------ hot path
    def forward(self, A, B, weight_id=0, precision='bf16x3', want_feature=False):
        """Se3TrackNet.forward on float32 (n,4,176,176) CUDA tensors -> (trans, rot, feature|None)."""
        self._check_img(A); self._check_img(B)
        n = A.shape[0]
        if B.shape[0] != n:
            raise ValueError('A and B batch sizes differ')
        trans = torch.empty(n, 3, dtype=torch.float32, device=self.device)
        rot = torch.empty(n, 3, dtype=torch.float32, device=self.device)
        feat = torch.empty(n, 256, 22, 22, dtype=torch.float32, device=self.device) if want_feature else None
        for i0 in range(0, n, self.max_batch):
            i1 = min(n, i0 + self.max_batch)
            _lib.check(self.lib.se3tn_forward(self._ctx, int(weight_id), _ptr(A[i0:i1]), _ptr(B[i0:i1]), i1 - i0,
                                              _ptr(trans[i0:i1]), _ptr(rot[i0:i1]),
                                              _ptr(feat[i0:i1]) if feat is not None else C.c_void_p(0),
                                              PREC[precision], _stream(self.device)), self._ctx)
        return trans, rot, feat

    def preprocess(self, frame_rgb, frame_depth, K, poses, object_width, rgbA, depthA, weight_ids=None,
                   precision='bf16x3', want_tensors=False, want_crops=False):
        n = poses.shape[0]
        self._check_frame('preprocess', frame_rgb, frame_depth, poses, object_width, (rgbA, depthA), n)
        H, W = frame_depth.shape
        Kh = self._k4(K)
        outA = outB = crop_rgb = crop_depth = None
        if want_tensors:
            outA = torch.empty(n, 4, IMAGE_SIZE, IMAGE_SIZE, dtype=torch.float32, device=self.device)
            outB = torch.empty_like(outA)
        if want_crops:
            crop_rgb = torch.empty(n, IMAGE_SIZE, IMAGE_SIZE, 3, dtype=torch.uint8, device=self.device)
            crop_depth = torch.empty(n, IMAGE_SIZE, IMAGE_SIZE, dtype=torch.uint16, device=self.device)
        _lib.check(self.lib.se3tn_preprocess(self._ctx, _ptr(frame_rgb), _ptr(frame_depth), H, W,
                                             Kh.ctypes.data_as(C.c_void_p), _ptr(poses), _ptr(object_width),
                                             _ptr(rgbA), _ptr(depthA), _ptr(weight_ids), n, PREC[precision],
                                             _ptr(outA), _ptr(outB), _ptr(crop_rgb), _ptr(crop_depth),
                                             _stream(self.device)), self._ctx)
        return outA, outB, crop_rgb, crop_depth

    def normalize(self, rgbA, depthA, rgbB, depthB, poses, weight_ids=None, precision='bf16x3', want_tensors=True):
        """processData's post-transforms on existing 176x176 crops (all CUDA tensors)."""
        n = poses.shape[0]
        outA = outB = None
        if want_tensors:
            outA = torch.empty(n, 4, IMAGE_SIZE, IMAGE_SIZE, dtype=torch.float32, device=self.device)
            outB = torch.empty_like(outA)
        _lib.check(self.lib.se3tn_normalize(self._ctx, _ptr(rgbA), _ptr(depthA), _ptr(rgbB), _ptr(depthB), _ptr(poses),
                                            _ptr(weight_ids), n, PREC[precision], _ptr(outA), _ptr(outB),
                                            _stream(self.device)), self._ctx)
        return outA, outB

    def compute_bbox(self, poses, K, widths, scale=(1000., 1000., 1000.)):
        n = poses.shape[0]
        out = torch.empty(n, 4, 2, dtype=torch.int32, device=self.device)
        Kh = self._k4(K); sc = np.ascontiguousarray(scale, dtype=np.float64)
        _lib.check(self.lib.se3tn_compute_bbox(self._ctx, _ptr(poses), Kh.ctypes.data_as(C.c_void_p), _ptr(widths),
                                               sc.ctypes.data_as(C.c_void_p), _ptr(out), n, _stream(self.device)), self._ctx)
        return out

    def crop_bbox(self, frame_rgb, frame_depth, bbox, out_hw=(IMAGE_SIZE, IMAGE_SIZE)):
        n = bbox.shape[0]
        H, W = frame_depth.shape
        crop_rgb = torch.empty(n, out_hw[0], out_hw[1], 3, dtype=torch.uint8, device=self.device)
        crop_depth = torch.empty(n, out_hw[0], out_hw[1], dtype=torch.uint16, device=self.device)
        _lib.check(self.lib.se3tn_crop_bbox(self._ctx, _ptr(frame_rgb), _ptr(frame_depth), H, W, _ptr(bbox), n,
                                            int(out_hw[0]), int(out_hw[1]), _ptr(crop_rgb), _ptr(crop_depth),
                                            _stream(self.device)), self._ctx)
        return crop_rgb, crop_depth

    def forward_preprocessed(self, n, weight_id=0, first=0, precision='bf16x3', want_feature=False):
        trans = torch.empty(n, 3, dtype=torch.float32, device=self.device)
        rot = torch.empty(n, 3, dtype=torch.float32, device=self.device)
        feat = torch.empty(n, 256, 22, 22, dtype=torch.float32, device=self.device) if want_feature else None
        _lib.check(self.lib.se3tn_forward_preprocessed(self._ctx, int(weight_id), int(first), n, _ptr(trans), _ptr(rot),
                                                       _ptr(feat), PREC[precision], _stream(self.device)), self._ctx)
        return trans, rot, feat

    def pose_update(self, poses, trans, rot, trans_normalizer, rot_normalizer, out=None):
        n = poses.shape[0]
        if poses.dtype != torch.float64 or not poses.is_contiguous() or poses.shape[1:] != (4, 4):
            raise ValueError('poses must be a contiguous float64 (n,4,4) CUDA tensor')
        out = torch.empty_like(poses) if out is None else out
        _lib.check(self.lib.se3tn_pose_update(self._ctx, _ptr(poses), _ptr(trans), _ptr(rot), float(trans_normalizer),
                                              float(rot_normalizer), _ptr(out), n, _stream(self.device)), self._ctx)
        return out

    def so3_log(self, poses_a, poses_b, trans_normalizer, rot_normalizer):
        n = poses_a.shape[0]
        tl = torch.empty(n, 3, dtype=torch.float64, device=self.device)
        rl = torch.empty(n, 3, dtype=torch.float64, device=self.device)
        _lib.check(self.lib.se3tn_so3_log(self._ctx, _ptr(poses_a), _ptr(poses_b), float(trans_normalizer),
                                          float(rot_normalizer), _ptr(tl), _ptr(rl), n, _stream(self.device)), self._ctx)
        return tl, rl

    def track_batch(self, frame_rgb, frame_depth, K, poses, object_width, rgbA, depthA,
                    trans_normalizer, rot_normalizer, weight_ids_host=None, weight_ids_dev=None,
                    precision='bf16x3', out_poses=None, out_trans=None, out_rot=None, fill_depth=None):
        """n independent tracks of one frame: K0 -> conv stack -> K6, all enqueued on the current stream.  fill_depth: the
        observed depth is hole-filled inside the step first (depth_fill_spec); frame_depth itself is never written."""
        return self._track('track_batch', frame_rgb, frame_depth, K, poses, object_width, (rgbA, depthA), None, trans_normalizer,
                           rot_normalizer, weight_ids_host, weight_ids_dev, precision, out_poses, out_trans, out_rot, fill_depth, 1)[:3]

    def track_render(self, frame_rgb, frame_depth, K, poses, object_width, trans_normalizer, rot_normalizer,
                     weight_ids_host=None, weight_ids_dev=None, precision='bf16x3', mode='vispy', image_hw=None,
                     out_poses=None, out_trans=None, out_rot=None, fill_depth=None, iterations=1, out_rounds=None,
                     fit=None, out_fit=None, icp=None, out_icp_poses=None, out_icp=None):
        """track_batch with input A rendered inside the step (se3tn_track_render): the models at `poses` are drawn, then
        K0 -> conv stack -> K6, all enqueued on the current stream.  Track i draws mesh weight_ids[i] (mesh 0 without ids).
        mode / image_hw as in render(), fill_depth as in track_batch.  CUDA tensors in and out; nothing is synchronised.
        out_poses may be poses itself: the tracks' poses are then updated in place (include/se3tn.h).  iterations: k rounds
        of render -> network -> pose update on this frame in the one step, exactly what k chained calls with iterations=1
        compute (se3tn_track_opts.iterations, 1..8); out_trans / out_rot hold the last round's outputs.  out_rounds: a float64
        CUDA tensor (k, n, 4, 4) that receives every round's poses from the same step (se3tn_track_arrays.round_poses): entry
        r - 1 is what a call with iterations=r returns.  The step with it is a CUDA graph of its own.  fit: tau in mm (fit_spec)
        turns on the fit check of the step (se3tn_track_opts.fit_tau_mm): every track's model is drawn at its new pose and
        compared with the observed depth, and the call returns a fourth value, out_fit: an int32 CUDA tensor (n, 6) of the rows
        (model, observed, inlier, front, behind, residual), allocated when None and filled on the current stream.  icp (icp_spec):
        M iterations of point-to-plane ICP against the observed depth after the last round and before the fit check
        (se3tn_track_opts.icp); the call then also returns the last iteration's stats, a float64 CUDA tensor (n, 4) of inliers,
        rms_mm, step_mm, step_deg, after the fit rows when the fit is on (out_icp, allocated when None; the step itself writes an
        Engine-owned block, so its graph is replayed frame after frame).  out_icp_poses: a float64 CUDA tensor (M, n, 4, 4) that
        receives the poses after every ICP iteration."""
        P, tr, ro, rows, stats, _ = self._track(
            'track_render', frame_rgb, frame_depth, K, poses, object_width, (), self._render_mode(mode, image_hw), trans_normalizer,
            rot_normalizer, weight_ids_host, weight_ids_dev, precision, out_poses, out_trans, out_rot, fill_depth, iterations, fit,
            icp=icp, out_rounds=out_rounds, out_fit=out_fit, out_icp_poses=out_icp_poses, out_icp=out_icp)
        return (P, tr, ro) + tuple(x for x in (rows, stats) if x is not None)

    def _track(self, fn, frame_rgb, frame_depth, K, poses, object_width, A, render, trans_normalizer, rot_normalizer,
               weight_ids_host, weight_ids_dev, precision, out_poses, out_trans, out_rot, fill_depth, iterations, fit=None,
               icp=None, hyp=None, draw_keys=None, out_rounds=None, out_fit=None, out_icp_poses=None, out_icp=None, out_choice=None,
               out_hyp_poses=None):
        """The device route of every tracking method, one C call: track_batch (A = (rgbA, depthA), render None), track_render
        and track_hypotheses (A = (), render = _render_mode's triple; hyp: hypothesis_spec's options).  -> (poses, trans, rot,
        fit rows, ICP stats, choice), each of the last three None when the step has none."""
        n = poses.shape[0]
        iterations = self.refine_iterations(iterations)
        tau = self.fit_spec(fit)
        icp = self.icp_spec(icp)
        if icp is None and out_icp_poses is not None:
            raise ValueError('%s: out_icp_poses needs icp' % fn)
        self._check_frame(fn, frame_rgb, frame_depth, poses, object_width, A, n)
        S = 1 if hyp is None else hyp.hypotheses
        if n * S > self.max_batch:
            raise ValueError('n x hypotheses = %d exceeds max_batch=%d' % (n * S, self.max_batch))
        wh = self._host_ids(fn, weight_ids_host, n)
        fill = self.depth_fill_spec(fill_depth)
        Kh = self._k4(K)
        new = lambda shape, dt, t: torch.empty(*shape, dtype=dt, device=self.device) if t is None else t
        out_poses = torch.empty_like(poses) if out_poses is None else out_poses
        out_trans, out_rot = new((n, 3), torch.float32, out_trans), new((n, 3), torch.float32, out_rot)
        if wh is not None and weight_ids_dev is None:
            weight_ids_dev = torch.from_numpy(wh).to(self.device)
        out_fit = new((n, _lib.FIT_COLS), torch.int32, out_fit) if tau or hyp is not None else None
        out_choice = new((n,), torch.int32, out_choice) if hyp is not None else None
        out_icp = new((n, _lib.ICP_COLS), torch.float64, out_icp) if icp is not None else None
        if icp is not None and getattr(self, '_icp_rows', None) is None:
            self._icp_rows = torch.empty(self.max_batch, _lib.ICP_COLS, dtype=torch.float64, device=self.device)
        for name, t, dt, shape in (('draw_keys', draw_keys, torch.int64, (n,)),
                                   ('out_rounds', out_rounds, torch.float64, (iterations, n) + (() if hyp is None else (S,)) + (4, 4)),
                                   ('out_fit', out_fit, torch.int32, (n, _lib.FIT_COLS)), ('out_choice', out_choice, torch.int32, (n,)),
                                   ('out_hyp_poses', out_hyp_poses, torch.float64, (n, S, 4, 4)),
                                   ('out_icp', out_icp, torch.float64, (n, _lib.ICP_COLS)),
                                   ('out_icp_poses', out_icp_poses, torch.float64, (0 if icp is None else icp.iterations, n, 4, 4))):
            if t is not None:
                self._check_dev(name, t, dt, shape)
        H, W = frame_depth.shape
        head = (self._ctx, _ptr(frame_rgb), _ptr(frame_depth), H, W, _hptr(Kh), _ptr(poses), _ptr(object_width))
        tail = (_hptr(wh), _ptr(weight_ids_dev), n, float(trans_normalizer), float(rot_normalizer), PREC[precision],
                _ptr(out_trans), _ptr(out_rot), _ptr(out_poses), self._track_opts(fill, iterations, tau, icp, hyp))
        if render is None:
            rc = self.lib.se3tn_track_batch(*head, *map(_ptr, A), *tail, _stream(self.device))
        else:                                            # without hypotheses the step's fit rows stay in the context's block
            arrays = _track_arrays(_ptr, draw_keys=draw_keys, round_poses=out_rounds, hyp_poses=out_hyp_poses,
                                   icp_poses=out_icp_poses, out_fit=out_fit if hyp is not None else None, out_choice=out_choice,
                                   out_icp=self._icp_rows if icp is not None else None)
            rc = self.lib.se3tn_track_render(*head, *render, *tail, arrays, _stream(self.device))
        _lib.check(rc, self._ctx)
        if tau and hyp is None:
            out_fit.copy_(self._fit_rows_view()[:n])     # the next step overwrites the context's rows
        if icp is not None:
            out_icp.copy_(self._icp_rows[:n])            # the next ICP step overwrites the Engine's rows
        return out_poses, out_trans, out_rot, out_fit, out_icp, out_choice

    def track_host(self, frame_rgb, frame_depth, K, poses, object_width, rgbA, depthA, trans_normalizer, rot_normalizer,
                   weight_ids=None, precision='bf16x3', want_residuals=False, fill_depth=None):
        """The reference's calling pattern as one library call: numpy arrays in, numpy poses out, synchronous (se3tn_track_host).
        frame_rgb uint8 (H,W,3), frame_depth uint16 (H,W), poses float64 (n,4,4), object_width float64 (n), rgbA uint8
        (n,176,176,3), depthA uint16 (n,176,176), weight_ids int32 (n) or None -- all C-contiguous.  fill_depth as in
        track_batch: a live sensor's raw depth frame goes in as it is (the whole frame is uploaded then)."""
        out, tr, ro, *_ = self._track_host('track_host', frame_rgb, frame_depth, K, poses, object_width, (rgbA, depthA), None,
                                           trans_normalizer, rot_normalizer, weight_ids, precision, want_residuals, fill_depth, 1)
        return (out, tr, ro) if want_residuals else out

    def track_render_host(self, frame_rgb, frame_depth, K, poses, object_width, trans_normalizer, rot_normalizer,
                          weight_ids=None, precision='bf16x3', mode='vispy', image_hw=None, want_residuals=False, fill_depth=None,
                          iterations=1, fit=None, icp=None):
        """track_host with input A rendered on the device inside the step (se3tn_track_render_host): the previous poses and
        the frame are all it takes.  Arguments as track_host without rgbA / depthA; track i draws mesh weight_ids[i] (mesh 0
        without ids); mode / image_hw as in render(); iterations as in track_render (k > 1 uploads the whole frame).  fit as in
        track_render (the whole depth frame is uploaded then): the fit rows come last in what the call returns, an int32 numpy
        array (n, 6).  icp as in track_render (the whole depth frame is uploaded then): its stats come last, a float64 numpy
        array (n, 4)."""
        out, tr, ro, rows, stats, _ = self._track_host(
            'track_render_host', frame_rgb, frame_depth, K, poses, object_width, (), self._render_mode(mode, image_hw),
            trans_normalizer, rot_normalizer, weight_ids, precision, want_residuals, fill_depth, iterations, fit, icp)
        res = ((out, tr, ro) if want_residuals else (out,)) + tuple(x for x in (rows, stats) if x is not None)
        return res if len(res) > 1 else out

    def _track_host(self, fn, frame_rgb, frame_depth, K, poses, object_width, A, render, trans_normalizer, rot_normalizer,
                    weight_ids, precision, want_residuals, fill_depth, iterations, fit=None, icp=None, hyp=None, draw_keys=None):
        """The host route of every tracking method, one C call: track_host (A = (rgbA, depthA), render None),
        track_render_host and track_hypotheses_host (A = (), render = _render_mode's triple; hyp: hypothesis_spec's options).
        -> (poses, trans, rot, fit rows, ICP stats, choice) as numpy arrays, each None when the call has none."""
        n = int(poses.shape[0])
        iterations = self.refine_iterations(iterations)
        tau = self.fit_spec(fit)
        icp = self.icp_spec(icp)
        for name, a, dt, shape in self._track_inputs(fn, frame_rgb, frame_depth, poses, object_width, A, n):
            if not (isinstance(a, np.ndarray) and a.dtype == dt and a.shape == shape and a.flags['C_CONTIGUOUS']):
                raise ValueError('%s: %s must be a C-contiguous %s array of shape %s' % (fn, name, dt, shape))
        if draw_keys is not None:
            draw_keys = np.ascontiguousarray(draw_keys, dtype=np.int64)
            if draw_keys.shape != (n,):
                raise ValueError('%s: draw_keys must have one entry per track' % fn)
        wid = self._host_ids(fn, weight_ids, n)
        fill = self.depth_fill_spec(fill_depth)
        Kh = self._k4(K)
        out = np.empty((n, 4, 4), dtype=np.float64)
        tr = np.empty((n, 3), dtype=np.float32) if want_residuals else None
        ro = np.empty((n, 3), dtype=np.float32) if want_residuals else None
        rows = np.empty((n, _lib.FIT_COLS), dtype=np.int32) if tau else None
        stats = np.empty((n, _lib.ICP_COLS), dtype=np.float64) if icp is not None else None
        choice = np.empty(n, dtype=np.int32) if hyp is not None else None
        H, W = frame_depth.shape
        head = (self._ctx, _hptr(frame_rgb), _hptr(frame_depth), H, W, _hptr(Kh), _hptr(poses), _hptr(object_width))
        tail = (_hptr(wid), n, float(trans_normalizer), float(rot_normalizer), PREC[precision], _hptr(out), _hptr(tr), _hptr(ro),
                self._track_opts(fill, iterations, tau, icp, hyp))
        if render is None:
            rc = self.lib.se3tn_track_host(*head, *map(_hptr, A), *tail, _stream(self.device))
        else:
            arrays = _track_arrays(_hptr, draw_keys=draw_keys, out_fit=rows, out_choice=choice, out_icp=stats)
            rc = self.lib.se3tn_track_render_host(*head, *render, *tail, arrays, _stream(self.device))
        _lib.check(rc, self._ctx)
        return out, tr, ro, rows, stats, choice

    # ------------------------------------------------------------------ multi-hypothesis tracking
    @staticmethod
    def hypothesis_spec(hypotheses, seed, max_translation, max_rotation_deg):
        """se3tn_hypothesis_opts of a hypothesis call: S in [1, MAX_HYPOTHESES], a 64-bit seed, the spread in metres (finite, in
        (0, 1]) and degrees (in (0, 180]); else a ValueError."""
        S = hypotheses
        if isinstance(S, (bool, np.bool_)) or not isinstance(S, (int, np.integer)) or not 1 <= S <= _lib.MAX_HYPOTHESES:
            raise ValueError('hypotheses must be an integer in [1, %d], not %r' % (_lib.MAX_HYPOTHESES, S))
        if isinstance(seed, (bool, np.bool_)) or not isinstance(seed, (int, np.integer)):
            raise ValueError('seed must be an integer, not %r' % (seed,))
        mt, mr = float(max_translation), float(max_rotation_deg)
        if not (math.isfinite(mt) and 0 < mt <= 1):
            raise ValueError('max_translation must be finite and in (0, 1] m, not %r' % (max_translation,))
        if not 0 < mr <= 180:
            raise ValueError('max_rotation_deg must be in (0, 180], not %r' % (max_rotation_deg,))
        seed = int(seed) & ((1 << 64) - 1)
        return _lib.HypothesisOpts(hypotheses=int(S), seed=seed - (1 << 64) if seed >= 1 << 63 else seed, max_translation=mt,
                                   max_rotation_deg=mr)

    def draw_hypotheses(self, poses, draw_keys, hypotheses, max_translation, max_rotation_deg, seed=0, want_draws=False):
        """The starts a hypothesis step expands n tracks into (se3tn_draw_hypotheses): poses float64 (n,4,4) and draw_keys int64
        (n) CUDA tensors (draw_keys may be None when hypotheses is 1) -> float64 (n,S,4,4) [, float64 (n,S,8) draws: the
        translation's U_theta, U_phi, the rotation axis' U_theta, U_phi, m_T (m), m_R (degrees), tries_T, tries_R]."""
        n = int(poses.shape[0])
        hyp = self.hypothesis_spec(hypotheses, seed, max_translation, max_rotation_deg)
        self._check_dev('poses', poses, torch.float64, (n, 4, 4))
        if draw_keys is not None:
            self._check_dev('draw_keys', draw_keys, torch.int64, (n,))
        S = hyp.hypotheses
        out = torch.empty(n, S, 4, 4, dtype=torch.float64, device=self.device)
        draws = torch.empty(n, S, _lib.HYP_DRAWS, dtype=torch.float64, device=self.device) if want_draws else None
        _lib.check(self.lib.se3tn_draw_hypotheses(self._ctx, _ptr(poses), _ptr(draw_keys), n, C.byref(hyp), _ptr(out), _ptr(draws),
                                                  _stream(self.device)), self._ctx)
        return (out, draws) if want_draws else out

    def track_hypotheses(self, frame_rgb, frame_depth, K, poses, object_width, trans_normalizer, rot_normalizer, draw_keys,
                         hypotheses, max_translation, max_rotation_deg, seed=0, fit=None, weight_ids_host=None, weight_ids_dev=None,
                         precision='bf16x3', mode='vispy', image_hw=None, out_poses=None, out_trans=None, out_rot=None,
                         fill_depth=None, iterations=1, out_choice=None, out_fit=None, out_hyp_poses=None, out_rounds=None):
        """track_render from S start hypotheses per track, keeping the one whose model fits the frame best
        (se3tn_track_opts.hyp), enqueued on the current stream.  draw_keys int64 (n) CUDA tensor: each track's draw key (None
        only with hypotheses=1); the spread is max_translation m / max_rotation_deg degrees; fit: tau in mm, required (fit_spec).
        -> (poses (n,4,4), choice int32 (n), fit rows int32 (n,6)), then out_hyp_poses (n,S,4,4) and out_rounds (k,n,S,4,4)
        when given (float64 CUDA tensors: every hypothesis after the last round, and after every round).  out_poses may be
        poses itself."""
        hyp = self.hypothesis_spec(hypotheses, seed, max_translation, max_rotation_deg)
        P, _, _, rows, _, choice = self._track(
            'track_hypotheses', frame_rgb, frame_depth, K, poses, object_width, (), self._render_mode(mode, image_hw), trans_normalizer,
            rot_normalizer, weight_ids_host, weight_ids_dev, precision, out_poses, out_trans, out_rot, fill_depth, iterations, fit,
            hyp=hyp, draw_keys=draw_keys, out_rounds=out_rounds, out_fit=out_fit, out_choice=out_choice, out_hyp_poses=out_hyp_poses)
        return (P, choice, rows) + tuple(t for t in (out_hyp_poses, out_rounds) if t is not None)

    def track_hypotheses_host(self, frame_rgb, frame_depth, K, poses, object_width, trans_normalizer, rot_normalizer, draw_keys,
                              hypotheses, max_translation, max_rotation_deg, seed=0, fit=None, weight_ids=None, precision='bf16x3',
                              mode='vispy', image_hw=None, fill_depth=None, iterations=1):
        """track_hypotheses with numpy arrays in and out, synchronous (se3tn_track_render_host): arguments as
        track_render_host, draw_keys int64 (n) numpy or None (hypotheses=1).  -> (poses (n,4,4), choice int32 (n), fit rows
        int32 (n,6))."""
        hyp = self.hypothesis_spec(hypotheses, seed, max_translation, max_rotation_deg)
        out, _, _, rows, _, choice = self._track_host(
            'track_hypotheses_host', frame_rgb, frame_depth, K, poses, object_width, (), self._render_mode(mode, image_hw),
            trans_normalizer, rot_normalizer, weight_ids, precision, False, fill_depth, iterations, fit, hyp=hyp, draw_keys=draw_keys)
        return out, choice, rows

    # ------------------------------------------------------------------ checkpoint validation
    # init_spec's defaults: starting guesses, not tuned on a real sensor: 300 x 24 = 7,200 candidates about 12 x 15 degrees
    # apart, the 8 best refined by 5 ICP iterations at icp_spec's gate, a 20 mm inlier gate, at least 100 mask pixels with depth
    INIT_DEFAULTS = dict(viewpoints=300, inplane=24, keep=8, tau_mm=20, min_pixels=100, icp=5)
    INIT_STATUS = {1: 'the {} is empty', 2: 'too few {} pixels have depth (min_pixels)'}
    INIT_ARRAYS = ('stats', 't0', 'cand_rows', 'kept_rows', 'kept_poses', 'icp_poses', 'icp_rows', 'icp_stats')

    @staticmethod
    def init_spec(init=None):
        """se3tn_init_opts from None (INIT_DEFAULTS) or a dict of any of viewpoints (1..4096), inplane (1..360; viewpoints x
        inplane <= 65536), keep (1..MAX_INIT_KEEP), tau_mm (1..1000), min_pixels (1..176*176) and icp (icp_spec's argument;
        None / 0: the best grid candidate without refinement); the rest from INIT_DEFAULTS.  Else a ValueError."""
        spec = dict(Engine.INIT_DEFAULTS)
        if init is not None:
            if not isinstance(init, dict):
                raise ValueError('init must be None or a dict, not %r' % (init,))
            unknown = set(init) - set(spec)
            if unknown:
                raise ValueError('init: unknown fields %s' % sorted(unknown))
            spec.update(init)
        limits = {'viewpoints': (1, 4096), 'inplane': (1, 360), 'keep': (1, _lib.MAX_INIT_KEEP), 'tau_mm': (1, 1000),
                  'min_pixels': (1, IMAGE_SIZE * IMAGE_SIZE)}
        for k, (lo, hi) in limits.items():
            v = spec[k]
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
                raise ValueError('init %s must be an integer in [%d, %d], not %r' % (k, lo, hi, v))
        if spec['viewpoints'] * spec['inplane'] > 65536:
            raise ValueError('init viewpoints x inplane = %d exceeds 65536' % (spec['viewpoints'] * spec['inplane']))
        if spec['keep'] > spec['viewpoints'] * spec['inplane']:
            raise ValueError('init keep=%d exceeds the %d candidates' % (spec['keep'], spec['viewpoints'] * spec['inplane']))
        icp = Engine.icp_spec(spec['icp'])
        return _lib.InitOpts(viewpoints=int(spec['viewpoints']), inplane=int(spec['inplane']), keep=int(spec['keep']),
                             tau_mm=int(spec['tau_mm']), min_pixels=int(spec['min_pixels']), icp=None if icp is None else C.pointer(icp))

    def init_poses(self, frame_depth, seg, K, labels, object_width, weight_ids=None, mode='vispy', image_hw=None, init=None, out=None):
        """Start poses for n objects of one frame from their segmentation labels and the depth (se3tn_init_poses): a rotation
        grid at each mask's centroid ray and median depth, rendered and scored against the depth and the mask, the best `keep`
        refined by ICP.  frame_depth uint16 (H,W) mm and seg uint8 (H,W) CUDA tensors; K 3x3 or (fx,fy,cx,cy); labels (n) ints
        in 1..255; object_width float64 CUDA (n) mm; weight_ids int32 (n) host array or None (mesh 0); mode / image_hw as in
        render(); init: init_spec's argument.  out: a dict that may hold 'poses' (float64 (n,4,4)), 'rows' (int32 (n,8)) and any
        of INIT_ARRAYS (include/se3tn.h's se3tn_init_arrays, shaped (n, ...)) as CUDA tensors to fill.  -> (poses float64 (n,4,4),
        all NaN for an object whose status is not 0, rows int32 (n, INIT_COLS): status, candidate, model, maskc, overlap, pairs,
        inlier, delta_mm), queued on the current stream."""
        return self._init('init_poses', frame_depth, K, object_width, weight_ids, mode, image_hw, init, out, seg, labels, None)

    @staticmethod
    def init_status(status, source):
        """The text of an init row's status (INIT_STATUS) for a start from a 'mask' or a 'box'."""
        return Engine.INIT_STATUS.get(int(status), '?').format(source)

    def _init(self, fn, frame_depth, K, object_width, weight_ids, mode, image_hw, init, out, seg, rows, D):
        """init_poses' and init_boxes' checks and their one library call.  A start from a label image: seg, its labels as rows
        and D None; from boxes: seg None, and the boxes as rows and D as box_spec gives them."""
        opts = self.init_spec(init)
        H, W = frame_depth.shape
        self._check_dev('frame_depth', frame_depth, torch.uint16, (H, W))
        if D is None:
            rows = np.ascontiguousarray(rows, dtype=np.int32).reshape(-1)
            self._check_dev('seg', seg, torch.uint8, (H, W))
        n = int(rows.shape[0])
        self._check_dev('object_width', object_width, torch.float64, (n,))
        wh = self._host_ids(fn, weight_ids, n)
        wd = torch.from_numpy(wh).to(self.device) if wh is not None else None
        out = dict(out or {})
        unknown = set(out) - {'poses', 'rows'} - set(self.INIT_ARRAYS)
        if unknown:
            raise ValueError('%s: unknown outputs %s' % (fn, sorted(unknown)))
        VR, Kk = opts.viewpoints * opts.inplane, opts.keep
        shapes = dict(poses=((n, 4, 4), torch.float64), rows=((n, _lib.INIT_COLS), torch.int32),
                      stats=((n, _lib.INIT_STATS), torch.int64), t0=((n, 3) if D is None else (n, D, 3), torch.float64),
                      cand_rows=((n, (D or 1) * VR, _lib.INIT_COLS), torch.int32), kept_rows=((n, Kk, _lib.INIT_COLS), torch.int32),
                      kept_poses=((n, Kk, 4, 4), torch.float64), icp_poses=((n, Kk, 4, 4), torch.float64),
                      icp_rows=((n, Kk, _lib.INIT_COLS), torch.int32), icp_stats=((n, Kk, _lib.ICP_COLS), torch.float64))
        for k in ('poses', 'rows'):
            if out.get(k) is None:
                out[k] = torch.empty(shapes[k][0], dtype=shapes[k][1], device=self.device)
        for k, t in out.items():
            if t is not None:
                self._check_dev('out[%r]' % k, t, shapes[k][1], shapes[k][0])
        arrays = _lib.InitArrays(**{k: _ptr(out.get(k)).value for k in self.INIT_ARRAYS})
        rmode, rH, rW = self._render_mode(mode, image_hw)
        call, src = (self.lib.se3tn_init_poses, (_ptr(frame_depth), _ptr(seg), int(H), int(W), _hptr(self._k4(K)), _hptr(rows))) \
            if D is None else (self.lib.se3tn_init_boxes, (_ptr(frame_depth), int(H), int(W), _hptr(self._k4(K)), _hptr(rows), D))
        _lib.check(call(self._ctx, *src, _ptr(object_width), rmode, rH, rW, _hptr(wh), _ptr(wd), n, C.byref(opts), _ptr(out['poses']),
                        _ptr(out['rows']), C.byref(arrays), _stream(self.device)), self._ctx)
        return out['poses'], out['rows']

    # init_boxes' default depth count: a starting guess, like INIT_DEFAULTS -- the quantiles 1/8, 3/8, 5/8 and 7/8 of the box's
    # depths, so that one of them lies on the object when the background fills up to half of the box
    INIT_BOX_DEPTHS = 4
    MAX_INIT_DEPTHS = 8

    @staticmethod
    def depths_spec(depths):
        """init_boxes' depth candidates D checked as an integer in [1, MAX_INIT_DEPTHS] -> int."""
        if isinstance(depths, (bool, np.bool_)) or not isinstance(depths, (int, np.integer)) or not 1 <= depths <= Engine.MAX_INIT_DEPTHS:
            raise ValueError('init depths must be an integer in [1, %d], not %r' % (Engine.MAX_INIT_DEPTHS, depths))
        return int(depths)

    @staticmethod
    def box_spec(boxes, depths=INIT_BOX_DEPTHS):
        """boxes (n, 4) integers (x0, y0, x1, y1), half-open, as a contiguous int32 array, and depths_spec(depths).  Float boxes
        are a ValueError: round a detector's box with box_pixels first."""
        depths = Engine.depths_spec(depths)
        b = np.asarray(boxes)
        if b.size and (b.dtype == np.bool_ or not np.issubdtype(b.dtype, np.integer)):
            raise ValueError('boxes must be integers (x0, y0, x1, y1), not %s' % b.dtype)
        if b.size % 4 or (b.size and b.shape[-1] != 4):
            raise ValueError('boxes must be (n, 4), not %s' % (b.shape,))
        if b.size and (b.min() < -2 ** 31 or b.max() >= 2 ** 31):
            raise ValueError('boxes must fit int32')
        return np.ascontiguousarray(b, dtype=np.int32).reshape(-1, 4), int(depths)

    @staticmethod
    def box_pixels(box, H, W):
        """A detector's (x0, y0, x1, y1) in frame pixels, floats allowed, as the half-open integer box init_boxes takes: rounded
        outwards (floor x0 / y0, ceil x1 / y1) and clipped to the H x W frame.  Non-finite values are a ValueError."""
        b = np.asarray(box, dtype=np.float64).reshape(-1)
        if b.shape != (4,) or not np.isfinite(b).all():
            raise ValueError('box must be four finite numbers (x0, y0, x1, y1), not %r' % (box,))
        x0, y0 = np.floor(b[0]), np.floor(b[1])
        x1, y1 = np.ceil(b[2]), np.ceil(b[3])
        clip = lambda v, hi: int(min(max(v, 0), hi))
        x0, x1, y0, y1 = clip(x0, W), clip(x1, W), clip(y0, H), clip(y1, H)
        return np.array([x0, y0, max(x0, x1), max(y0, y1)], np.int32)

    def init_boxes(self, frame_depth, boxes, K, object_width, weight_ids=None, mode='vispy', image_hw=None, init=None,
                   depths=INIT_BOX_DEPTHS, out=None):
        """Start poses for n objects of one frame from 2D boxes and the depth (se3tn_init_boxes): init_poses' rule with each
        object's pixels the box's, D = depths depth candidates along the ray through the box centre (the quantiles
        (2 d + 1) / 2 D of the box's depths), and the D V R candidates of an object ranked together.  frame_depth uint16 (H,W)
        mm CUDA tensor; boxes (n, 4) ints (x0, y0, x1, y1), half-open, inside the frame, may overlap; depths in [1,
        MAX_INIT_DEPTHS]; the rest as init_poses.  out as init_poses', with t0 (n, D, 3) and cand_rows (n, D V R, INIT_COLS);
        column 1 of a row is the candidate d V R + v R + r.  -> (poses float64 (n,4,4), NaN where the status is not 0 -- 1: the
        box is empty, 2: too few of its pixels have depth --, rows int32 (n, INIT_COLS)), queued on the current stream."""
        return self._init('init_boxes', frame_depth, K, object_width, weight_ids, mode, image_hw, init, out, None, *self.box_spec(boxes, depths))

    # ------------------------------------------------------------------ re-initialisation of lost tracks
    # reinit_spec's defaults: guesses, not tuned -- `predict --fit --score` shows how well the inlier fraction separates lost
    # from kept tracks on a data set, which is what to choose them by
    REINIT_DEFAULTS = dict(below=0.5, after=3)

    @staticmethod
    def reinit_source(fn, n, seg=None, labels=None, boxes=None, depths=INIT_BOX_DEPTHS):
        """reinit's seg (uint8, numpy or a tensor) with labels (n ints in 1..255), or boxes and depths, for n tracks, checked ->
        _init's seg, rows and D, a row per track: (seg as given, labels, None), (None, boxes, D), or all None without either."""
        if seg is not None and boxes is not None:
            raise ValueError('%s: give seg / labels or boxes, not both' % fn)
        lab = np.ascontiguousarray([] if labels is None else labels, dtype=np.int64).reshape(-1)
        if (seg is not None or labels is not None) and (lab.shape != (n,) or (seg is not None and n and (lab.min() < 1 or lab.max() > 255))):
            raise ValueError('%s: labels must be %d ints in 1..255, not %r' % (fn, n, labels))
        if boxes is not None:
            b, D = Engine.box_spec(boxes, depths)
            if b.shape != (n, 4):
                raise ValueError('%s: boxes must be (%d, 4), not %s' % (fn, n, b.shape))
            return None, b, D
        if seg is not None and seg.dtype not in (np.uint8, torch.uint8):
            raise ValueError('%s: seg must be a uint8 label image, not %s' % (fn, seg.dtype))
        return seg, (None if seg is None else lab), None

    @staticmethod
    def reinit_spec(below=0.5, after=3):
        """se3tn_reinit_opts: below, the inlier fraction under which a track counts as below, in (0, 1] and exact in three
        decimals (it is passed as permille: 0.5 -> 500; 0.1234 is a ValueError); after, the frames in a row below that make a
        track lost, an integer in [1, 1000]."""
        if isinstance(below, (bool, np.bool_)) or not isinstance(below, (int, float, np.integer, np.floating)):
            raise ValueError('reinit below must be a number in (0, 1], not %r' % (below,))
        try:
            permille = decimal.Decimal(repr(float(below))) * 1000
        except decimal.InvalidOperation:
            raise ValueError('reinit below must be a number in (0, 1], not %r' % (below,)) from None
        if not permille.is_finite() or permille != permille.to_integral_value() or not 1 <= permille <= 1000:
            raise ValueError('reinit below must be in (0, 1] with at most three decimals (a whole permille), not %r' % (below,))
        if isinstance(after, (bool, np.bool_)) or not isinstance(after, (int, np.integer)) or not 1 <= after <= 1000:
            raise ValueError('reinit after must be an integer in [1, 1000], not %r' % (after,))
        return _lib.ReinitOpts(below_permille=int(permille), after=int(after))

    def lost_tracks(self, fit_rows, streak, below=0.5, after=3, out_event=None, out_lost=None):
        """The loss rule over one step's fit rows (se3tn_lost_tracks), queued on the current stream: fit_rows int32 (n, 6) and
        streak int32 (n) CUDA tensors, the streak updated in place.  -> (event int32 (n): 1 below, 0 not; lost int32 (n + 1):
        the count of lost tracks, then their indices in ascending order)."""
        opts = self.reinit_spec(below, after)
        n = int(fit_rows.shape[0])
        self._check_dev('fit_rows', fit_rows, torch.int32, (n, _lib.FIT_COLS))
        self._check_dev('streak', streak, torch.int32, (n,))
        out_event = torch.empty(n, dtype=torch.int32, device=self.device) if out_event is None else out_event
        out_lost = torch.empty(n + 1, dtype=torch.int32, device=self.device) if out_lost is None else out_lost
        self._check_dev('out_event', out_event, torch.int32, (n,))
        self._check_dev('out_lost', out_lost, torch.int32, (n + 1,))
        _lib.check(self.lib.se3tn_lost_tracks(self._ctx, _ptr(fit_rows), n, C.byref(opts), _ptr(streak), _ptr(out_event),
                                              _ptr(out_lost), _stream(self.device)), self._ctx)
        return out_event, out_lost

    def fit_poses(self, frame_depth, K, poses, object_width, fit, weight_ids=None, mode='vispy', image_hw=None, out=None):
        """The tracking step's fit check at given poses (se3tn_fit_poses), queued on the current stream: frame_depth uint16
        (H,W) mm, poses float64 (n,4,4), object_width float64 (n) CUDA tensors; fit: tau in mm (fit_spec, required); weight_ids
        int32 (n) host array or None (mesh 0); mode / image_hw as in render().  -> int32 (n, 6) rows (model, observed, inlier,
        front, behind, residual), exactly those of a track_render step with the same fit at these poses on this frame."""
        tau = self.fit_spec(fit)
        if not tau:
            raise ValueError('fit_poses: fit must be a tau in mm, not %r' % (fit,))
        n = int(poses.shape[0])
        H, W = frame_depth.shape
        self._check_dev('frame_depth', frame_depth, torch.uint16, (H, W))
        self._check_dev('poses', poses, torch.float64, (n, 4, 4))
        self._check_dev('object_width', object_width, torch.float64, (n,))
        wh = self._host_ids('fit_poses', weight_ids, n)
        wd = torch.from_numpy(wh).to(self.device) if wh is not None else None
        out = torch.empty(n, _lib.FIT_COLS, dtype=torch.int32, device=self.device) if out is None else out
        self._check_dev('out', out, torch.int32, (n, _lib.FIT_COLS))
        rmode, rH, rW = self._render_mode(mode, image_hw)
        _lib.check(self.lib.se3tn_fit_poses(self._ctx, _ptr(frame_depth), int(H), int(W), _hptr(self._k4(K)), _ptr(poses),
                                            _ptr(object_width), rmode, rH, rW, _hptr(wh), _ptr(wd), n, int(tau), _ptr(out),
                                            _stream(self.device)), self._ctx)
        return out

    def accept_starts(self, lost, starts, init_rows, start_fit, poses, fit_rows, streak, event):
        """The accept rule for the starts of the lost tracks (se3tn_accept_starts), queued on the current stream: lost int32 (m)
        host array of track indices; starts float64 (m,4,4), init_rows int32 (m, INIT_COLS), start_fit int32 (m, 6) CUDA
        tensors.  poses float64 (n,4,4), fit_rows int32 (n,6), streak and event int32 (n) CUDA tensors are updated in place:
        a restarted track takes its start's pose and row (event 2), a start without init status 0 is event 3, one that fits no
        better event 4; the m streaks go back to 0."""
        idx = np.ascontiguousarray(lost, dtype=np.int32).reshape(-1)
        m, n = int(idx.shape[0]), int(poses.shape[0])
        for name, t, dt, shape in (('starts', starts, torch.float64, (m, 4, 4)), ('init_rows', init_rows, torch.int32, (m, _lib.INIT_COLS)),
                                   ('start_fit', start_fit, torch.int32, (m, _lib.FIT_COLS)), ('poses', poses, torch.float64, (n, 4, 4)),
                                   ('fit_rows', fit_rows, torch.int32, (n, _lib.FIT_COLS)), ('streak', streak, torch.int32, (n,)),
                                   ('event', event, torch.int32, (n,))):
            self._check_dev(name, t, dt, shape)
        idx_d = torch.from_numpy(idx).to(self.device)
        _lib.check(self.lib.se3tn_accept_starts(self._ctx, _hptr(idx), _ptr(idx_d), m, _ptr(starts), _ptr(init_rows), _ptr(start_fit),
                                                n, _ptr(poses), _ptr(fit_rows), _ptr(streak), _ptr(event), _stream(self.device)), self._ctx)

    def reinit(self, frame_depth, seg, K, labels, object_width, poses, fit_rows, streak, fit, below=0.5, after=3, weight_ids=None,
               mode='vispy', image_hw=None, init=None, fill_depth=None, boxes=None, depths=INIT_BOX_DEPTHS):
        """Re-initialise the lost tracks of one tracking step from their masks (include/se3tn.h): the loss rule over the step's
        fit rows (lost_tracks), the lost list copied back through pinned memory (one synchronisation of the current stream,
        the call's only one), then, when some track is lost and seg is given, one init_poses call on the lost tracks in
        ascending order, fit_poses at their starts and accept_starts.
        poses float64 (n,4,4) and fit_rows int32 (n,6) CUDA tensors (the step's output and its fit rows) are updated in place;
        streak int32 (n) CUDA tensor, the tracks' streaks, persists across calls (zeros at the start).  frame_depth uint16 (H,W)
        mm and seg uint8 (H,W) label image (or None: no attempt) are CUDA tensors or numpy arrays, uploaded only when a track is
        lost; fill_depth as in track_render: the depth is filled first, as the step filled it.  labels (n) ints in 1..255,
        object_width float64 CUDA (n), weight_ids int32 (n) host array or None (mesh 0), mode / image_hw as in render(): the
        step's.  fit: the step's tau in mm; init: init_spec's argument.  boxes: instead of seg (at most one of the two), each
        track's (x0, y0, x1, y1) box in this frame, ints (n, 4) as init_boxes takes them; the lost tracks' rows go through one
        init_boxes call with `depths`, and labels may be None.  -> event int32 (n) CUDA tensor: 0 not below, 1 below and no
        attempt, 2 restarted, 3 no start, 4 start rejected."""
        tau = self.fit_spec(fit)
        if not tau:
            raise ValueError('reinit: fit must be the step\'s tau in mm, not %r' % (fit,))
        n = int(poses.shape[0])
        seg, rows, D = self.reinit_source('reinit', n, seg, labels, boxes, depths)
        wh = self._host_ids('reinit', weight_ids, n)
        event, lost = self.lost_tracks(fit_rows, streak, below, after)
        pin = getattr(self, '_reinit_pin', None)
        if pin is None or pin.numel() < n + 1:
            pin = self._reinit_pin = torch.empty(max(n, self.max_batch) + 1, dtype=torch.int32, pin_memory=True)
        pin[:n + 1].copy_(lost, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        m = int(pin[0])
        if m == 0 or rows is None:
            return event
        idx = pin[1:1 + m].numpy().copy()
        as_dev = lambda a, dt: a.to(self.device, dt).contiguous() if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a)).to(self.device, dt)
        depth_d = as_dev(frame_depth, torch.uint16)
        on, max_depth, extrapolate, blur = self.depth_fill_spec(fill_depth)
        if on:
            depth_d = self.fill_depth(depth_d, max_depth, extrapolate=bool(extrapolate), blur_type='gaussian' if blur else 'bilateral')
        sub_ids = None if wh is None else wh[idx]
        width = object_width.index_select(0, lost[1:1 + m].long())
        starts, init_rows = self._init('reinit', depth_d, K, width, sub_ids, mode, image_hw, init, None,
                                       None if seg is None else as_dev(seg, torch.uint8), rows[idx], D)
        start_fit = self.fit_poses(depth_d, K, starts, width, tau, weight_ids=sub_ids, mode=mode, image_hw=image_hw)
        self.accept_starts(idx, starts, init_rows, start_fit, poses, fit_rows, streak, event)
        return event

    def eval_pairs(self, rgbA, depthA, rgbB, depthB, A_in_cam, B_in_cam, trans_normalizer, rot_normalizer,
                   weight_ids_host=None, weight_ids_dev=None, precision='bf16x3', want_terms=False, want_labels=False,
                   out_trans=None, out_rot=None, out_sums=None, out_sq=None, out_labels=None, augment=None, segB=None,
                   pair_index=None, out_rgbB=None, out_depthB=None):
        """The loss of n ready-made pairs in one step (se3tn_eval_pairs): processData's post-transforms, the network in eval mode
        and Se3TrackNet.loss's terms, enqueued on the current stream.  rgbA / rgbB uint8 (n,176,176,3), depthA / depthB uint16
        (n,176,176), A_in_cam / B_in_cam float64 (n,4,4), all contiguous CUDA tensors.  -> (trans (n,3), rot (n,3), sums (2,)
        float32: the summed translation / rotation squared errors, sq (n,6) float32 or None, labels (n,6) float64 or None).
        MSE = sums / (3 n).  Pass out_* tensors to keep the step's addresses, and so its CUDA graph, across calls.

        augment: an se3tn_augment (augment_config) to evaluate input B under the reference's train-time augmentations
        (se3tn_eval_pairs_augmented): pair_index int64 (n) CUDA tensor, each pair's index (the key of its draws), segB uint8
        (n,176,176) CUDA tensor or None (maskB = depthB > 100); out_rgbB / out_depthB receive the augmented crops when given."""
        n = int(A_in_cam.shape[0])
        for name, t, dt, shape in (('rgbA', rgbA, torch.uint8, (n, IMAGE_SIZE, IMAGE_SIZE, 3)), ('rgbB', rgbB, torch.uint8, (n, IMAGE_SIZE, IMAGE_SIZE, 3)),
                                   ('depthA', depthA, torch.uint16, (n, IMAGE_SIZE, IMAGE_SIZE)), ('depthB', depthB, torch.uint16, (n, IMAGE_SIZE, IMAGE_SIZE)),
                                   ('A_in_cam', A_in_cam, torch.float64, (n, 4, 4)), ('B_in_cam', B_in_cam, torch.float64, (n, 4, 4))):
            self._check_dev(name, t, dt, shape)
        out_trans = torch.empty(n, 3, dtype=torch.float32, device=self.device) if out_trans is None else out_trans
        out_rot = torch.empty(n, 3, dtype=torch.float32, device=self.device) if out_rot is None else out_rot
        out_sums = torch.empty(2, dtype=torch.float32, device=self.device) if out_sums is None else out_sums
        if out_sq is None and want_terms:
            out_sq = torch.empty(n, 6, dtype=torch.float32, device=self.device)
        if out_labels is None and want_labels:
            out_labels = torch.empty(n, 6, dtype=torch.float64, device=self.device)
        for name, t, dt, shape in (('out_trans', out_trans, torch.float32, (n, 3)), ('out_rot', out_rot, torch.float32, (n, 3)),
                                   ('out_sums', out_sums, torch.float32, (2,)), ('out_sq', out_sq, torch.float32, (n, 6)),
                                   ('out_labels', out_labels, torch.float64, (n, 6))):
            if t is not None:
                self._check_dev(name, t, dt, shape)
        wh = None
        if weight_ids_host is not None:
            wh = np.ascontiguousarray(weight_ids_host, dtype=np.int32)
            if wh.shape != (n,):
                raise ValueError('eval_pairs: weight_ids_host must have one entry per pair')
            if weight_ids_dev is None:
                weight_ids_dev = torch.from_numpy(wh).to(self.device)
        args = (self._ctx, _ptr(rgbA), _ptr(depthA), _ptr(rgbB), _ptr(depthB), _ptr(A_in_cam), _ptr(B_in_cam),
                wh.ctypes.data_as(C.c_void_p) if wh is not None else C.c_void_p(0), _ptr(weight_ids_dev), n,
                float(trans_normalizer), float(rot_normalizer), PREC[precision],
                _ptr(out_trans), _ptr(out_rot), _ptr(out_sq), _ptr(out_labels), _ptr(out_sums))
        if augment is None:
            if segB is not None or pair_index is not None or out_rgbB is not None or out_depthB is not None:
                raise ValueError('eval_pairs: segB, pair_index and out_rgbB / out_depthB go with augment')
            _lib.check(self.lib.se3tn_eval_pairs(*args, _stream(self.device)), self._ctx)
        else:
            self._check_augment_inputs(n, segB, pair_index, out_rgbB=out_rgbB, out_depthB=out_depthB)
            _lib.check(self.lib.se3tn_eval_pairs_augmented(*args, _ptr(segB), _ptr(pair_index), C.byref(augment), _ptr(out_rgbB),
                                                           _ptr(out_depthB), _stream(self.device)), self._ctx)
        return out_trans, out_rot, out_sums, out_sq, out_labels

    # ------------------------------------------------------------------ augmentation (se3tn_augment)
    @staticmethod
    def augment_config(seed=0, hsv=None, bright=None, noise=None, blur=None, cover=None):
        """An se3tn_augment: each stage None (off) or a dict of its arguments -- hsv (h, s, v, prob), bright (lo, hi), noise
        (rgb, depth, prob), blur (max_kernel, prob), cover (prob).  data_augmentation.chain_config builds it from the reference's
        classes."""
        a = _lib.Augment()
        a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        if hsv is not None:
            a.hsv_jitter = 1; a.hsv_prob = hsv['prob']
            for k, c in enumerate('hsv'):
                a.hsv_noise[k] = hsv[c]
        if bright is not None:
            a.change_bright = 1; a.bright_mag[0] = bright['lo']; a.bright_mag[1] = bright['hi']
        if noise is not None:
            a.gaussian_noise = 1; a.noise_rgb = noise['rgb']; a.noise_depth = noise['depth']; a.noise_prob = noise['prob']
        if blur is not None:
            a.gaussian_blur = 1; a.blur_max_kernel = int(blur['max_kernel']); a.blur_prob = blur['prob']
        if cover is not None:
            a.black_cover = 1; a.cover_prob = cover['prob']
        return a

    def augment_draws(self, augment, depthB, pair_index, segB=None, want_noise=False):
        """The draws eval_pairs(augment=...) uses for these pairs (se3tn_augment_draws): depthB uint16 (n,176,176), pair_index
        int64 (n), segB uint8 (n,176,176) or None, CUDA tensors -> (params float64 (n, AUG_PARAMS), noise_rgb float64 (n,176,176,3),
        noise_depth float64 (n,176,176)), the noise fields None without want_noise."""
        n = int(pair_index.shape[0])
        self._check_augment_inputs(n, segB, pair_index, depthB=depthB)
        params = torch.empty(n, _lib.AUG_PARAMS, dtype=torch.float64, device=self.device)
        nr = torch.empty(n, IMAGE_SIZE, IMAGE_SIZE, 3, dtype=torch.float64, device=self.device) if want_noise else None
        nd = torch.empty(n, IMAGE_SIZE, IMAGE_SIZE, dtype=torch.float64, device=self.device) if want_noise else None
        _lib.check(self.lib.se3tn_augment_draws(self._ctx, C.byref(augment), _ptr(depthB), _ptr(segB), _ptr(pair_index), n, _ptr(params),
                                                _ptr(nr), _ptr(nd), _stream(self.device)), self._ctx)
        return params, nr, nd

    def augment_crops(self, augment, rgbB, depthB, pair_index, segB=None, out_rgbB=None, out_depthB=None):
        """The augmented input B of these pairs, as eval_pairs(augment=...) forms it (se3tn_augment_crops): CUDA tensors as
        augment_draws plus rgbB uint8 (n,176,176,3) -> (rgbB, depthB) augmented."""
        n = int(pair_index.shape[0])
        out_rgbB = torch.empty(n, IMAGE_SIZE, IMAGE_SIZE, 3, dtype=torch.uint8, device=self.device) if out_rgbB is None else out_rgbB
        out_depthB = torch.empty(n, IMAGE_SIZE, IMAGE_SIZE, dtype=torch.uint16, device=self.device) if out_depthB is None else out_depthB
        self._check_augment_inputs(n, segB, pair_index, rgbB=rgbB, depthB=depthB, out_rgbB=out_rgbB, out_depthB=out_depthB)
        _lib.check(self.lib.se3tn_augment_crops(self._ctx, C.byref(augment), _ptr(rgbB), _ptr(depthB), _ptr(segB), _ptr(pair_index), n,
                                                _ptr(out_rgbB), _ptr(out_depthB), _stream(self.device)), self._ctx)
        return out_rgbB, out_depthB

    def _check_augment_inputs(self, n, segB, pair_index, **images):
        img = (n, IMAGE_SIZE, IMAGE_SIZE)
        if pair_index is None:
            raise ValueError('augmentation needs pair_index: the int64 index of each pair, the key of its draws')
        self._check_dev('pair_index', pair_index, torch.int64, (n,))
        if segB is not None:
            self._check_dev('segB', segB, torch.uint8, img)
        for name, t in images.items():
            if t is not None:
                self._check_dev(name, t, torch.uint8 if 'rgb' in name else torch.uint16, img + ((3,) if 'rgb' in name else ()))

    def pair_loss(self, trans, rot, trans_label, rot_label, out_sums=None):
        """Se3TrackNet.loss's sums on existing predictions (se3tn_pair_loss): float32 (n,3) predictions, float64 (n,3) labels,
        contiguous CUDA tensors -> float32 (2,) CUDA tensor of the summed translation / rotation squared errors, added exactly as
        eval_pairs adds them."""
        n = int(trans.shape[0])
        for name, t, dt in (('trans', trans, torch.float32), ('rot', rot, torch.float32),
                            ('trans_label', trans_label, torch.float64), ('rot_label', rot_label, torch.float64)):
            self._check_dev(name, t, dt, (n, 3))
        out_sums = torch.empty(2, dtype=torch.float32, device=self.device) if out_sums is None else out_sums
        self._check_dev('out_sums', out_sums, torch.float32, (2,))
        _lib.check(self.lib.se3tn_pair_loss(self._ctx, _ptr(trans), _ptr(rot), _ptr(trans_label), _ptr(rot_label), n, _ptr(out_sums),
                                            _stream(self.device)), self._ctx)
        return out_sums

    # ------------------------------------------------------------------ metrics (SURVEY 8f row 1)
    def add_adi(self, model_pts, pred, gt, want_add=True, want_adi=True):
        """ADD / ADD-S (reference Utils.py:72-98) of n pose pairs: float64 CUDA tensors model (m,3), pred/gt (n,4,4)."""
        n = pred.shape[0]
        out_add = torch.empty(n, dtype=torch.float64, device=self.device) if want_add else None
        out_adi = torch.empty(n, dtype=torch.float64, device=self.device) if want_adi else None
        _lib.check(self.lib.se3tn_add_adi(self._ctx, _ptr(model_pts), int(model_pts.shape[0]), _ptr(pred), _ptr(gt), n,
                                          _ptr(out_add), _ptr(out_adi), _stream(self.device)), self._ctx)
        return out_add, out_adi

    def vocap(self, errs):
        """VOCap (reference eval_ycb.py:45-64) of a float64 CUDA error vector -> python float in [0,1]."""
        ap = C.c_double(0.0)
        _lib.check(self.lib.se3tn_vocap(self._ctx, _ptr(errs), int(errs.numel()), C.byref(ap), _stream(self.device)), self._ctx)
        return ap.value

    def add_adi_sets(self, points, pose_set, pred, gt, set_offsets=None, want_add=True, want_adi=True):
        """add_adi for the poses of several objects in one launch (se3tn_add_adi_sets).  points: a list of each object's (m_s,3)
        float64 model points (numpy arrays or tensors), or one float64 CUDA table (M,3) with set_offsets (S+1) int32 giving each
        object's rows.  pose_set (n) int32: the object of each pose; pred / gt float64 CUDA tensors (n,4,4).
        -> (out_add, out_adi) float64 CUDA tensors (n), bit-identical to add_adi on each pose's own points."""
        table, offs, ids = self._point_sets('add_adi_sets', points, set_offsets, pose_set)
        n = int(ids.shape[0])
        self._check_dev('pred', pred, torch.float64, (n, 4, 4))
        self._check_dev('gt', gt, torch.float64, (n, 4, 4))
        out_add = torch.empty(n, dtype=torch.float64, device=self.device) if want_add else None
        out_adi = torch.empty(n, dtype=torch.float64, device=self.device) if want_adi else None
        _lib.check(self.lib.se3tn_add_adi_sets(self._ctx, _ptr(table), int(table.shape[0]), _hptr(offs), int(offs.shape[0]) - 1, _hptr(ids),
                                               _ptr(pred), _ptr(gt), n, _ptr(out_add), _ptr(out_adi), _stream(self.device)), self._ctx)
        return out_add, out_adi

    def pose_errors_sets(self, points, pose_set, pred, gt, set_offsets=None, keep=None):
        """Translation error (mm), rotation angle (degrees), ADD and ADD-S of n poses in one launch (se3tn_pose_errors_sets).
        points / set_offsets / pose_set / pred / gt as add_adi_sets takes them; keep: None or a uint8 CUDA tensor (n), a 0 row
        left unscored.  -> (errors float64 CUDA (n, 4), set ids int32 CUDA (n): a kept row's pose_set entry, -1 for the others);
        a row that is not kept has NaN errors.  ADD / ADD-S are add_adi_sets' values bit for bit."""
        table, offs, ids = self._point_sets('pose_errors_sets', points, set_offsets, pose_set)
        n = int(ids.shape[0])
        self._check_dev('pred', pred, torch.float64, (n, 4, 4))
        self._check_dev('gt', gt, torch.float64, (n, 4, 4))
        if keep is not None:
            self._check_dev('keep', keep, torch.uint8, (n,))
        out = torch.empty((n, 4), dtype=torch.float64, device=self.device)
        out_set = torch.empty(n, dtype=torch.int32, device=self.device)
        _lib.check(self.lib.se3tn_pose_errors_sets(self._ctx, _ptr(table), int(table.shape[0]), _hptr(offs), int(offs.shape[0]) - 1,
                                                   _hptr(ids), _ptr(pred), _ptr(gt), _ptr(keep), n, _ptr(out), _ptr(out_set),
                                                   _stream(self.device)), self._ctx)
        return out, out_set

    def vocap_sets(self, errs, err_set, n_sets):
        """VOCap of each set's errors and of all of them (se3tn_vocap_sets): errs float64 CUDA tensor (n), err_set (n) int32
        set ids in [0, n_sets) -> float64 numpy (n_sets+1,): one AP per set, then the pooled AP, each as vocap() computes it."""
        n = int(errs.numel())
        self._check_dev('errs', errs, torch.float64, (n,))
        ids = err_set.to(self.device, torch.int32).contiguous() if torch.is_tensor(err_set) else \
            torch.from_numpy(np.ascontiguousarray(err_set, dtype=np.int32)).to(self.device)
        if ids.shape != (n,):
            raise ValueError('vocap_sets: err_set must have one id per error')
        out = np.zeros(int(n_sets) + 1, dtype=np.float64)
        _lib.check(self.lib.se3tn_vocap_sets(self._ctx, _ptr(errs), _ptr(ids), n, int(n_sets), _hptr(out), _stream(self.device)), self._ctx)
        return out

    def _point_sets(self, fn, points, set_offsets, pose_set):
        """add_adi_sets' points / set_offsets / pose_set -> (float64 CUDA table (M,3), int32 offsets (S+1), int32 ids (n)), host
        arrays for the offsets and ids."""
        if torch.is_tensor(points):
            table = points
            if set_offsets is None:
                raise ValueError('%s: a point table needs set_offsets' % fn)
        else:
            sets = [np.asarray(p.cpu().numpy() if torch.is_tensor(p) else p, dtype=np.float64).reshape(-1, 3) for p in points]
            set_offsets = np.cumsum([0] + [len(p) for p in sets])
            table = torch.from_numpy(np.ascontiguousarray(np.concatenate(sets) if sets else np.zeros((0, 3)))).to(self.device)
        offs = np.ascontiguousarray(set_offsets, dtype=np.int32)
        ids = np.ascontiguousarray(pose_set.cpu().numpy() if torch.is_tensor(pose_set) else pose_set, dtype=np.int32).reshape(-1)
        if offs.ndim != 1 or offs.shape[0] < 2:
            raise ValueError('%s: set_offsets must hold S+1 >= 2 offsets' % fn)
        self._check_dev('points', table, torch.float64, (table.shape[0], 3))
        return table, offs, ids

    def metrics_scratch_bytes(self):
        """Device bytes the context holds for add_adi_sets / vocap_sets / draw_tracks."""
        return int(self.lib.se3tn_metrics_scratch_bytes(self._ctx))

    # ------------------------------------------------------------------ result videos
    def draw_tracks(self, frame_rgb, K, poses, points, set_offsets, track_set, label=None, label_order='under', out=None):
        """Each track's model points drawn over one frame, as the reference's result videos draw them (se3tn_draw_tracks).
        frame_rgb uint8 CUDA (H,W,3), H and W even; K 3x3 or (fx,fy,cx,cy); poses float64 CUDA (n,4,4); points float64 CUDA (M,3),
        set_offsets (S+1) and track_set (n) int32 host arrays: track i draws points [set_offsets[s], set_offsets[s+1]), s =
        track_set[i].  label: None or (y0, mask), mask a uint8 CUDA (rows, W) strip from row y0 that is non-zero where the
        label's pixels are (label_strip renders one); label_order 'under' (getResultsYcb) or 'over' (predictSequenceYcb /
        YcbInEOAT) the points.  -> uint8 CUDA (n, H/2, W/2, 3) BGR images (into `out` when given), queued on the current stream."""
        H, W = int(frame_rgb.shape[0]), int(frame_rgb.shape[1])
        offs = np.ascontiguousarray(set_offsets, dtype=np.int32).reshape(-1)
        ids = np.ascontiguousarray(track_set, dtype=np.int32).reshape(-1)
        n = int(ids.shape[0])
        if offs.shape[0] < 2:
            raise ValueError('draw_tracks: set_offsets must hold S+1 >= 2 offsets')
        if label_order not in LABEL_ORDER:
            raise ValueError('draw_tracks: label_order must be one of %s' % ', '.join(LABEL_ORDER))
        self._check_dev('frame_rgb', frame_rgb, torch.uint8, (H, W, 3))
        self._check_dev('poses', poses, torch.float64, (n, 4, 4))
        self._check_dev('points', points, torch.float64, (points.shape[0], 3))
        y0, mask = (0, None) if label is None else (int(label[0]), label[1])
        if mask is not None:
            self._check_dev('label mask', mask, torch.uint8, (mask.shape[0], W))
        if out is None:
            out = torch.empty((n, H // 2, W // 2, 3), dtype=torch.uint8, device=self.device)
        self._check_dev('out', out, torch.uint8, (n, H // 2, W // 2, 3))
        _lib.check(self.lib.se3tn_draw_tracks(self._ctx, _ptr(frame_rgb), H, W, _hptr(self._k4(K)), _ptr(poses), n,
                                              _ptr(points), int(points.shape[0]), _hptr(offs), int(offs.shape[0]) - 1, _hptr(ids),
                                              _ptr(mask), y0, 0 if mask is None else int(mask.shape[0]), LABEL_ORDER[label_order],
                                              _ptr(out), _stream(self.device)), self._ctx)
        return out

    # ------------------------------------------------------------------ input A renderer (SURVEY 8f row 2)
    def set_mesh(self, mesh, mesh_id=0):
        """Upload a CAD model (dict pos float32 (nv,3), nrm float32 (nv,3), col uint8 (nv,3), faces int32 (nf,3)) -- the
        vertex / index buffers of the reference's VispyRenderer (vispy_renderer.py:108-129)."""
        pos = np.ascontiguousarray(mesh['pos'], dtype=np.float32); nrm = np.ascontiguousarray(mesh['nrm'], dtype=np.float32)
        col = np.ascontiguousarray(mesh['col'], dtype=np.uint8); faces = np.ascontiguousarray(mesh['faces'], dtype=np.int32)
        if pos.ndim != 2 or pos.shape[1] != 3 or nrm.shape != pos.shape or col.shape != pos.shape or faces.ndim != 2 or faces.shape[1] != 3:
            raise ValueError('mesh arrays must be pos/nrm/col (nv,3) and faces (nf,3)')
        _lib.check(self.lib.se3tn_set_mesh(self._ctx, int(mesh_id), pos.ctypes.data, nrm.ctypes.data, col.ctypes.data, faces.ctypes.data,
                                           int(pos.shape[0]), int(faces.shape[0])), self._ctx)

    def render(self, K, poses, object_width, mesh_ids=None, out_rgb=None, out_depth=None, mode='vispy', image_hw=None):
        """Tracker.render_window for n tracks (reference predict.py:193-215): float64 CUDA poses (n,4,4) and widths (n) ->
        rgbA uint8 (n,176,176,3), depthA uint16 (n,176,176) CUDA tensors.  mode 'vispy' (lit, the crop window is the GL viewport) or
        'pyrender' (unlit render of the whole image_hw = (H, W) camera image, then crop_bbox; dataset_info['renderer'] == 'pyrenderer')."""
        n = int(poses.shape[0])
        rgb = out_rgb if out_rgb is not None else torch.empty((n, 176, 176, 3), dtype=torch.uint8, device=self.device)
        dep = out_depth if out_depth is not None else torch.empty((n, 176, 176), dtype=torch.uint16, device=self.device)
        Kh = self._k4(K)
        rmode, H, W = self._render_mode(mode, image_hw)
        _lib.check(self.lib.se3tn_render_ex(self._ctx, Kh.ctypes.data_as(C.c_void_p), _ptr(poses), _ptr(object_width), _ptr(mesh_ids), n,
                                            rmode, H, W, _ptr(rgb), _ptr(dep), _stream(self.device)), self._ctx)
        return rgb, dep

    # ------------------------------------------------------------------ held-out pairs (produce_train_pair_data.py)
    def crop_bbox_seg(self, frame_rgb, frame_depth, seg, bbox, out_hw=(IMAGE_SIZE, IMAGE_SIZE), class_ids=None):
        """crop_bbox with the segmentation plane (se3tn_crop_bbox_seg): seg uint8 CUDA (H,W) -> (rgb, depth, seg, count).  Without
        class_ids seg holds the labels and count is None; with class_ids (int32 CUDA (n)) seg is (label == class id) as 0 / 1 and
        count (int32 (n)) the number of ones."""
        n = int(bbox.shape[0])
        H, W = frame_depth.shape
        self._check_dev('seg', seg, torch.uint8, (H, W))
        crop_rgb = torch.empty(n, out_hw[0], out_hw[1], 3, dtype=torch.uint8, device=self.device)
        crop_depth = torch.empty(n, out_hw[0], out_hw[1], dtype=torch.uint16, device=self.device)
        crop_seg = torch.empty(n, out_hw[0], out_hw[1], dtype=torch.uint8, device=self.device)
        count = torch.empty(n, dtype=torch.int32, device=self.device) if class_ids is not None else None
        _lib.check(self.lib.se3tn_crop_bbox_seg(self._ctx, _ptr(frame_rgb), _ptr(frame_depth), _ptr(seg), H, W, _ptr(bbox), _ptr(class_ids),
                                                n, int(out_hw[0]), int(out_hw[1]), _ptr(crop_rgb), _ptr(crop_depth), _ptr(crop_seg),
                                                _ptr(count), _stream(self.device)), self._ctx)
        return crop_rgb, crop_depth, crop_seg, count

    def visibility(self, seg, K, poses, class_ids, mesh_ids=None, out_visible=None, out_covered=None):
        """The visibility check's two counts for m rows of one frame (se3tn_visibility): seg uint8 CUDA (H,W), K 3x3 or (fx,fy,cx,cy),
        poses float64 CUDA (m,4,4), class_ids int32 (m) (host or CUDA), mesh_ids int32 (m) host array or None (mesh 0).  The camera
        image is the seg frame's size.  -> (visible, covered) int32 CUDA (m): #(seg == class id) and the pixels of the model's
        full-image pyrender-mode render whose float32 depth is > 0.1."""
        m = int(poses.shape[0])
        H, W = seg.shape
        self._check_dev('seg', seg, torch.uint8, (H, W))
        self._check_dev('poses', poses, torch.float64, (m, 4, 4))
        cid = self._dev_ids(class_ids, m)
        mh = self._host_ids('visibility', mesh_ids, m)
        md = torch.from_numpy(mh).to(self.device) if mh is not None else None
        vis = torch.empty(m, dtype=torch.int32, device=self.device) if out_visible is None else out_visible
        cov = torch.empty(m, dtype=torch.int32, device=self.device) if out_covered is None else out_covered
        self._check_dev('out_visible', vis, torch.int32, (m,)); self._check_dev('out_covered', cov, torch.int32, (m,))
        _lib.check(self.lib.se3tn_visibility(self._ctx, _ptr(seg), int(H), int(W), _hptr(self._k4(K)), _ptr(poses), _hptr(mh), _ptr(md),
                                             _ptr(cid), m, _ptr(vis), _ptr(cov), _stream(self.device)), self._ctx)
        return vis, cov

    def perturb_pairs(self, frame_rgb, frame_depth, seg, K, A_in_cam, object_width, class_ids, mesh_ids=None, mesh_ids_dev=None, out=None):
        """One ProducerPurturb.generate step for n samples of one frame (se3tn_perturb_pairs): compute_bbox of each A_in_cam, A rendered
        in the pyrender mode over the frame-sized camera image and cropped, B / depthB / segB cropped from the frame through the same
        window.  frame_rgb uint8 (H,W,3), frame_depth uint16 (H,W), seg uint8 (H,W), A_in_cam float64 (n,4,4), object_width float64
        (n), class_ids int32 (n): CUDA tensors; mesh_ids int32 host array (n) or None (mesh 0).  out: a dict of output tensors to
        reuse (keeps the step's addresses, so its CUDA graph).  -> dict rgbA, depthA, rgbB, depthB, segB (0/1), count (int32 (n))."""
        n = int(A_in_cam.shape[0])
        H, W = frame_depth.shape
        for name, t, dt, shape in (('frame_rgb', frame_rgb, torch.uint8, (H, W, 3)), ('frame_depth', frame_depth, torch.uint16, (H, W)),
                                   ('seg', seg, torch.uint8, (H, W)), ('A_in_cam', A_in_cam, torch.float64, (n, 4, 4)),
                                   ('object_width', object_width, torch.float64, (n,)), ('class_ids', class_ids, torch.int32, (n,))):
            self._check_dev(name, t, dt, shape)
        mh = self._host_ids('perturb_pairs', mesh_ids, n)
        if mh is not None and mesh_ids_dev is None:
            mesh_ids_dev = torch.from_numpy(mh).to(self.device)
        img = (n, IMAGE_SIZE, IMAGE_SIZE)
        spec = dict(rgbA=(img + (3,), torch.uint8), depthA=(img, torch.uint16), rgbB=(img + (3,), torch.uint8), depthB=(img, torch.uint16),
                    segB=(img, torch.uint8), count=((n,), torch.int32))
        out = dict(out) if out is not None else {}
        for k, (shape, dt) in spec.items():
            if k not in out:
                out[k] = torch.empty(shape, dtype=dt, device=self.device)
            self._check_dev('out[%r]' % k, out[k], dt, shape)
        _lib.check(self.lib.se3tn_perturb_pairs(self._ctx, _ptr(frame_rgb), _ptr(frame_depth), _ptr(seg), int(H), int(W), _hptr(self._k4(K)),
                                                _ptr(A_in_cam), _ptr(object_width), _hptr(mh), _ptr(mesh_ids_dev), _ptr(class_ids), n,
                                                *(_ptr(out[k]) for k in spec), _stream(self.device)), self._ctx)
        return out

    def append_pairs(self, pairs, A_in_cam, B_in_cam, queue_ids, tails_host, tails_dev, queues, queue_ids_dev=None):
        """The kept rows of a pair step appended to per-queue validation batches in one launch (se3tn_append_pairs).  pairs:
        perturb_pairs' output dict (rgbA, depthA, rgbB, depthB, count) of n rows; A_in_cam, B_in_cam float64 CUDA (n,4,4);
        queue_ids int32 host array (n), uploaded unless queue_ids_dev is given; tails_host int32 host array (Q): what tails_dev
        (int32 CUDA (Q)) holds when the append runs, read only by the capacity check; queues: dict rgbA, depthA, rgbB, depthB,
        A_in_cam, B_in_cam of CUDA tensors (Q, cap, ...) in eval_pairs' layout.  A row is kept when its count reaches
        _lib.PAIR_MIN_SEG; tails_dev advances on the device.  When queues also holds 'segB' (uint8 (Q, cap, 176, 176)), each kept
        row's pairs['segB'] goes with it, in the same launch (se3tn_append_pairs_seg)."""
        n = int(A_in_cam.shape[0])
        Q, cap = int(queues['rgbA'].shape[0]), int(queues['rgbA'].shape[1])
        img = (IMAGE_SIZE, IMAGE_SIZE)
        seg = 'segB' in queues
        for name, t, dt, shape in (('rgbA', pairs['rgbA'], torch.uint8, (n,) + img + (3,)), ('depthA', pairs['depthA'], torch.uint16, (n,) + img),
                                   ('rgbB', pairs['rgbB'], torch.uint8, (n,) + img + (3,)), ('depthB', pairs['depthB'], torch.uint16, (n,) + img),
                                   ('count', pairs['count'], torch.int32, (n,)), ('A_in_cam', A_in_cam, torch.float64, (n, 4, 4)),
                                   ('B_in_cam', B_in_cam, torch.float64, (n, 4, 4)), ('tails_dev', tails_dev, torch.int32, (Q,))) + \
                ((('segB', pairs.get('segB'), torch.uint8, (n,) + img),) if seg else ()):
            self._check_dev(name, t, dt, shape)
        for name, dt, shape in (('rgbA', torch.uint8, img + (3,)), ('depthA', torch.uint16, img), ('rgbB', torch.uint8, img + (3,)),
                                ('depthB', torch.uint16, img), ('A_in_cam', torch.float64, (4, 4)), ('B_in_cam', torch.float64, (4, 4))) + \
                ((('segB', torch.uint8, img),) if seg else ()):
            self._check_dev('queues[%r]' % name, queues[name], dt, (Q, cap) + shape)
        qh = self._host_ids('append_pairs', queue_ids, n)
        th = np.ascontiguousarray(tails_host, dtype=np.int32)
        if th.shape != (Q,):
            raise ValueError('append_pairs: tails_host must have one entry per queue')
        if queue_ids_dev is None:
            queue_ids_dev = torch.from_numpy(qh).to(self.device)
        args = (self._ctx, *(_ptr(pairs[k]) for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'count')), _ptr(A_in_cam), _ptr(B_in_cam),
                _hptr(qh), _ptr(queue_ids_dev), n, Q, cap, _hptr(th), _ptr(tails_dev),
                *(_ptr(queues[k]) for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A_in_cam', 'B_in_cam')))
        if seg:
            _lib.check(self.lib.se3tn_append_pairs_seg(*args, _ptr(pairs['segB']), _ptr(queues['segB']), _stream(self.device)), self._ctx)
        else:
            _lib.check(self.lib.se3tn_append_pairs(*args, _stream(self.device)), self._ctx)

    def _dev_ids(self, ids, n):
        """int32 (n) ids as a contiguous CUDA tensor (host arrays are uploaded)."""
        t = ids.to(self.device, torch.int32).contiguous() if torch.is_tensor(ids) else \
            torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)).to(self.device)
        if t.shape != (n,):
            raise ValueError('expected %d ids, got %s' % (n, tuple(t.shape)))
        return t

    @staticmethod
    def _render_mode(mode, image_hw):
        """(SE3TN_RENDER_* value, H, W) of a render mode name and the camera image size it needs."""
        if mode not in ('vispy', 'pyrender'):
            raise ValueError("render mode must be 'vispy' or 'pyrender'")
        if mode == 'pyrender' and image_hw is None:
            raise ValueError("render(mode='pyrender') needs image_hw=(H, W), the camera image pyrender draws")
        H, W = (int(image_hw[0]), int(image_hw[1])) if image_hw is not None else (0, 0)
        return (_lib.RENDER_PYRENDER if mode == 'pyrender' else _lib.RENDER_VISPY), H, W

    # ------------------------------------------------------------------ pose exchange over a raw NCCL communicator (SURVEY 8e)
    def allgather_poses_nccl(self, nccl_comm, local_poses, out=None, world_size=None):
        """se3tn_allgather_poses: for hosts that own an ncclComm_t (an int / c_void_p handle).  torch.distributed users call
        dist.all_gather_poses instead.  local_poses (n,4,4) float64 CUDA -> (world*n,4,4), rank-major."""
        n = int(local_poses.shape[0])
        if out is None:
            if world_size is None:
                raise ValueError('need out= or world_size=')
            out = torch.empty((world_size * n, 4, 4), dtype=torch.float64, device=self.device)
        _lib.check(self.lib.se3tn_allgather_poses(self._ctx, C.c_void_p(int(nccl_comm)), _ptr(local_poses), _ptr(out), n, _stream(self.device)), self._ctx)
        return out

    # ------------------------------------------------------------------ live-sensor depth (SURVEY 8f row 4)
    def fill_depth(self, depth_mm, max_depth=2.0, want_metres=False, extrapolate=False, blur_type='bilateral'):
        """fill_depth (reference Utils.py:455-514; predict_ros.py:38-41 uses the defaults): uint16 mm CUDA tensor (H,W) ->
        uint16 mm CUDA tensor (and float32 metres with want_metres)."""
        if depth_mm.dtype != torch.uint16 or depth_mm.dim() != 2 or not depth_mm.is_cuda or not depth_mm.is_contiguous():
            raise ValueError('depth_mm must be a contiguous uint16 CUDA tensor (H,W)')
        if blur_type not in ('bilateral', 'gaussian'):
            raise ValueError("blur_type must be 'bilateral' or 'gaussian'")
        H, W = depth_mm.shape
        out = torch.empty_like(depth_mm)
        out_m = torch.empty((H, W), dtype=torch.float32, device=self.device) if want_metres else None
        _lib.check(self.lib.se3tn_fill_depth_ex(self._ctx, _ptr(depth_mm), int(H), int(W), float(max_depth), int(bool(extrapolate)),
                                                1 if blur_type == 'gaussian' else 0, _ptr(out), _ptr(out_m), _stream(self.device)), self._ctx)
        return (out, out_m) if want_metres else out

    @staticmethod
    def depth_fill_spec(fill_depth):
        """(enable, max_depth, extrapolate, blur_type), se3tn_track_opts' fill, from the tracking calls' fill_depth argument:
        None / False: the frame's depth is used as it is.  True: fill_depth as the reference's ROS node calls it before every
        on_track (predict_ros.py:38-41: max_depth 2.0 m, no extrapolation, bilateral).  A dict with any of max_depth /
        extrapolate / blur_type: those arguments of fill_depth, the rest as with True."""
        if fill_depth is None or isinstance(fill_depth, (bool, np.bool_)):
            return (1, 2.0, 0, 0) if fill_depth else (0, 0.0, 0, 0)
        if not isinstance(fill_depth, dict) or not set(fill_depth) <= {'max_depth', 'extrapolate', 'blur_type'}:
            raise ValueError('fill_depth must be None, a bool or a dict with max_depth / extrapolate / blur_type')
        blur_type = fill_depth.get('blur_type', 'bilateral')
        if blur_type not in ('bilateral', 'gaussian'):
            raise ValueError("blur_type must be 'bilateral' or 'gaussian'")
        max_depth = float(fill_depth.get('max_depth', 2.0))
        if not (math.isfinite(max_depth) and max_depth > 0):
            raise ValueError('max_depth must be finite and > 0')
        return (1, max_depth, int(bool(fill_depth.get('extrapolate', False))), 1 if blur_type == 'gaussian' else 0)

    @staticmethod
    def refine_iterations(k):
        """The refinement count of a tracking call as an int: 1..MAX_REFINE_ITERATIONS (se3tn_track_opts.iterations), else a
        ValueError."""
        if isinstance(k, (bool, np.bool_)) or not isinstance(k, (int, np.integer)) or not 1 <= k <= _lib.MAX_REFINE_ITERATIONS:
            raise ValueError('iterations must be an integer in [1, %d], not %r' % (_lib.MAX_REFINE_ITERATIONS, k))
        return int(k)

    @staticmethod
    def fit_spec(fit):
        """The fit check of a tracking call as se3tn_track_opts' fit_tau_mm: None -> 0 (off), an integer in [1, 1000] -> itself,
        else a ValueError."""
        if fit is None:
            return 0
        if isinstance(fit, (bool, np.bool_)) or not isinstance(fit, (int, np.integer)) or not 1 <= fit <= 1000:
            raise ValueError('fit must be None or an integer tau in mm in [1, 1000], not %r' % (fit,))
        return int(fit)

    # icp_spec's defaults for an integer M: starting guesses (a gate a little wider than a depth sensor's noise at a metre, and
    # enough pixels for six unknowns to be well determined), not tuned on a real sensor or a trained checkpoint
    ICP_TAU_DEFAULT = 20
    ICP_MIN_INLIERS_DEFAULT = 100

    @staticmethod
    def icp_spec(icp):
        """The depth refinement of a tracking call as se3tn_icp_opts, or None (off): None / 0 -> None; an integer M in
        [1, MAX_ICP_ITERATIONS] -> M iterations at tau ICP_TAU_DEFAULT mm and min_inliers ICP_MIN_INLIERS_DEFAULT; a dict with
        'iterations' and optional 'tau_mm' (1..1000) and 'min_inliers' (6..176*176) sets those fields.  Else a ValueError."""
        if icp is None or (isinstance(icp, (int, np.integer)) and not isinstance(icp, (bool, np.bool_)) and icp == 0):
            return None
        spec = dict(icp) if isinstance(icp, dict) else {'iterations': icp}
        unknown = set(spec) - {'iterations', 'tau_mm', 'min_inliers'}
        if unknown:
            raise ValueError('icp: unknown fields %s' % sorted(unknown))
        spec.setdefault('tau_mm', Engine.ICP_TAU_DEFAULT)
        spec.setdefault('min_inliers', Engine.ICP_MIN_INLIERS_DEFAULT)
        limits = {'iterations': (1, _lib.MAX_ICP_ITERATIONS), 'tau_mm': (1, 1000), 'min_inliers': (6, IMAGE_SIZE * IMAGE_SIZE)}
        for k, (lo, hi) in limits.items():
            v = spec.get(k)
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
                raise ValueError('icp %s must be an integer in [%d, %d], not %r' % (k, lo, hi, v))
        return _lib.IcpOpts(iterations=int(spec['iterations']), tau_mm=int(spec['tau_mm']), min_inliers=int(spec['min_inliers']))

    @staticmethod
    def _track_opts(fill, iterations, tau, icp=None, hyp=None):
        """The se3tn_track_opts of one tracking call, by reference: depth_fill_spec's tuple, the refinement count, the fit
        check's tau, and icp_spec's and hypothesis_spec's options or None.  Every call passes all of them, so Trackers that
        share an Engine each get their own.  The reference keeps the struct, and the struct the options it points to, alive."""
        on, max_depth, extrapolate, blur = fill
        ref = lambda o: None if o is None else C.pointer(o)
        return C.byref(_lib.TrackOpts(fill_depth=on, fill_extrapolate=extrapolate, fill_blur=blur, iterations=iterations,
                                      fill_max_depth=max_depth, fit_tau_mm=tau, icp=ref(icp), hyp=ref(hyp)))

    def _fit_rows_view(self):
        """An int32 CUDA tensor (max_batch, 6) over the context's fit rows (se3tn_fit_rows; the address never changes)."""
        if getattr(self, '_fit_rows', None) is None:
            p = C.c_void_p()
            _lib.check(self.lib.se3tn_fit_rows(self._ctx, C.byref(p)), self._ctx)
            shape = (self.max_batch, _lib.FIT_COLS)

            class _Rows:                                 # a borrowed device array: no stream, so torch adds no synchronisation
                __cuda_array_interface__ = {'shape': shape, 'typestr': '<i4', 'data': (p.value, False), 'version': 2}
            with torch.cuda.device(self.device):
                self._fit_rows = torch.as_tensor(_Rows(), device=self.device)
        return self._fit_rows

    # ------------------------------------------------------------------ introspection
    def debug_buffer(self, buf_id, n):
        """A float32 view (n, floats_per_image) of an internal NHWC activation buffer."""
        p = C.c_void_p(); fpi = C.c_size_t()
        _lib.check(self.lib.se3tn_debug_buffer(self._ctx, buf_id, C.byref(p), C.byref(fpi)), self._ctx)
        offb = p.value - self._workspace.data_ptr()
        nbytes = n * fpi.value * 4
        return self._workspace[offb:offb + nbytes].view(torch.float32).view(n, fpi.value)

    def set_profiling(self, enable=True):
        _lib.check(self.lib.se3tn_set_profiling(self._ctx, int(bool(enable))), self._ctx)

    def get_profile(self):
        """Device ms of each kernel of the last call (PROFILE_SLOTS slots, see include/se3tn.h)."""
        ms = (C.c_float * _lib.PROFILE_SLOTS)()
        _lib.check(self.lib.se3tn_get_profile(self._ctx, ms), self._ctx)
        return np.array(ms[:], dtype=np.float64)

    def get_trace(self):
        """(14, 256, 8) uint64 globaltimer stamps of the last forward's conv CTAs (needs SE3TN_TRACE=1 at Engine creation)."""
        return self._trace_words()[:14 * 256 * 8].reshape(14, 256, 8)

    def get_tile_trace(self):
        """(8, TRACE_TILES, 4) uint64 per-tile stamps of the last forward's 8 resident-weight conv launches (include/se3tn.h)."""
        return self._trace_words()[14 * 256 * 8:].reshape(8, _lib.TRACE_TILES, 4)

    def _trace_words(self):
        out = np.zeros(14 * 256 * 8 + 8 * _lib.TRACE_TILES * 4, dtype=np.uint64)
        _lib.check(self.lib.se3tn_get_trace(self._ctx, out.ctypes.data_as(C.c_void_p)), self._ctx)
        return out

    def last_launch_count(self):
        return self.lib.se3tn_last_launch_count(self._ctx)

    def last_step_was_graph(self):
        """True when the last track_batch / track_render call replayed (or just captured and launched) a CUDA graph of the whole step."""
        return bool(self.lib.se3tn_last_step_was_graph(self._ctx))

    # ------------------------------------------------------------------ checks
    def _check_img(self, t):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 4 and
                tuple(t.shape[1:]) == (4, IMAGE_SIZE, IMAGE_SIZE)):
            raise ValueError('expected a contiguous float32 CUDA tensor of shape (n,4,176,176), got %s %s' % (t.dtype, tuple(t.shape)))

    def _check_dev(self, name, t, dtype, shape):
        if not (isinstance(t, torch.Tensor) and t.get_device() == self.device.index and t.dtype == dtype and t.is_contiguous()
                and t.shape == tuple(shape)):
            raise ValueError('%s must be a contiguous %s CUDA tensor of shape %s on %s' % (name, dtype, tuple(shape), self.device))

    @staticmethod
    def _track_inputs(fn, frame_rgb, frame_depth, poses, object_width, A, n):
        """(name, value, dtype name, shape) of each input of the tracking call fn; A is (rgbA, depthA), or () when the call
        renders input A."""
        hw = tuple(frame_depth.shape)
        if len(hw) != 2:
            raise ValueError('%s: frame_depth must be (H, W)' % fn)
        rows = (('frame_rgb', frame_rgb, 'uint8', hw + (3,)), ('frame_depth', frame_depth, 'uint16', hw),
                ('poses', poses, 'float64', (n, 4, 4)), ('object_width', object_width, 'float64', (n,)))
        return rows + tuple(zip(('rgbA', 'depthA'), A, ('uint8', 'uint16'), ((n, IMAGE_SIZE, IMAGE_SIZE, 3), (n, IMAGE_SIZE, IMAGE_SIZE))))

    def _check_frame(self, fn, frame_rgb, frame_depth, poses, object_width, A, n):
        """The CUDA tensors of a tracking call.  A None input is passed on as a null pointer, which the library rejects."""
        for name, t, dt, shape in self._track_inputs(fn, frame_rgb, frame_depth, poses, object_width, A, n):
            if t is not None:
                self._check_dev(name, t, getattr(torch, dt), shape)
        if n > self.max_batch:
            raise ValueError('n=%d exceeds max_batch=%d' % (n, self.max_batch))

    @staticmethod
    def _host_ids(fn, weight_ids, n):
        """weight_ids as a C-contiguous int32 (n) host array, or None."""
        if weight_ids is None:
            return None
        wid = np.ascontiguousarray(weight_ids, dtype=np.int32)
        if wid.shape != (n,):
            raise ValueError('%s: weight_ids must have one entry per track' % fn)
        return wid

    @staticmethod
    def _k4(K):
        K = np.asarray(K, dtype=np.float64)
        if K.shape == (3, 3):
            return np.ascontiguousarray([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], dtype=np.float64)
        if K.shape == (4,):
            return np.ascontiguousarray(K)
        raise ValueError('K must be 3x3 or (fx,fy,cx,cy)')
