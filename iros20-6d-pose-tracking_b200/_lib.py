"""ctypes binding of libse3tn.so (the C ABI in include/se3tn.h).  No torch types cross it."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libse3tn.so')

OK, ERR_INVALID, ERR_CUDA, ERR_NOMEM, ERR_STATE, ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5
PREC_TF32, PREC_FP32, PREC_BF16X3, PREC_BF16, PREC_FP8, PREC_FP16 = 0, 1, 2, 3, 4, 5
FP8_SCALES = 8
RENDER_VISPY, RENDER_PYRENDER = 0, 1
LABEL_UNDER_POINTS, LABEL_OVER_POINTS = 0, 1
WEIGHT_BLOB_FLOATS = 13528326
PROFILE_SLOTS = 22
TRACE_TILES = 5184
PAIR_MIN_SEG = 100
MAX_REFINE_ITERATIONS = 8
FIT_COLS = 6
AUG_PARAMS = 24
AUG_MAX_CORNERS = 64
MAX_HYPOTHESES = 32
HYP_DRAWS = 8
MAX_ICP_ITERATIONS = 16
ICP_COLS = 4
INIT_COLS = 8
INIT_STATS = 6
MAX_INIT_KEEP = 32
REINIT_NONE, REINIT_BELOW, REINIT_RESTARTED, REINIT_NO_START, REINIT_REJECTED = 0, 1, 2, 3, 4

_vp, _i, _d, _sz = C.c_void_p, C.c_int, C.c_double, C.c_size_t

# name -> (restype, argtypes); mirrors include/se3tn.h one to one
SIGNATURES = {
    'se3tn_workspace_bytes': (_sz, [_i]),
    'se3tn_weight_set_bytes': (_sz, []),
    'se3tn_create': (_i, [_i, _i, _vp, C.POINTER(_vp)]),
    'se3tn_destroy': (None, [_vp]),
    'se3tn_last_error': (C.c_char_p, [_vp]),
    'se3tn_load_weights': (_i, [_vp, _i, _vp, _sz]),
    'se3tn_set_stats': (_i, [_vp, _i, _vp, _vp, _i]),
    'se3tn_calibrate_fp8': (_i, [_vp, _i, _vp, _vp, _i, _vp]),
    'se3tn_set_fp8_scales': (_i, [_vp, _i, _vp, _i]),
    'se3tn_get_fp8_scales': (_i, [_vp, _i, _vp, _i]),
    'se3tn_preprocess': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_normalize': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    'se3tn_compute_bbox': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    'se3tn_crop_bbox': (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    'se3tn_forward': (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp]),
    'se3tn_forward_preprocessed': (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp]),
    'se3tn_pose_update': (_i, [_vp, _vp, _vp, _vp, _d, _d, _vp, _i, _vp]),
    'se3tn_so3_log': (_i, [_vp, _vp, _vp, _d, _d, _vp, _vp, _i, _vp]),
    'se3tn_track_batch': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _d, _d, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_add_adi': (_i, [_vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    'se3tn_vocap': (_i, [_vp, _vp, _i, C.POINTER(_d), _vp]),
    'se3tn_add_adi_sets': (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    'se3tn_pose_errors_sets': (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    'se3tn_vocap_sets': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    'se3tn_draw_tracks': (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    'se3tn_allgather_poses': (_i, [_vp, _vp, _vp, _vp, _i, _vp]),
    'se3tn_track_host': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _d, _d, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_track_render': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _d, _d, _i, _vp, _vp, _vp, _vp, _vp,
                                _vp]),
    'se3tn_track_render_host': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _d, _d, _i, _vp, _vp, _vp, _vp, _vp,
                                     _vp]),
    'se3tn_draw_hypotheses': (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    'se3tn_init_poses': (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_init_boxes': (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_lost_tracks': (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_fit_poses': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _vp, _vp]),
    'se3tn_accept_starts': (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_fill_depth': (_i, [_vp, _vp, _i, _i, _d, _vp, _vp, _vp]),
    'se3tn_fill_depth_ex': (_i, [_vp, _vp, _i, _i, _d, _i, _i, _vp, _vp, _vp]),
    'se3tn_fit_rows': (_i, [_vp, C.POINTER(_vp)]),
    'se3tn_set_mesh': (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i]),
    'se3tn_render': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    'se3tn_render_ex': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    'se3tn_eval_pairs': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _d, _d, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_pair_loss': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp]),
    'se3tn_eval_pairs_augmented': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _d, _d, _i, _vp, _vp, _vp, _vp, _vp,
                                        _vp, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_augment_draws': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    'se3tn_augment_crops': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    'se3tn_crop_bbox_seg': (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_visibility': (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    'se3tn_perturb_pairs': (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_append_pairs': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp,
                                _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_append_pairs_seg': (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp,
                                    _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'se3tn_debug_buffer': (_i, [_vp, _i, C.POINTER(_vp), C.POINTER(_sz)]),
    'se3tn_last_launch_count': (_i, [_vp]),
    'se3tn_get_trace': (_i, [_vp, _vp]),
    'se3tn_last_step_was_graph': (_i, [_vp]),
    'se3tn_metrics_scratch_bytes': (_sz, [_vp]),
    'se3tn_set_profiling': (_i, [_vp, _i]),
    'se3tn_get_profile': (_i, [_vp, _vp]),
}



class Augment(C.Structure):
    """se3tn_augment (include/se3tn.h)."""
    _fields_ = [('seed', C.c_uint64), ('hsv_jitter', C.c_int32), ('change_bright', C.c_int32), ('gaussian_noise', C.c_int32),
                ('gaussian_blur', C.c_int32), ('black_cover', C.c_int32), ('depth_missing', C.c_int32), ('hsv_prob', _d),
                ('hsv_noise', _d * 3), ('bright_mag', _d * 2), ('noise_prob', _d), ('noise_rgb', _d), ('noise_depth', _d),
                ('blur_prob', _d), ('blur_max_kernel', C.c_int32), ('reserved', C.c_int32), ('cover_prob', _d)]


class HypothesisOpts(C.Structure):
    """se3tn_hypothesis_opts (include/se3tn.h)."""
    _fields_ = [('hypotheses', C.c_int32), ('reserved', C.c_int32), ('seed', C.c_int64), ('max_translation', _d),
                ('max_rotation_deg', _d)]


class IcpOpts(C.Structure):
    """se3tn_icp_opts (include/se3tn.h)."""
    _fields_ = [('iterations', C.c_int32), ('tau_mm', C.c_int32), ('min_inliers', C.c_int32), ('reserved', C.c_int32)]


class TrackOpts(C.Structure):
    """se3tn_track_opts (include/se3tn.h)."""
    _fields_ = [('fill_depth', C.c_int32), ('fill_extrapolate', C.c_int32), ('fill_blur', C.c_int32), ('iterations', C.c_int32),
                ('fill_max_depth', _d), ('fit_tau_mm', C.c_int32), ('reserved', C.c_int32), ('icp', C.POINTER(IcpOpts)),
                ('hyp', C.POINTER(HypothesisOpts))]


class TrackArrays(C.Structure):
    """se3tn_track_arrays (include/se3tn.h): device pointers for se3tn_track_render, host pointers for _render_host."""
    _fields_ = [('draw_keys', _vp), ('round_poses', _vp), ('hyp_poses', _vp), ('icp_poses', _vp), ('out_fit', _vp),
                ('out_choice', _vp), ('out_icp', _vp)]


class InitOpts(C.Structure):
    """se3tn_init_opts (include/se3tn.h)."""
    _fields_ = [('viewpoints', C.c_int32), ('inplane', C.c_int32), ('keep', C.c_int32), ('tau_mm', C.c_int32),
                ('min_pixels', C.c_int32), ('reserved', C.c_int32), ('icp', C.POINTER(IcpOpts))]


class InitArrays(C.Structure):
    """se3tn_init_arrays (include/se3tn.h): device pointers, NULL where not wanted."""
    _fields_ = [('stats', _vp), ('t0', _vp), ('cand_rows', _vp), ('kept_rows', _vp), ('kept_poses', _vp), ('icp_poses', _vp),
                ('icp_rows', _vp), ('icp_stats', _vp)]


class ReinitOpts(C.Structure):
    """se3tn_reinit_opts (include/se3tn.h)."""
    _fields_ = [('below_permille', C.c_int32), ('after', C.c_int32), ('reserved', C.c_int32 * 2)]


_lib = None


def build_library(force=False):
    from . import build as _build
    return _build.build(force=force)


def load():
    """Load (building first if the .so is missing and nvcc exists).  Never falls back to anything:
    a missing library is an error."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        build_library()
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class Se3tnError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__('libse3tn error %d: %s' % (code, msg))
        self.code = code


def check(code, ctx=None):
    if code != OK:
        msg = load().se3tn_last_error(ctx)
        raise Se3tnError(code, msg.decode() if msg else '')
