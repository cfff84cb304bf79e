"""CPU-only: se3tn_track_opts in include/se3tn.h and _lib.TrackOpts agree field for field, and every tracking call is declared and
bound with the options pointer in the same place."""
import ctypes as C, importlib, os, re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CTYPES = {'int32_t': C.c_int32, 'double': C.c_double}


def _header():
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)


def test_track_opts_matches_the_header():
    m = re.search(r'\bstruct\s+se3tn_track_opts\s*\{([^}]*)\}\s*;', _header())
    assert m, 'struct se3tn_track_opts is not defined'
    fields = []
    for decl in filter(None, (d.strip() for d in m.group(1).split(';'))):
        typ, names = decl.split(None, 1)
        fields += [(name.strip(), CTYPES[typ]) for name in names.split(',')]
    L = importlib.import_module('iros20-6d-pose-tracking_b200._lib')
    assert L.TrackOpts._fields_ == fields
    assert C.sizeof(L.TrackOpts) == 32
    assert [f[0] for f in fields] == ['fill_depth', 'fill_extrapolate', 'fill_blur', 'iterations', 'fill_max_depth', 'fit_tau_mm',
                                      'reserved']


def test_tracking_calls_take_opts():
    src = _header()
    L = importlib.import_module('iros20-6d-pose-tracking_b200._lib')
    # the options come after the outputs; the render calls then take round_poses / out_fit, and the stream is always last
    for name, after in (('se3tn_track_batch', 1), ('se3tn_track_host', 1), ('se3tn_track_render', 2), ('se3tn_track_render_host', 2)):
        m = re.search(r'\bint\s+%s\s*\(([^)]*)\)\s*;' % name, src)
        assert m, name + ' is not declared'
        params = [' '.join(p.split()) for p in m.group(1).split(',')]
        assert params[-after - 1] == 'const se3tn_track_opts* opts', name
        assert params[-1] == 'void* stream', name
        res, args = L.SIGNATURES[name]
        assert res is L._i and len(args) == len(params) and args[-after - 1] is L._vp, name
