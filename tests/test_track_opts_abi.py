"""CPU-only: se3tn_track_opts and se3tn_track_arrays in include/se3tn.h and _lib.TrackOpts / _lib.TrackArrays agree field for
field, the four tracking calls are declared and bound with the options (and the render calls the arrays) in the same place, and
the per-extra calls the options replaced are gone."""
import ctypes as C, importlib, os, re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = 'iros20-6d-pose-tracking_b200'
SCALARS = {'int32_t': C.c_int32, 'double': C.c_double}


def _header():
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)


def _fields(name):
    """(name, C type) of each member of struct `name`; a pointer member maps to what _lib binds it as."""
    m = re.search(r'\bstruct\s+%s\s*\{([^}]*)\}' % name, _header())
    assert m, 'struct %s is not defined' % name
    L = importlib.import_module(PKG + '._lib')
    pointees = {'se3tn_icp_opts': C.POINTER(L.IcpOpts), 'se3tn_hypothesis_opts': C.POINTER(L.HypothesisOpts)}
    fields = []
    for decl in filter(None, (' '.join(d.split()) for d in m.group(1).split(';'))):
        typ, names = re.match(r'((?:const )?\w+\s*\*?)\s*(.*)', decl).groups()
        typ = typ.replace(' ', '')
        for f in names.split(','):
            if typ.endswith('*'):
                base = typ.replace('const', '').rstrip('*')
                fields.append((f.strip(), pointees.get(base, L._vp)))
            else:
                fields.append((f.strip(), SCALARS[typ]))
    return fields


def test_track_opts_matches_the_header():
    L = importlib.import_module(PKG + '._lib')
    fields = _fields('se3tn_track_opts')
    assert L.TrackOpts._fields_ == fields
    assert C.sizeof(L.TrackOpts) == 48
    assert [f[0] for f in fields] == ['fill_depth', 'fill_extrapolate', 'fill_blur', 'iterations', 'fill_max_depth', 'fit_tau_mm',
                                      'reserved', 'icp', 'hyp']


def test_track_arrays_match_the_header():
    L = importlib.import_module(PKG + '._lib')
    fields = _fields('se3tn_track_arrays')
    assert L.TrackArrays._fields_ == fields
    assert [f[0] for f in fields] == ['draw_keys', 'round_poses', 'hyp_poses', 'icp_poses', 'out_fit', 'out_choice', 'out_icp']
    assert C.sizeof(L.TrackArrays) == 7 * C.sizeof(C.c_void_p)


def test_tracking_calls_take_opts():
    src = _header()
    L = importlib.import_module(PKG + '._lib')
    # the options come after the outputs; the render calls then take the arrays, and the stream is always last
    for name, tail in (('se3tn_track_batch', ['const se3tn_track_opts* opts']),
                       ('se3tn_track_host', ['const se3tn_track_opts* opts']),
                       ('se3tn_track_render', ['const se3tn_track_opts* opts', 'const se3tn_track_arrays* arrays']),
                       ('se3tn_track_render_host', ['const se3tn_track_opts* opts', 'const se3tn_track_arrays* arrays'])):
        m = re.search(r'\bint\s+%s\s*\(([^)]*)\)\s*;' % name, src)
        assert m, name + ' is not declared'
        params = [' '.join(p.split()) for p in m.group(1).split(',')]
        assert params[-len(tail) - 1:] == tail + ['void* stream'], name
        res, args = L.SIGNATURES[name]
        assert res is L._i and len(args) == len(params) and all(a is L._vp for a in args[-len(tail) - 1:]), name


def test_per_extra_calls_are_gone():
    src = open(os.path.join(ROOT, 'include', 'se3tn.h')).read()
    L = importlib.import_module(PKG + '._lib')
    for name in ('se3tn_track_icp', 'se3tn_track_icp_host', 'se3tn_track_hypotheses', 'se3tn_track_hypotheses_host'):
        assert not re.search(r'\b%s\b' % name, src), name
        assert name not in L.SIGNATURES, name
    assert sorted(n for n in L.SIGNATURES if n.startswith('se3tn_track_')) == [
        'se3tn_track_batch', 'se3tn_track_host', 'se3tn_track_render', 'se3tn_track_render_host']
