"""CPU-only: the in-step depth fill's setter is declared in include/se3tn.h and bound by _lib.py with the same arguments."""
import importlib, os, re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_set_depth_fill_declared_and_bound():
    src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'se3tn.h')).read(), flags=re.S)
    m = re.search(r'\bint\s+se3tn_set_depth_fill\s*\(([^)]*)\)\s*;', src)
    assert m, 'se3tn_set_depth_fill is not declared'
    params = [p.strip() for p in m.group(1).split(',')]
    assert [p.split()[0] for p in params] == ['se3tn_ctx*', 'int', 'double', 'int', 'int']
    L = importlib.import_module('iros20-6d-pose-tracking_b200._lib')
    res, args = L.SIGNATURES['se3tn_set_depth_fill']
    assert res is L._i and len(args) == len(params)
    assert args == [L._vp, L._i, L._d, L._i, L._i]
