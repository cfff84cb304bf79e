"""The Python binding sizes Engine.get_trace / get_tile_trace from the same trace layout the C header defines."""
import os
import re


def test_trace_words_match_header(pkg):
    from importlib import import_module
    L = import_module(pkg.__name__ + '._lib')
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'se3tn.h')).read()
    assert int(re.search(r'#define SE3TN_TRACE_TILES\s+(\d+)', src).group(1)) == L.TRACE_TILES
    assert re.search(r'#define SE3TN_TRACE_WORDS\s+\(14 \* 256 \* 8 \+ 8 \* SE3TN_TRACE_TILES \* 4\)', src)
