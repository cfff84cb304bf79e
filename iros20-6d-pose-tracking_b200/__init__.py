"""H100-native se(3)-TrackNet inference hot path (Tracker.on_track of
wenbowen123/iros20-6d-pose-tracking): hand-written sm_90a CUDA behind a C ABI (libse3tn.so),
with a Python host layer that mirrors the reference's class surface.

    from <this package> import Se3TrackNet, Tracker, TrackDataset, Engine

Importing the package does not touch CUDA; constructing an Engine (directly or through the
drop-in classes) requires an H100 and the built library -- there is no fallback path.
"""
from .engine import Engine            # noqa: F401
from . import synth                   # noqa: F401


def __getattr__(name):                # lazy: the drop-in modules import cv2/yaml-free code only when used
    if name == 'Se3TrackNet':
        from .se3_tracknet import Se3TrackNet
        return Se3TrackNet
    if name == 'Tracker':
        from .predict import Tracker
        return Tracker
    if name == 'TrackDataset':
        from .datasets import TrackDataset
        return TrackDataset
    raise AttributeError(name)
