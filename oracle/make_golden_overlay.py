#!/usr/bin/env python
"""Generate tests/golden/golden_overlay.npz by running the reference's own project_points (predict.py:81-86) where the
reference exists; the drawing around it is the reference's cv2 lines as oracle/overlay_oracle.py restates them.

  python oracle/make_golden_overlay.py [--ref /root/reference]

The reference's predict.py is loaded as a module: its top level only imports and defines.  The imports it needs for tracking,
rendering and plotting (open3d, transformations, offscreen_renderer, vispy_renderer, matplotlib, mpl_toolkits) are stubbed
when they are not installed, as make_golden.py stubs open3d and transformations for Utils.py.  Nothing in the reference tree is
edited.  Inputs come from the product's deterministic generators (synth.py) and are stored in the fixture.
"""
import argparse, importlib, importlib.util, os, sys, types
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.dont_write_bytecode = True
synth = importlib.import_module('iros20-6d-pose-tracking_b200.synth')
import make_golden                                                    # noqa: E402
import overlay_oracle as OV                                           # noqa: E402


def reference_project_points(ref):
    """project_points of the reference's predict.py, loaded with the imports it does not need here stubbed."""
    make_golden.import_reference(ref)
    for name in ('offscreen_renderer', 'vispy_renderer', 'matplotlib', 'matplotlib.pyplot',
                 'mpl_toolkits', 'mpl_toolkits.mplot3d', 'mpl_toolkits.mplot3d.axes3d'):
        try:
            importlib.import_module(name)
        except ImportError:
            sys.modules[name] = types.ModuleType(name)
    sys.modules['vispy_renderer'].VispyRenderer = getattr(sys.modules['vispy_renderer'], 'VispyRenderer', object)
    sys.modules['mpl_toolkits.mplot3d'].axes3d = sys.modules['mpl_toolkits.mplot3d.axes3d']
    sys.modules['mpl_toolkits'].mplot3d = sys.modules['mpl_toolkits.mplot3d']
    sys.modules['matplotlib'].pyplot = sys.modules['matplotlib.pyplot']
    scripts = os.path.join(ref, 'scripts')
    if scripts not in sys.path:
        sys.path.insert(0, scripts)
    spec = importlib.util.spec_from_file_location('reference_predict', os.path.join(ref, 'predict.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.project_points


def overlay_golden(ref, out):
    """Frames drawn as the reference's result videos draw them, on points the reference's own project_points places (moved by
    the pose in the order oracle/overlay_oracle.py states), in both label orders."""
    project_points = reference_project_points(ref)
    rng = np.random.default_rng(5)
    K = synth.CAMERA_K
    ov = {'K': K}
    for c, (H, W, text) in enumerate(((480, 640, 'frame:1'), (480, 640, 'frame:9999999'), (96, 128, 'frame:42'))):
        frame = np.kron(rng.integers(0, 256, (H // 16, W // 16, 3)), np.ones((16, 16, 1))).astype(np.uint8)   # compresses well
        frame[rng.random((H, W)) < 0.002] = 255                      # saturated pixels
        Kc = K.copy(); Kc[0, 2] = K[0, 2] * W / 640; Kc[1, 2] = K[1, 2] * H / 480
        pts = synth.mesh(3, seed=c)['pos'].astype(np.float64)
        pose = synth.raw_poses(1, seed=40 + c)[0]
        # the object's centre over the label (W/2 + 60, H - 60) in case 1, near the frame's edges in the others
        u, v = [(W - 20, 30), (W // 2 + 60, H - 60), (10, H - 10)][c]
        z = pose[2, 3]
        pose[0, 3], pose[1, 3] = (u - Kc[0, 2]) * z / Kc[0, 0], (v - Kc[1, 2]) * z / Kc[1, 1]
        uvs = project_points(OV.transform(pts, pose), Kc)
        ov['frame_%d' % c], ov['K_%d' % c], ov['pose_%d' % c], ov['points_%d' % c] = frame, Kc, pose, pts
        ov['text_%d' % c] = np.array(text)
        for order in ('under', 'over'):
            ov['out_%d_%s' % (c, order)] = OV.draw(frame, uvs, text, order)
    np.savez_compressed(os.path.join(out, 'golden_overlay.npz'), **ov)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ref', default='/root/reference')
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden'))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    overlay_golden(args.ref, args.out)
    print('golden_overlay.npz', os.path.getsize(os.path.join(args.out, 'golden_overlay.npz')))


if __name__ == '__main__':
    main()
