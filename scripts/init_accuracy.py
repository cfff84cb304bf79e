"""How close Engine.init_poses' and Engine.init_boxes' starts land, with their defaults, on synthetic frames: 8 scenes of
oracle/init_ref.py's labelled_scene (8 objects each at random rotations, 64 poses) in front of init_box_ref.with_background's
tilted plane (1.1 to 1.3 m wherever the scene has no depth, so every box holds background depth), each drawn as it is and with
a partial occlusion (the left 30 % of every mask's columns covered by a flat occluder 100 mm in front of the object, which takes
those pixels' label away).  Each variant is started from the masks, and from each object's full tight box (the occluder lies
inside it) at D = 1 and at Engine.INIT_BOX_DEPTHS depths.  Rows:
`grid` the top grid candidate (kept pose 0), `icp` the returned pose, `best of K` the refined candidate of lowest ADD-S (the
bound any final choice can reach).  Prints the card's name and power limit read in the same run, then per variant and row
the mean / median ADD-S (mm) and rotation error (degrees) over the poses, and how many of them have ADD-S below 10 mm.

    python scripts/init_accuracy.py [--scenes 8]"""
import argparse, importlib, itertools, os, subprocess, sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import init_box_ref  # noqa: E402
import init_ref  # noqa: E402
import se3_oracle as so  # noqa: E402
PKG = 'iros20-6d-pose-tracking_b200'


def occlude(depth, seg, n):
    depth, seg = depth.copy(), seg.copy()
    for k in range(1, n + 1):
        v, u = np.nonzero(seg == k)
        if len(u) == 0:
            continue
        cut = u.min() + 0.3 * (u.max() - u.min())
        sel = u <= cut
        front = np.maximum(depth[v[sel], u[sel]].astype(np.int64) - 100, 1)
        depth[v[sel], u[sel]] = front.astype(np.uint16)
        seg[v[sel], u[sel]] = 0
    return depth, seg


def rot_err(P, Q):
    c = (np.trace(P[:3, :3].T @ Q[:3, :3]) - 1) / 2
    return np.degrees(np.arccos(np.clip(c, -1, 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenes', type=int, default=8)
    args = ap.parse_args()
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip())
    pkg = importlib.import_module(PKG)
    synth = pkg.synth
    K = synth.CAMERA_K
    e = pkg.Engine(max_batch=64)
    e.set_mesh(synth.mesh(), 0)
    spec = e.init_spec()
    Kk = spec.keep
    starts = ('mask', 'box D=1', 'box D=%d' % e.INIT_BOX_DEPTHS)
    variants = [(v, st) for v in ('full', 'occluded') for st in starts]
    res = {v: {r: ([], []) for r in ('grid', 'icp', 'best of K')} for v in variants}
    failed = {v: 0 for v in variants}
    for s in range(args.scenes):
        mesh, gts, _, D, seg = init_ref.labelled_scene(synth, 8, seed=100 + s)
        pts = mesh['pos'].astype(np.float64)
        boxes = np.stack([init_box_ref.tight_box(seg, k) for k in range(1, 9)])      # the full boxes, before any occlusion
        occluded = occlude(D, seg, 8)
        for (variant, (d, m)), st in itertools.product((('full', (D, seg)), ('occluded', occluded)), starts):
            d = init_box_ref.with_background(d, K)
            n = 8
            out = dict(kept_poses=torch.empty(n, Kk, 4, 4, dtype=torch.float64, device=e.device),
                       icp_poses=torch.empty(n, Kk, 4, 4, dtype=torch.float64, device=e.device))
            ow = torch.full((n,), 200.0, dtype=torch.float64, device=e.device)
            if st == 'mask':
                P, R = e.init_poses(torch.from_numpy(d).cuda(), torch.from_numpy(m).cuda(), K, list(range(1, n + 1)), ow, out=out)
            else:
                P, R = e.init_boxes(torch.from_numpy(d).cuda(), boxes, K, ow, depths=int(st.split('=')[1]), out=out)
            P, R = P.cpu().numpy(), R.cpu().numpy()
            kp, ip = out['kept_poses'].cpu().numpy(), out['icp_poses'].cpu().numpy()
            key = (variant, st)
            for i in range(n):
                if R[i, 0] != 0:
                    failed[key] += 1
                    continue
                adds = [so.adi(ip[i, k], gts[i], pts) * 1000 for k in range(Kk)]
                for row, pose in (('grid', kp[i, 0]), ('icp', P[i]), ('best of K', ip[i, int(np.argmin(adds))])):
                    res[key][row][0].append(so.adi(pose, gts[i], pts) * 1000)
                    res[key][row][1].append(rot_err(pose, gts[i]))
    for variant, rows in res.items():
        print('%s, %s (%d poses, %d failed)' % (variant[0], variant[1], len(rows['icp'][0]), failed[variant]))
        print('| row | ADD-S mean / median, mm | rotation mean / median, degrees | ADD-S < 10 mm |')
        print('|---|---|---|---|')
        for row, (a, r) in rows.items():
            a, r = np.array(a), np.array(r)
            print('| %s | %.1f / %.1f | %.1f / %.1f | %d / %d |' % (row, a.mean(), np.median(a), r.mean(), np.median(r), (a < 10).sum(), len(a)))
    e.close()


if __name__ == '__main__':
    main()
