"""GPU bring-up diagnostic (not a test): runs each piece against the oracle and prints where
things diverge.  python scripts/first_light.py [N]
The per-layer check with bounds derived from each mode's arithmetic is tests/test_gpu_layers.py."""
import importlib, os, sys, time, traceback
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
pkg = importlib.import_module('iros20-6d-pose-tracking_b200')
synth = pkg.synth
import se3_oracle as O
import layer_ref as R

BUFS = ['X0A','X0B','Y1A','Y1B','P1A','P1B','T1','T2','U','CAT','F1','T4','F2','H1','H2','H3']
N = int(sys.argv[1]) if len(sys.argv) > 1 else 2
MODE = sys.argv[2] if len(sys.argv) > 2 else 'all'   # 'base' = everything but the tensor-core convs, 'tc' = tensor-core convs only
dev = torch.device('cuda:0')
print(torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0))
eng = pkg.Engine(max_batch=max(N, 64))
print('engine created (all tensor maps encoded)')
sd = synth.make_state_dict(0)
eng.load_state_dict(sd, 0)
A, B = synth.tensor_pairs(N, seed=0)
ref, inter = O.forward(sd, A, B, return_intermediates=True)
ref6 = torch.cat((ref['trans'], ref['rot']), 1)
Ad, Bd = A.to(dev), B.to(dev)

def report(tag, trans, rot):
    out = torch.cat((trans, rot), 1).cpu()
    err = (out - ref6).abs(); tol = 1e-4 + 1e-3 * ref6.abs()
    print('%s: max abs err %.3e  max err/tol %.3f  finite=%s' % (tag, err.max().item(), (err / tol).max().item(), bool(torch.isfinite(out).all())))
    return out

snap = {}
try:
    t, r, f = eng.forward(Ad, Bd, precision='fp32', want_feature=True)
    torch.cuda.synchronize()
    report('fp32 direct path vs oracle', t, r)
    print('  feature max abs err %.3e' % (f.cpu() - ref['feature']).abs().max().item())
    for i, name in enumerate(BUFS):
        snap[name] = eng.debug_buffer(i, N).clone()
    # NHWC buffer vs oracle NCHW intermediates
    def cmp(buf, ref_t, C, HW, coff=0, cs=None):
        cs = cs or C
        x = snap[buf].view(N, HW, cs)[:, :, coff:coff + C].permute(0, 2, 1).reshape(ref_t.shape).cpu()
        return (x - ref_t).abs().max().item()
    print('  Y1A', cmp('Y1A', inter['a1'], 64, 88 * 88), 'P1A', cmp('P1A', inter['a1p'], 64, 44 * 44),
          'CAT.a', cmp('CAT', inter['a2'], 64, 44 * 44, 0, 128), 'CAT.b', cmp('CAT', inter['b3'], 64, 44 * 44, 64, 128),
          'F1', cmp('F1', inter['ab1'], 256, 484), 'F2', cmp('F2', inter['ab2'], 256, 484),
          'H1.t', cmp('H1', inter['trans1'], 512, 121, 0, 1024), 'H1.r', cmp('H1', inter['rot1'], 512, 121, 512, 1024),
          'H3.t', cmp('H3', inter['trans2'], 512, 121, 0, 1024), 'H3.r', cmp('H3', inter['rot2'], 512, 121, 512, 1024))
except Exception:
    traceback.print_exc()

def decoded(name, prec):
    """Buffer `name` of the N images as float32 NCHW, through the storage-format decoders of oracle/layer_ref.py."""
    fmt = R.buf_format(name, prec)
    nb = R.image_bytes(name, fmt)
    raw = eng.debug_buffer(R.BUF_ID[name], N).view(torch.uint8).reshape(-1)[:N * nb].cpu().numpy()
    return np.stack([R.decode(raw[i * nb:(i + 1) * nb], name, fmt).value for i in range(N)])


try:
    if MODE == 'base': raise SystemExit
    ref_bufs = {name: decoded(name, 'fp32') for name in snap}
    for prec in ('tf32', 'bf16x3', 'bf16'):
        t, r, f = eng.forward(Ad, Bd, precision=prec, want_feature=True)
        torch.cuda.synchronize()
        report('%s wgmma path vs oracle' % prec, t, r)
        for name in snap:
            if name in ('Y1A', 'Y1B', 'H3'):       # the tensor-core modes pool in the stems' and the last layer's epilogues
                continue
            cur = decoded(name, prec)
            d = np.abs(cur - ref_bufs[name])
            scale = np.abs(ref_bufs[name]).max() + 1e-30
            bad = (d > 0.02 * scale).mean()
            print('  %-4s %s-vs-fp32: max abs diff %.3e (scale %.3e) frac>2%%: %.4f nan=%d' % (name, prec, np.nanmax(d), scale, bad, int(np.isnan(cur).sum())))
    print('launches per forward:', eng.last_launch_count())
except SystemExit:
    pass
except Exception:
    traceback.print_exc()

# ---- preprocessing + pose update vs oracle
try:
    n = 6
    rgb, depth = synth.raw_frame(0)
    poses = synth.raw_poses(n, seed=0)
    poses[1, :3, 3] = (-0.13, -0.1, 0.5)          # clipped window
    rgbA, depthA = synth.rendered_views(n, poses, seed=2)
    mean, std = synth.default_mean_std()
    eng.set_stats(mean, std, 0)
    ow = np.full(n, 200.0)
    tA, tB, crgb, cdepth = eng.preprocess(torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev), synth.CAMERA_K,
                                          torch.from_numpy(poses).to(dev), torch.from_numpy(ow).to(dev),
                                          torch.from_numpy(rgbA).to(dev), torch.from_numpy(depthA).to(dev),
                                          want_tensors=True, want_crops=True)
    torch.cuda.synchronize()
    for i in range(n):
        bb = O.compute_bbox(poses[i], synth.CAMERA_K, 200.0, scale=(1000, 1000, 1000))
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        (dA_, dB_), _ = O.process_data(rgbA[i], depthA[i], poses[i], rB, dB, np.eye(4), mean, std)
        print('  track %d crop rgb equal %s depth equal %s dataA equal %s dataB equal %s (maxdiff %.3e)' % (
            i, np.array_equal(crgb[i].cpu().numpy(), rB), np.array_equal(cdepth[i].cpu().numpy(), dB),
            np.array_equal(tA[i].cpu().numpy(), dA_), np.array_equal(tB[i].cpu().numpy(), dB_),
            np.abs(tB[i].cpu().numpy() - dB_).max()))
    rng = np.random.default_rng(0)
    tr = rng.uniform(-1, 1, (n, 3)).astype(np.float32); ro = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    out = eng.pose_update(torch.from_numpy(poses).to(dev), torch.from_numpy(tr).to(dev), torch.from_numpy(ro).to(dev), 0.03, 5 * np.pi / 180)
    refp = np.stack([O.process_predict(poses[i], (tr[i], ro[i])) for i in range(n)])
    print('  pose update max abs diff %.3e' % np.abs(out.cpu().numpy() - refp).max())
    gtB = synth.raw_poses(n, seed=3); gtB[:, :3, 3] = poses[:, :3, 3] + 0.01
    tl, rl = eng.so3_log(torch.from_numpy(poses).to(dev), torch.from_numpy(gtB).to(dev), 0.03, 5 * np.pi / 180)
    labs = [O.process_data(rgbA[i], depthA[i], poses[i], rgbA[i], depthA[i], gtB[i], mean, std)[1] for i in range(n)]
    print('  so3 log max abs diff trans %.3e rot %.3e' % (np.abs(tl.cpu().numpy() - np.stack([l[0] for l in labs])).max(),
                                                         np.abs(rl.cpu().numpy() - np.stack([l[1] for l in labs])).max()))
except Exception:
    traceback.print_exc()

# ---- timing
try:
    for prec in (('fp32',) if MODE == 'base' else ('tf32',) if MODE == 'tc' else ('tf32', 'fp32')):
        for nb in (1, 64):
            A2, B2 = synth.tensor_pairs(nb, seed=1); A2 = A2.to(dev); B2 = B2.to(dev)
            for _ in range(3): eng.forward(A2, B2, precision=prec)
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            iters = 10 if prec == 'tf32' else 3
            e0.record()
            for _ in range(iters): eng.forward(A2, B2, precision=prec)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            print('  %s N=%d: %.3f ms/forward  %.1f pairs/s  %.1f TFLOP/s' % (prec, nb, ms, nb / ms * 1e3, nb * 5.527e9 / ms / 1e9))
except Exception:
    traceback.print_exc()
print('done')
