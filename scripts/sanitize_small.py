"""Small invocation of every kernel family for compute-sanitizer (memcheck / racecheck)."""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
pkg = importlib.import_module('iros20-6d-pose-tracking_b200'); synth = pkg.synth
n = 3
eng = pkg.Engine(max_batch=4)
mean, std = synth.default_mean_std()
for wid in (0, 1):
    eng.load_state_dict(synth.make_state_dict(wid), wid); eng.set_stats(mean, std, wid)
eng.set_mesh(synth.mesh(2, seed=0), 0); eng.set_mesh(synth.mesh(0, seed=1), 1)
K = synth.CAMERA_K
rgb, depth = synth.raw_frame(0)
poses = torch.from_numpy(synth.raw_poses(n, seed=0)).cuda(); ow = torch.full((n,), 200.0, dtype=torch.float64, device='cuda')
ids = torch.tensor([0, 1, 0], dtype=torch.int32, device='cuda')
rgbA, depA = eng.render(K, poses, ow, ids)
rgbP, depP = eng.render(K, poses, ow, ids, mode='pyrender', image_hw=(480, 640))
R, D = torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda()
for prec in ('bf16x3', 'tf32', 'bf16', 'fp32'):
    out, _, _ = eng.track_batch(R, D, K, poses, ow, rgbA, depA, 0.03, 5 * np.pi / 180, weight_ids_host=np.array([0, 1, 0], np.int32) if prec != 'fp32' else None, precision=prec)
host = eng.track_host(rgb, depth, K, poses.cpu().numpy(), ow.cpu().numpy(), rgbA.cpu().numpy(), depA.cpu().numpy(), 0.03, 5 * np.pi / 180, weight_ids=np.array([0, 1, 0], np.int32))
for mode, hw in (('vispy', None), ('pyrender', (480, 640))):
    for prec in ('bf16x3', 'fp32'):
        eng.track_render(R, D, K, poses, ow, 0.03, 5 * np.pi / 180, weight_ids_host=np.array([0, 1, 0], np.int32), precision=prec, mode=mode, image_hw=hw)
    eng.track_render_host(rgb, depth, K, poses.cpu().numpy(), ow.cpu().numpy(), 0.03, 5 * np.pi / 180, weight_ids=np.array([0, 1, 0], np.int32), mode=mode, image_hw=hw)
filled = eng.fill_depth(D[:96, :128].contiguous())
# the calls above (n = 3) run the trunk's split-K latency mode; n = 6 runs its throughput mode
eng6 = pkg.Engine(max_batch=6); eng6.load_state_dict(synth.make_state_dict(0), 0)
A6, B6 = synth.tensor_pairs(6, seed=2); A6 = A6.cuda(); B6 = B6.cuda()
for prec in ('bf16x3', 'tf32', 'bf16'):
    eng6.forward(A6, B6, precision=prec)
# the resident launches run ping-pong where a CTA has more than one tile: the stems already do at n = 3 and 6, the 64-channel
# layers (16 tiles per image) only from n = 9 on
eng20 = pkg.Engine(max_batch=20); eng20.load_state_dict(synth.make_state_dict(0), 0)
A20, B20 = synth.tensor_pairs(20, seed=3); A20 = A20.cuda(); B20 = B20.cuda()
for prec in ('bf16x3', 'tf32', 'bf16'):
    eng20.forward(A20, B20, precision=prec)
m = torch.from_numpy(synth.model_points(500, 0)).cuda(); pr, gt = synth.pose_pairs(4, 0)
add, adi = eng.add_adi(m, torch.from_numpy(pr).cuda(), torch.from_numpy(gt).cuda()); ap = eng.vocap(adi)
torch.cuda.synchronize()
print('ok', float(out.abs().sum()), int(filled.to(torch.int32).sum()), ap)
