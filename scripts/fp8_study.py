"""Precision study (CPU, not product code): emulation of the 'fp8' mode's arithmetic (SE3TN_PREC_FP8) against the fp32
oracle, the evidence behind SE3TN_FP8_HEADROOM and the end-to-end tolerance of tests/test_gpu_fp8.py (DESIGN.md section 2).
Run from the repo root:  python scripts/fp8_study.py

Emulated exactly as the mode stores and multiplies: stems fp32-faithful (bf16x3), P1 / T / U stored bf16, the 64-channel
layers on bf16 weights, CAT written e4m3 by its two writers, the six trunk layers on e4m3 codes of the activations (one
power-of-two scale per tensor, per head group for H1 / H2) and of the weights (one per row), every trunk output stored
e4m3, the last layer pooled in fp32.  Scales from a calibration pass like se3tn_calibrate_fp8's (the fp32-faithful forward on
the calibration pairs, s = 2^ceil(log2(max|x| * H / 448))).  Sums are fp32 (torch CPU convs): the reduced-precision
accumulation FP8 wgmma is reported to use is NOT emulated; the per-layer gate bounds it separately.

Cases: config 1 (the shipped pair, weight seed 0); the raw-regime frame of the parity tests (seed 11, 64 tracks, weight
seeds 0 / 1 on 32 tracks each, each set calibrated on its own tracks); and a held-out case -- calibrated on that frame,
evaluated on another one (seed 12) -- which is what a tracker calibrated on its first frame meets later.  H is chosen by
the worst error over all cases."""
import importlib, os, sys, numpy as np, torch, torch.nn.functional as F
sys.path.insert(0, '.'); sys.path.insert(0, 'oracle')
synth = importlib.import_module('iros20-6d-pose-tracking_b200.synth')
import se3_oracle as O
torch.set_num_threads(os.cpu_count() or 8)
GOLDEN = os.path.join('tests', 'golden')
HS = (1, 2, 4, 8)


def pow2_scale(amax):                       # 2^ceil(log2(amax / 448)), 1 for 0 (per element of a tensor of maxima)
    m, e = torch.frexp(amax.double())
    s = torch.ldexp(torch.ones_like(m), (e - 9 + (m > 0.875).to(e.dtype)))
    return torch.where(amax > 0, s, torch.ones_like(s)).float()


def e4m3(x, s):                             # stored code * scale (s broadcast per channel)
    c = (x / s).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).to(torch.float32)
    return c * s


def rn_bf16(x): return x.to(torch.bfloat16).to(torch.float32)


def fold(sd, conv, bn):
    w = sd[conv + '.weight'].double(); b = sd[conv + '.bias'].double()
    g = sd[bn + '.weight'].double(); beta = sd[bn + '.bias'].double(); mu = sd[bn + '.running_mean'].double(); var = sd[bn + '.running_var'].double()
    s = g / torch.sqrt(var + 1e-5)
    return (w * s[:, None, None, None]).float(), ((b - mu) * s + beta).float()


def w8(w):                                  # e4m3 weights with one scale per output row
    s = pow2_scale(w.abs().amax((1, 2, 3)))[:, None, None, None]
    return e4m3(w, s)


def run(sd, A, B, scales=None):
    """scales None: the fp32-faithful calibration pass, -> the 8 tensors' max|x|.  Else the fp8 emulation -> 6-vector."""
    fp8 = scales is not None
    amax = {}
    ch = lambda k: torch.tensor(scales[k])[None, None, None, None] if fp8 else None

    def st(x, name, k=None):                # store a trunk tensor (or CAT): e4m3, or note its max for the calibration
        if not fp8:
            amax[name] = max(amax.get(name, 0.0), float(x.abs().max()))
            return x
        return e4m3(x, ch(k))

    def conv(x, w, b, stride, pad, mode):
        if fp8 and mode == 'bf16':
            w = rn_bf16(w)
        elif fp8 and mode == 'e4m3':
            w = w8(w)
        return F.conv2d(x, w, None, stride=stride, padding=pad) + b[None, :, None, None]

    def store64(x): return rn_bf16(x) if fp8 else x

    def block64(x, p, to_cat=False):
        w1, b1 = fold(sd, p + '.conv1', p + '.bn1'); w2, b2 = fold(sd, p + '.conv2', p + '.bn2')
        t = store64(F.relu(conv(x, w1, b1, 1, 1, 'bf16')))
        y = F.relu(conv(t, w2, b2, 1, 1, 'bf16') + x)
        return y if to_cat else store64(y)

    def stem(x, p):
        w, b = fold(sd, p + '.0', p + '.1')
        return store64(F.max_pool2d(F.selu(conv(x, w, b, 2, 3, 'fp32')), 3, 2, 1))

    a = block64(stem(A, 'convA1'), 'convA2', to_cat=True)
    b = stem(B, 'convB1'); b = block64(b, 'convB2'); b = block64(b, 'convB3', to_cat=True)
    cat = st(torch.cat((a, b), 1), 'CAT', 0)
    w, bb = fold(sd, 'convAB1.0', 'convAB1.1')
    f1 = st(F.selu(conv(cat, w, bb, 2, 1, 'e4m3')), 'F1', 1)
    w1, b1 = fold(sd, 'convAB2.conv1', 'convAB2.bn1'); w2, b2 = fold(sd, 'convAB2.conv2', 'convAB2.bn2')
    t4 = st(F.relu(conv(f1, w1, b1, 1, 1, 'e4m3')), 'T4', 2)
    f2 = st(F.relu(conv(t4, w2, b2, 1, 1, 'e4m3') + f1), 'F2', 3)
    outs = []
    for g, h in enumerate(('trans', 'rot')):
        w, bb = fold(sd, h + '_conv1.0', h + '_conv1.1')
        h1 = st(F.selu(conv(f2, w, bb, 2, 1, 'e4m3')), 'H1.' + h, 4 + g)
        w1, b1 = fold(sd, h + '_conv2.conv1', h + '_conv2.bn1'); w2, b2 = fold(sd, h + '_conv2.conv2', h + '_conv2.bn2')
        h2 = st(F.relu(conv(h1, w1, b1, 1, 1, 'e4m3')), 'H2.' + h, 6 + g)
        h3 = F.relu(conv(h2, w2, b2, 1, 1, 'e4m3') + h1)          # never stored: the fused fp32 pool
        outs.append(torch.tanh(F.linear(h3.mean((2, 3)), sd[h + '_out.0.weight'], sd[h + '_out.0.bias'])))
    if not fp8:
        return [amax[k] for k in ('CAT', 'F1', 'T4', 'F2', 'H1.trans', 'H1.rot', 'H2.trans', 'H2.rot')]
    return torch.cat(outs, 1)


def calibrate(amax, H):
    return [float(pow2_scale(torch.tensor([a * H]))[0]) for a in amax]


def raw_inputs(frame_seed, n, wid, stats):
    rgb, depth = synth.raw_frame(frame_seed); poses = synth.raw_poses(n, seed=frame_seed)
    rgbA, depthA = synth.rendered_views(n, poses, seed=frame_seed)
    As, Bs = [], []
    for i in range(n):
        bb = O.compute_bbox(poses[i], synth.CAMERA_K, 200.0, scale=(1000, 1000, 1000))
        rB, dB = O.crop_bbox(rgb, depth, bb, (176, 176))
        (a, b), _ = O.process_data(rgbA[i], depthA[i], poses[i], rB, dB, np.eye(4), *stats[int(wid[i])])
        As.append(torch.from_numpy(a)); Bs.append(torch.from_numpy(b))
    return torch.stack(As).float(), torch.stack(Bs).float()


def six(sd, A, B):
    r = O.forward(sd, A, B)
    return torch.cat((r['trans'], r['rot']), 1).float()


def main():
    import cv2
    mean, std = synth.default_mean_std()
    stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    sds = {0: synth.make_state_dict(0), 1: synth.make_state_dict(1)}
    cases = []                              # (name, set, A, B, calibration A, calibration B)
    rgbA = cv2.imread(os.path.join(GOLDEN, 'c1_rgbA.png'))[..., ::-1].copy()
    rgbB = cv2.imread(os.path.join(GOLDEN, 'c1_rgbB.png'))[..., ::-1].copy()
    (a, b), _ = O.process_data(rgbA, synth.depth_from_rgb(rgbA), synth.config1_pose(), rgbB, synth.depth_from_rgb(rgbB), np.eye(4), mean, std)
    A1, B1 = torch.from_numpy(a)[None].float(), torch.from_numpy(b)[None].float()
    cases.append(('config 1', 0, A1, B1, A1, B1))
    n = 64
    wid = np.repeat([0, 1], n // 2)
    A, B = raw_inputs(11, n, wid, stats)
    A2, B2 = raw_inputs(12, 16, np.zeros(16, int), stats)
    for w in (0, 1):
        sel = torch.from_numpy(np.flatnonzero(wid == w))
        cases.append(('raw n=64, set %d' % w, w, A[sel], B[sel], A[sel], B[sel]))
    cases.append(('held out, set 0', 0, A2, B2, A[:n // 2], B[:n // 2]))
    worst = {H: 0.0 for H in HS}
    with torch.no_grad():
        for name, w, Ae, Be, Ac, Bc in cases:
            ref = six(sds[w], Ae, Be)
            amax = run(sds[w], Ac, Bc)
            for H in HS:
                err = float((run(sds[w], Ae, Be, calibrate(amax, H)) - ref).abs().max())
                worst[H] = max(worst[H], err)
                print('%-18s H = %d: max |err| of the 6-vector %.4g' % (name, H, err), flush=True)
    best = min(HS, key=lambda H: worst[H])
    print('worst over all cases:', ', '.join('H = %d: %.4g' % (H, worst[H]) for H in HS), '-> H = %d' % best)


if __name__ == '__main__':
    main()
