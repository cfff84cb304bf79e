"""Precision study (CPU, not product code): exact emulation of TF32 / 3-product operand rounding per layer group on the
raw-regime inputs, against the fp32 oracle -- the evidence behind the bf16x3 default (DESIGN.md section 2).  Run from the repo root.
    python scripts/precision_raw.py          the per-layer-group study (6 tracks of frame seed 6)
    python scripts/precision_raw.py --fp16   the fp16 mode (precision_study.run_fp16) on the 64 tracks of frame seed 11, half on
                                             each weight seed, as tests/test_gpu_fp16.py runs them"""
import importlib, sys, numpy as np, torch, torch.nn.functional as F
sys.path.insert(0,'.'); sys.path.insert(0,'oracle')
synth = importlib.import_module('iros20-6d-pose-tracking_b200.synth')
import se3_oracle as O
torch.set_num_threads(8)
def rna_tf32(x):
    i = x.contiguous().view(torch.int32); i = (i + 0x1000) & ~0x1FFF; return i.view(torch.float32)
def ident(x): return x
def fold(sd, conv, bn):
    w = sd[conv+'.weight'].double(); b = sd[conv+'.bias'].double()
    g = sd[bn+'.weight'].double(); beta = sd[bn+'.bias'].double(); mu = sd[bn+'.running_mean'].double(); var = sd[bn+'.running_var'].double()
    s = g/torch.sqrt(var+1e-5)
    return (w*s[:,None,None,None]).float(), ((b-mu)*s+beta).float()
def split3(x):
    hi = rna_tf32(x); lo = rna_tf32(x - hi); return hi, lo
def run(sd, A, B, modes):
    # modes: dict layer-group -> 'tf32' | 'fp32' | '3x' ; store rounding always tf32 unless group mode fp32
    def conv(x, w, b, stride, pad, grp):
        m = modes.get(grp, 'tf32')
        if m == 'tf32':
            y = F.conv2d(rna_tf32(x).double(), rna_tf32(w).double(), None, stride=stride, padding=pad).float()
        elif m == '3x':
            xh, xl = split3(x); wh, wl = split3(w)
            y = (F.conv2d(xh.double(), wh.double(), None, stride=stride, padding=pad) + F.conv2d(xl.double(), wh.double(), None, stride=stride, padding=pad)
                 + F.conv2d(xh.double(), wl.double(), None, stride=stride, padding=pad)).float()
        else:
            y = F.conv2d(x.double(), w.double(), None, stride=stride, padding=pad).float()
        return y + b[None,:,None,None]
    def st(x, grp):   # storage rounding
        return x if modes.get(grp+'_store', modes.get(grp,'tf32')) in ('fp32','3x') else rna_tf32(x)
    def cbr(x, p, stride, pad, grp):
        w,b = fold(sd, p+'.0', p+'.1'); return st(F.selu(conv(x,w,b,stride,pad,grp)), grp)
    def block(x, p, grp):
        w1,b1 = fold(sd,p+'.conv1',p+'.bn1'); w2,b2 = fold(sd,p+'.conv2',p+'.bn2')
        t = st(F.relu(conv(x,w1,b1,1,1,grp)), grp)
        return st(F.relu(conv(t,w2,b2,1,1,grp)+x), grp)
    a = cbr(st(A,'stem'),'convA1',2,3,'stem'); a = F.max_pool2d(a,3,2,1); a = block(a,'convA2','c64')
    b = cbr(st(B,'stem'),'convB1',2,3,'stem'); b = F.max_pool2d(b,3,2,1); b = block(b,'convB2','c64'); b = block(b,'convB3','c64')
    ab = torch.cat((a,b),1); ab = cbr(ab,'convAB1',2,1,'ab'); ab = block(ab,'convAB2','ab')
    outs=[]
    for h in ('trans','rot'):
        x = cbr(ab,h+'_conv1',2,1,'head'); x = block(x,h+'_conv2','head')
        x = x.mean((2,3)); outs.append(torch.tanh(F.linear(x, sd[h+'_out.0.weight'], sd[h+'_out.0.bias'])))
    return torch.cat(outs,1)

def fp16_raw(n=64, seed=11):
    from precision_study import run_fp16
    rgb, depth = synth.raw_frame(seed); poses = synth.raw_poses(n, seed=seed); rgbA, depthA = synth.rendered_views(n, poses, seed=seed)
    mean, std = synth.default_mean_std(); stats = {0: (mean, std), 1: (mean + 1.5, std * 1.25)}
    wid = np.repeat([0, 1], n // 2)
    for w in (0, 1):
        sd = synth.make_state_dict(w); sel = np.nonzero(wid == w)[0]
        ds = [O.on_track(sd, poses[i], rgb, depth, rgbA[i], depthA[i], synth.CAMERA_K, 200.0, *stats[w], return_all=True)[1] for i in sel]
        A = torch.from_numpy(np.stack([d['dataA'] for d in ds])).float(); B = torch.from_numpy(np.stack([d['dataB'] for d in ds])).float()
        ref = torch.from_numpy(np.stack([np.concatenate([d['trans'], d['rot']]) for d in ds]))
        with torch.no_grad(): out = run_fp16(sd, A, B)
        err = (out.double() - ref).abs(); tol = 1e-4 + 1e-3 * ref.abs()
        print('fp16, raw regime, weight seed %d (%d tracks): max abs err %.3e  max err/tol %.3f  input absmax %.1f'
              % (w, len(sel), err.max().item(), (err / tol).max().item(), max(A.abs().max().item(), B.abs().max().item())))

if '--fp16' in sys.argv:
    fp16_raw(); sys.exit(0)

n=6
rgb, depth = synth.raw_frame(6); poses = synth.raw_poses(n, seed=6); rgbA, depthA = synth.rendered_views(n, poses, seed=6)
mean, std = synth.default_mean_std()
stats = {0:(mean,std), 1:(mean+1.5, std*1.25)}
wid=[0,0,0,1,1,1]
for w in (0,1):
    sd = synth.make_state_dict(w)
    As=[];Bs=[]
    for i in range(n):
        if wid[i]!=w: continue
        bb = O.compute_bbox(poses[i], synth.CAMERA_K, 200.0, scale=(1000,1000,1000)); rB,dB = O.crop_bbox(rgb, depth, bb, (176,176))
        (a,b),_ = O.process_data(rgbA[i], depthA[i], poses[i], rB, dB, np.eye(4), *stats[w]); As.append(torch.from_numpy(a)); Bs.append(torch.from_numpy(b))
    A=torch.stack(As); B=torch.stack(Bs)
    print('input absmax', A.abs().max().item(), B.abs().max().item())
    with torch.no_grad():
        ref = O.forward(sd,A,B); ref = torch.cat((ref['trans'],ref['rot']),1)
        for name,modes in [('all tf32',{}), ('stem 3x',{'stem':'3x'}), ('stem fp32',{'stem':'fp32'}), ('stem+c64 3x',{'stem':'3x','c64':'3x'}),
                           ('head 3x',{'head':'3x'}), ('ab 3x',{'ab':'3x'}), ('all 3x', {'stem':'3x','c64':'3x','ab':'3x','head':'3x'}),
                           ('stem,c64,ab 3x',{'stem':'3x','c64':'3x','ab':'3x'})]:
            out = run(sd,A,B,modes); err=(out-ref).abs(); tol=1e-4+1e-3*ref.abs()
            print(w, '%-16s max abs err %.3e  max err/tol %.3f' % (name, err.max().item(), (err/tol).max().item()))
