"""Precision study (CPU, not product code): TF32 / BF16 / FP16 operand-rounding emulation on tensor-regime inputs and on
config 1 (see precision_raw.py for the raw regime).  fp16 emulates SE3TN_PREC_FP16 exactly: bf16x3 stems, fp16 operands
(rne, saturating at 65504) everywhere else, every stored activation rounded to fp16.  Run from the repo root:
    python scripts/precision_study.py [n]"""
import importlib, sys, numpy as np, torch, torch.nn.functional as F
sys.path.insert(0,'.'); sys.path.insert(0,'oracle')
synth = importlib.import_module('iros20-6d-pose-tracking_b200.synth')
import se3_oracle as O
torch.set_num_threads(8)

def rna_tf32(x):
    i = x.contiguous().view(torch.int32)
    i = (i + 0x1000) & ~0x1FFF
    return i.view(torch.float32)
def rn_bf16(x): return x.to(torch.bfloat16).to(torch.float32)
def rn_fp16(x): return x.clamp(-65504., 65504.).to(torch.float16).to(torch.float32)   # cvt.rn.satfinite.f16x2.f32
def ident(x): return x

def bf16x3_conv(x, w, stride, pad, dt):
    """hi.w_hi + lo.w_hi + hi.w_lo of bf16 hi / lo splits: the arithmetic of the stems of the 2-byte modes"""
    xh = rn_bf16(x); xl = rn_bf16(x - xh); wh = rn_bf16(w); wl = rn_bf16(w - wh)
    c = lambda a, v: F.conv2d(a.to(dt), v.to(dt), None, stride=stride, padding=pad)
    return (c(xh, wh) + c(xl, wh) + c(xh, wl)).float()

def fold(sd, conv, bn):
    w = sd[conv+'.weight'].double(); b = sd[conv+'.bias'].double()
    g = sd[bn+'.weight'].double(); beta = sd[bn+'.bias'].double(); mu = sd[bn+'.running_mean'].double(); var = sd[bn+'.running_var'].double()
    s = g/torch.sqrt(var+1e-5)
    return (w*s[:,None,None,None]).float(), ((b-mu)*s+beta).float()

def selu(x): return F.selu(x)

def run(sd, A, B, rnd, dt=torch.float64, stem3=False):
    # stem3: the stems run bf16x3_conv on the unrounded input (their outputs are still stored with rnd)
    def conv(x, w, b, stride, pad, three=False):
        if three: y = bf16x3_conv(x, w, stride, pad, dt)
        else: y = F.conv2d(rnd(x).to(dt), rnd(w).to(dt), None, stride=stride, padding=pad).float()
        return y + b[None,:,None,None]
    def cbr(x, p, stride, pad, three=False):
        w,b = fold(sd, p+'.0', p+'.1'); return rnd(selu(conv(x,w,b,stride,pad,three)))
    def block(x, p):
        w1,b1 = fold(sd,p+'.conv1',p+'.bn1'); w2,b2 = fold(sd,p+'.conv2',p+'.bn2')
        t = rnd(F.relu(conv(x,w1,b1,1,1)))
        return rnd(F.relu(conv(t,w2,b2,1,1)+x))
    a = cbr(A if stem3 else rnd(A),'convA1',2,3,stem3); a = F.max_pool2d(a,3,2,1); a = block(a,'convA2')
    b = cbr(B if stem3 else rnd(B),'convB1',2,3,stem3); b = F.max_pool2d(b,3,2,1); b = block(b,'convB2'); b = block(b,'convB3')
    ab = torch.cat((a,b),1); ab = cbr(ab,'convAB1',2,1); ab = block(ab,'convAB2')
    outs=[]
    for h in ('trans','rot'):
        x = cbr(ab,h+'_conv1',2,1); x = block(x,h+'_conv2')
        x = x.mean((2,3))
        outs.append(torch.tanh(F.linear(x, sd[h+'_out.0.weight'], sd[h+'_out.0.bias'])))
    return torch.cat(outs,1)

def run_fp16(sd, A, B):
    return run(sd, A, B, rn_fp16, stem3=True)

def config1():
    """BASELINE config 1 (the shipped image pair, weight seed 0) as normalised inputs A, B"""
    import os, cv2
    g = os.path.join('tests', 'golden')
    rgbA = cv2.imread(os.path.join(g, 'c1_rgbA.png'))[..., ::-1].copy(); rgbB = cv2.imread(os.path.join(g, 'c1_rgbB.png'))[..., ::-1].copy()
    (a, b), _ = O.process_data(rgbA, synth.depth_from_rgb(rgbA), synth.config1_pose(), rgbB, synth.depth_from_rgb(rgbB), np.eye(4),
                               *synth.default_mean_std())
    return torch.from_numpy(a)[None].float(), torch.from_numpy(b)[None].float()

def report(tag, out, ref):
    err = (out-ref).abs(); tol = 1e-4+1e-3*ref.abs()
    print(tag, 'max abs err %.3e'%err.max().item(), 'max err/tol %.3f'%(err/tol).max().item(), 'ref absmax %.3f'%ref.abs().max().item())

if __name__ == '__main__':
    n = int(sys.argv[1]) if len(sys.argv)>1 else 8
    for seed in (0,1):
        sd = synth.make_state_dict(seed)
        A,B = synth.tensor_pairs(n, seed=seed)
        with torch.no_grad():
            ref = O.forward(sd,A,B); ref = torch.cat((ref['trans'],ref['rot']),1)
            for name,r in (('fp32-fold',ident),('tf32',rna_tf32),('bf16',rn_bf16)):
                report('%d %s' % (seed, name), run(sd,A,B,r), ref)
            report('%d fp16' % seed, run_fp16(sd,A,B), ref)
    with torch.no_grad():
        sd = synth.make_state_dict(0); A, B = config1()
        ref = O.forward(sd,A,B); ref = torch.cat((ref['trans'],ref['rot']),1)
        for name,r in (('tf32',rna_tf32),('bf16',rn_bf16)):
            report('config 1 %s' % name, run(sd,A,B,r), ref)
        report('config 1 fp16', run_fp16(sd,A,B), ref)
