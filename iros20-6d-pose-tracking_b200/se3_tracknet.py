"""Drop-in for the reference's se3_tracknet.py: same class name, constructor, load_state_dict /
cuda / eval / __call__ surface and output dict -- but forward() runs the hand-written sm_90a
kernels of libse3tn through the C ABI instead of torch.nn -> cuDNN.

Reference: se3_tracknet.py:52-121 (Se3TrackNet, its loss), network_modules.py:59-66,86-120.
Inference only: loss() evaluates the training loss without gradients (Problem.validate's use);
autograd and training are out of scope, so train(True) raises.
"""
import torch
from .engine import Engine


class Se3TrackNet(torch.nn.Module):
    def __init__(self, image_size=174, max_batch=64, precision='bf16x3', engine=None, weight_id=0):
        super().__init__()
        self.rot_dim = 3
        self.image_size = image_size          # unused by the reference too (fully convolutional, F5)
        self.max_batch = max_batch
        self.precision = precision
        self.weight_id = weight_id
        self._engine = engine
        self._sd = None
        self._loaded = False

    # -- nn.Module surface the reference's callers use (predict.py:153-158) ---------------------
    def load_state_dict(self, state_dict, strict=True):
        missing = [k for k in ('convA1.0.weight', 'trans_out.0.weight', 'rot_out.0.bias') if k not in state_dict]
        if missing:
            raise RuntimeError('not a Se3TrackNet state_dict, missing keys: %s' % missing)
        self._sd = {k: v.detach().cpu() for k, v in state_dict.items()}
        self._loaded = False
        if self._engine is not None:
            self._upload()
        return torch.nn.modules.module._IncompatibleKeys([], [])

    def state_dict(self, *args, **kwargs):
        return dict(self._sd) if self._sd is not None else {}

    def cuda(self, device=None):
        if self._engine is None:
            self._engine = Engine(max_batch=self.max_batch, device=device)
        if self._sd is not None and not self._loaded:
            self._upload()
        return self

    def to(self, *args, **kwargs):
        dev = args[0] if args else kwargs.get('device')
        if dev is not None and torch.device(dev).type == 'cuda':
            return self.cuda(torch.device(dev).index)
        raise RuntimeError('Se3TrackNet (H100) only lives on a CUDA device; there is no CPU path')

    def train(self, mode=True):
        if mode:
            raise NotImplementedError('this is the inference hot path only (training is out of scope)')
        return super().train(False)

    @property
    def engine(self):
        if self._engine is None:
            self.cuda()
        return self._engine

    def _upload(self):
        self._engine.load_state_dict(self._sd, self.weight_id)
        self._loaded = True

    # -- se3_tracknet.py:81-112 -------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, A, B, return_feature=True):
        if self._sd is None:
            raise RuntimeError('load_state_dict() must be called before forward()')
        eng = self.engine
        if not self._loaded:
            self._upload()
        A = A.to(eng.device, torch.float32).contiguous()
        B = B.to(eng.device, torch.float32).contiguous()
        trans, rot, feat = eng.forward(A, B, weight_id=self.weight_id, precision=self.precision,
                                       want_feature=return_feature)
        out = {'trans': trans, 'rot': rot}
        if return_feature:
            out['feature'] = feat
        return out

    # -- se3_tracknet.py:114-121 ------------------------------------------------------------------
    @torch.no_grad()
    def loss(self, predictions, targets):
        """{'trans', 'rot'}: nn.MSELoss of (predictions[k].float(), targets[k].float()) as float32 device scalars, summed by
        se3tn_pair_loss in the order the validation step uses (Engine.eval_pairs) and divided by the element count."""
        eng = self.engine
        trans = predictions[0].to(eng.device, torch.float32).contiguous()
        rot = predictions[1].to(eng.device, torch.float32).contiguous()
        # float64 holds any float32 target exactly, and the kernel rounds every label to float32 as .float() does
        tl = targets[0].to(eng.device, torch.float64).contiguous()
        rl = targets[1].to(eng.device, torch.float64).contiguous()
        for name, p, t in (('trans', trans, tl), ('rot', rot, rl)):
            if p.dim() != 2 or p.shape[1] != 3 or p.shape != t.shape:
                raise ValueError('loss: %s predictions and targets must both be (n,3), got %s and %s' % (name, tuple(p.shape), tuple(t.shape)))
        sums = eng.pair_loss(trans, rot, tl, rl)
        denom = float(3 * trans.shape[0])
        return {'trans': sums[0] / denom, 'rot': sums[1] / denom}
