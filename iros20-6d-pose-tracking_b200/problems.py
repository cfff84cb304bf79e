"""Drop-in for the reference's problems.py: Problem.validate (reference problems.py:106-132), the validation pass that picks
the checkpoint every Tracker loads (Problem.loop keeps the lowest validation loss as model_best_val.pth.tar, :146-151).
Training (Problem.train, Problem.loop, the optimiser) is out of scope and raises.

validate() returns the reference's number -- the mean over the loader's batches of each batch's nn.MSELoss, translation and
rotation, weighted by config['loss_weights'] -- but does not iterate the DataLoader.  It reads the dataset's file list and runs
each batch through se3tn_eval_pairs (Engine.eval_pairs): processData's post-transforms, the network and the loss terms in one
step on the device.  PNGs are decoded in a thread pool (cv2 releases the GIL) straight into a StagingRing of two pinned
staging sets, so decoding step k+1 overlaps step k on the GPU.  A batch larger than the engine's max_batch runs as several steps whose sums
are added in order.  The pairs are taken in file order (the reference's validation loader does not shuffle, train.py:143-149).

    python -m <package>.problems --val_dir DIR --ckpt model_best_val.pth.tar --mean_std_path DIR --dataset_info dataset_info.yml
                                 [--precision bf16x3|tf32|bf16|fp16|fp8|fp32|all] [--batch_size 200]
"""
import argparse
import contextlib
import os

import numpy as np
import torch

from .datasets import TrackDataset, read_pair, resize_pair
from .engine import PREC, IMAGE_SIZE
from .staging import StagingRing


class Problem:
    def __init__(self, model, train_data_loader, valid_data_loader, config=None, optimizer=None, scheduler=None):
        self.train_data = train_data_loader
        self.valid_data = valid_data_loader
        self.optimizer = optimizer
        self.scheduler = scheduler
        self.model = model.cuda()
        self.config = config
        self.loss_weights = self.config['loss_weights']
        self.best_eval = np.inf
        self.best_val = np.inf
        self.best_train = np.inf
        ds = (train_data_loader if train_data_loader is not None else valid_data_loader).dataset
        self.dataset_info = ds.dataset_info
        self.K = getattr(ds, 'cam_K', None)

    def train(self, epoch):
        raise NotImplementedError('training is out of scope: this library validates checkpoints, it does not train them')

    def loop(self, total_epochs, output_path, save_all_checkpoints=False):
        raise NotImplementedError('training is out of scope: this library validates checkpoints, it does not train them')

    def validate(self, epoch=None, precision=None):
        """problems.py:106-132: trans_loss * loss_weights['trans'] + rot_loss * loss_weights['rot']."""
        r = self.validation_losses(precision)
        return r['trans'] * self.loss_weights['trans'] + r['rot'] * self.loss_weights['rot']

    def validation_losses(self, precision=None, keep_predictions=False):
        """-> dict(trans, rot: the means over batches of each batch's MSE (python floats), batch_trans / batch_rot: the per-batch
        MSEs (float32), predictions: (N,6) float32 numpy of every pair's network output when keep_predictions)."""
        loader = self.valid_data
        return evaluate(self.model, loader.dataset, int(loader.batch_size), bool(getattr(loader, 'drop_last', False)),
                        precision or self.model.precision, keep_predictions)


def batch_plan(n_pairs, batch_size, max_batch, drop_last=False):
    """The loader's batches as [start, end) ranges (the last one partial unless drop_last), each cut into steps of at most
    max_batch pairs: -> list of (batch index, start, end)."""
    if batch_size <= 0 or max_batch <= 0:
        raise ValueError('batch_size and max_batch must be positive')
    steps = []
    n_batches = n_pairs // batch_size if drop_last else -(-n_pairs // batch_size)
    for b in range(n_batches):
        b0, b1 = b * batch_size, min(n_pairs, (b + 1) * batch_size)
        for s in range(b0, b1, max_batch):
            steps.append((b, s, min(b1, s + max_batch)))
    return steps


def batch_means(step_sums, steps):
    """Per-batch MSE from per-step float32 sums (n_steps, 2): a batch's steps are added in order in float32 and divided by its
    3 x pairs element count in float32, as nn.MSELoss's mean -> (trans (n_batches,), rot (n_batches,)) float32."""
    n_batches = steps[-1][0] + 1 if steps else 0
    acc = np.zeros((n_batches, 2), dtype=np.float32)
    cnt = np.zeros(n_batches, dtype=np.int64)
    for (b, s, e), sums in zip(steps, np.asarray(step_sums, dtype=np.float32)):
        acc[b] = acc[b] + sums
        cnt[b] += e - s
    mse = acc / (3 * cnt).astype(np.float32)[:, None]
    return mse[:, 0], mse[:, 1]


def _mean_over_batches(x):
    """problems.py:128-129: np.array(list of .item() floats).mean()."""
    return float(np.array([float(v) for v in x]).mean())


def evaluate(model, dataset, batch_size, drop_last=False, precision='bf16x3', keep_predictions=False, workers=None):
    """The validation pass of `model` (the Se3TrackNet drop-in) over `dataset`'s pairs; see the module docstring."""
    eng = model.engine
    if not model._loaded:
        model._upload()
    wid = int(model.weight_id)
    eng.set_stats(np.asarray(dataset.images_mean), np.asarray(dataset.images_std), wid)
    res = int(dataset.dataset_info['resolution']) if dataset.dataset_info is not None else IMAGE_SIZE
    if res != IMAGE_SIZE:
        raise NotImplementedError('libse3tn is built for the reference resolution of 176 (dataset_info.yml:15)')
    PREC[precision]                                         # an unknown mode fails here
    files = list(dataset.rgbA_files)
    cap = eng.max_batch
    steps = batch_plan(len(files), batch_size, cap, drop_last)
    if not steps:
        raise ValueError('no validation batch: %d pairs under %r' % (len(files), dataset.root))
    dev = eng.device
    img = (IMAGE_SIZE, IMAGE_SIZE)

    # the pinned sets decode step k+1 while step k runs; the one device set is what the steps read (uploads ordered on the stream)
    ring = StagingRing(dict(rgbA=((cap,) + img + (3,), torch.uint8), depthA=((cap,) + img, torch.uint16),
                            rgbB=((cap,) + img + (3,), torch.uint8), depthB=((cap,) + img, torch.uint16),
                            poses=((cap, 2, 4, 4), torch.float64)), 2, dev)
    d = ring.dev
    A_in_cam, B_in_cam = torch.empty(cap, 4, 4, dtype=torch.float64, device=dev), torch.empty(cap, 4, 4, dtype=torch.float64, device=dev)
    out_trans, out_rot = torch.empty(cap, 3, dtype=torch.float32, device=dev), torch.empty(cap, 3, dtype=torch.float32, device=dev)
    out_sums = torch.empty(2, dtype=torch.float32, device=dev)
    all_sums = torch.empty(len(steps), 2, dtype=torch.float32, device=dev)
    preds = torch.empty(len(files), 6, dtype=torch.float32, device=dev) if keep_predictions else None
    ids_host = np.full(cap, wid, dtype=np.int32) if wid != 0 else None
    ids_dev = torch.from_numpy(ids_host).to(dev) if ids_host is not None else None
    tn, rn = dataset.trans_normalizer, dataset.rot_normalizer

    def decode_into(h, j, path):
        """One pair into row j of staging set h; a pair stored at another size comes back whole for the device resize."""
        p = read_pair(path)
        h['poses'].numpy()[j, 0] = p['A_in_cam']; h['poses'].numpy()[j, 1] = p['B_in_cam']
        if p['rgbB'].shape[0] != res:
            return p
        maskB = p['segB'] if p['segB'] is not None else (p['depthB'] > 100)
        if not np.sum(maskB) > 0:
            raise AssertionError('%s: the pair has an empty maskB (datasets.py:104)' % path)
        for k in ('rgbA', 'depthA', 'rgbB', 'depthB'):
            h[k].numpy()[j] = p[k]
        return None

    items = [[(decode_into, j, files[s + j]) for j in range(e - s)] for _, s, e in steps]
    rows = [e - s for _, s, e in steps]
    with contextlib.closing(ring.uploads(items, workers or min(16, os.cpu_count() or 4), rows)) as uploads:
        for k, decoded in enumerate(uploads):
            _, s, e = steps[k]
            n = e - s
            A_in_cam[:n].copy_(d['poses'][:n, 0]); B_in_cam[:n].copy_(d['poses'][:n, 1])
            for j, p in enumerate(decoded):
                if p is None:
                    continue
                rA, dA, rB, dB, seg = resize_pair(eng, p, res)          # datasets.py:95-104 on the device
                mask_sum = int((seg if seg is not None else (dB > 100)).sum().item())
                if mask_sum <= 0:
                    raise AssertionError('%s: the pair has an empty maskB (datasets.py:104)' % files[s + j])
                d['rgbA'][j].copy_(rA); d['depthA'][j].copy_(dA); d['rgbB'][j].copy_(rB); d['depthB'][j].copy_(dB)
            if precision == 'fp8' and k == 0:              # the set's activation scales from the first validation batch
                eng.calibrate_fp8_pairs(d['rgbA'][:n], d['depthA'][:n], d['rgbB'][:n], d['depthB'][:n], A_in_cam[:n],
                                        ids_host[:n] if ids_host is not None else None)
            eng.eval_pairs(d['rgbA'][:n], d['depthA'][:n], d['rgbB'][:n], d['depthB'][:n], A_in_cam[:n], B_in_cam[:n], tn, rn,
                           weight_ids_host=ids_host[:n] if ids_host is not None else None,
                           weight_ids_dev=ids_dev[:n] if ids_dev is not None else None, precision=precision,
                           out_trans=out_trans[:n], out_rot=out_rot[:n], out_sums=out_sums)
            all_sums[k].copy_(out_sums)
            if preds is not None:
                preds[s:e, :3].copy_(out_trans[:n]); preds[s:e, 3:].copy_(out_rot[:n])
    step_sums = all_sums.cpu().numpy()
    bt, br = batch_means(step_sums, steps)
    return dict(trans=_mean_over_batches(bt), rot=_mean_over_batches(br), batch_trans=bt, batch_rot=br,
                predictions=preds.cpu().numpy() if preds is not None else None)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Validation loss of a se(3)-TrackNet checkpoint on a folder of training pairs "
                                             "(the reference's Problem.validate), per precision mode")
    ap.add_argument('--val_dir', required=True, help='folder of *rgbA.png / rgbB / depthA / depthB / [segB] / meta.npz pairs')
    ap.add_argument('--ckpt', required=True, help="checkpoint with a 'state_dict' (e.g. model_best_val.pth.tar)")
    ap.add_argument('--mean_std_path', required=True, help='folder holding mean.npy and std.npy (train.py:124-125)')
    ap.add_argument('--dataset_info', required=True, help='dataset_info.yml (resolution, max_translation, max_rotation)')
    ap.add_argument('--precision', default='bf16x3', choices=sorted(PREC) + ['all'])
    ap.add_argument('--batch_size', type=int, default=200, help='the validation loader batch size (train.py:146)')
    ap.add_argument('--max_batch', type=int, default=200, help='pairs per device step (a larger batch runs as several steps)')
    args = ap.parse_args(argv)
    import yaml
    from .se3_tracknet import Se3TrackNet
    with open(args.dataset_info) as f:
        info = yaml.safe_load(f)
    mean = np.load(os.path.join(args.mean_std_path, 'mean.npy'))
    std = np.load(os.path.join(args.mean_std_path, 'std.npy'))
    ds = TrackDataset(args.val_dir, 'val', mean, std, None, None, None, dataset_info=info,
                      trans_normalizer=info['max_translation'], rot_normalizer=info['max_rotation'] * np.pi / 180)
    loader = torch.utils.data.DataLoader(ds, batch_size=args.batch_size, shuffle=False, drop_last=False)
    ckpt = torch.load(args.ckpt, map_location='cpu')
    model = Se3TrackNet(image_size=int(info['resolution']), max_batch=min(args.max_batch, args.batch_size))
    model.load_state_dict(ckpt['state_dict'] if 'state_dict' in ckpt else ckpt)
    prob = Problem(model, None, loader, config={'loss_weights': {'trans': 1, 'rot': 1}})   # config.yml:13-15
    modes = ['fp32', 'bf16x3', 'tf32', 'bf16'] if args.precision == 'all' else [args.precision]
    print('%d pairs, batch %d, %s' % (len(ds), args.batch_size, torch.cuda.get_device_name(model.engine.device)))
    print('%-8s %14s %14s %14s %s' % ('mode', 'trans loss', 'rot loss', 'total', 'max |d6| vs fp32' if len(modes) > 1 else ''))
    ref = None
    for m in modes:
        r = prob.validation_losses(m, keep_predictions=len(modes) > 1)
        w = prob.loss_weights
        dev6 = ''
        if len(modes) > 1:
            if ref is None:
                ref = r['predictions']
            dev6 = '%.3e' % float(np.abs(r['predictions'] - ref).max())
        print('%-8s %14.8g %14.8g %14.8g %s' % (m, r['trans'], r['rot'], r['trans'] * w['trans'] + r['rot'] * w['rot'], dev6))


if __name__ == '__main__':
    main()
