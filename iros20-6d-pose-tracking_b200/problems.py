"""Drop-in for the reference's problems.py: Problem.validate (reference problems.py:106-132), the validation pass that picks
the checkpoint every Tracker loads (Problem.loop keeps the lowest validation loss as model_best_val.pth.tar, :146-151).
Training (Problem.train, Problem.loop, the optimiser) is out of scope and raises.

validate() returns the reference's number -- the mean over the loader's batches of each batch's nn.MSELoss, translation and
rotation, weighted by config['loss_weights'] -- but does not iterate the DataLoader.  It reads the dataset's file list and runs
each batch through se3tn_eval_pairs (Engine.eval_pairs): processData's post-transforms, the network and the loss terms in one
step on the device.  PNGs are decoded in a thread pool (cv2 releases the GIL) straight into a StagingRing of two pinned
staging sets, so decoding step k+1 overlaps step k on the GPU.  A batch larger than the engine's max_batch runs as several steps whose sums
are added in order.  The pairs are taken in file order (the reference's validation loader does not shuffle, train.py:143-149).

    python -m <package>.problems --val_dir DIR --ckpt CKPT[,CKPT...] --mean_std_path DIR[,DIR...] --dataset_info dataset_info.yml
                                 [--precision bf16x3|tf32|bf16|fp16|fp8|fp32|all] [--batch_size 200] [--augment config.yml [--seed S]]
    python -m <package>.problems --ycb_dir DIR --class_ids all|3,5 --ckpt_dir TPL --mean_std_path TPL --train_data_path TPL
                                 --model_path TPL [--num_sample 10] [--seed 0] [--precision MODE|all] [--batch_size 200] [--max_batch 200]
                                 [--augment config.yml]

The second form scores every class's checkpoint on the perturbed pairs of the YCB-Video key frames in one pass (validate_ycbv):
bit-identical to `produce_train_pair_data --mode ycbv` followed by the first form on each class's folder, without the files.

Both forms take several checkpoints, comma-separated, with one statistics folder shared by all or one per checkpoint: the pairs
are decoded (or cut) once and every step runs once per checkpoint and mode, each result what a run of that checkpoint alone
gives; the table then names, per mode, the checkpoint with the lowest total loss.

--augment evaluates either form under the reference's train-time augmentations (train.py:85-92, built from config.yml's
data_augmentation block), as the reference's own validation loss is computed: input B of every pair is augmented once per step
(se3tn_augment_crops), each pair's draws keyed by (--seed, its index in the sorted file list), so every checkpoint and every
mode of --precision all sees the same augmented pairs.  With --ycb_dir, --seed seeds both the perturbations and the
augmentation, and a pair's index is that of the file `produce_train_pair_data --mode ycbv --seed S` would write for it: the
result is `--val_dir <class folder> --augment config.yml --seed S` on that folder, bit for bit.
"""
import argparse
import contextlib
import os
import random

import numpy as np
import torch

from .datasets import TrackDataset, read_pair, resize_pair, segB_plane
from .engine import PREC, IMAGE_SIZE, check_weight_sets_fit
from .predict import CKPT_ID_STRIDE
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


def evaluate(model, dataset, batch_size, drop_last=False, precision='bf16x3', keep_predictions=False, workers=None, stats=None):
    """The validation pass of `model` (the Se3TrackNet drop-in) over `dataset`'s pairs; see the module docstring.

    The list form compares checkpoints in one pass: `model` a list of Se3TrackNet on one Engine under distinct weight ids and / or
    `precision` a list of modes.  Each step's pairs are decoded once (and with --augment, input B augmented once, by
    se3tn_augment_crops) and then run once per variant (model index, mode), each on its own weight set and step sums, so every
    variant's result is bit for bit what a one-model call gives.  stats: [(mean, std)] per model, default the dataset's for all
    (train.py writes mean / std per training run).  fp8 calibrates each model's set on the first step as its steps see it.
    -> {(model index, mode): the one-model call's dict}.  The one-model call returns that dict alone."""
    many = isinstance(model, (list, tuple)) or isinstance(precision, (list, tuple))
    models = list(model) if isinstance(model, (list, tuple)) else [model]
    modes = list(precision) if isinstance(precision, (list, tuple)) else [precision]
    if not models or not modes:
        raise ValueError('evaluate needs at least one model and one precision mode')
    for m in modes:
        PREC[m]                                             # an unknown mode fails here
    eng = models[0].engine
    wids = [int(mdl.weight_id) for mdl in models]
    if any(mdl.engine is not eng for mdl in models) or len(set(wids)) != len(wids):
        raise ValueError('the models of one pass share one Engine under distinct weight ids (got ids %s)' % wids)
    if stats is None:
        stats = [(dataset.images_mean, dataset.images_std)] * len(models)
    if len(stats) != len(models):
        raise ValueError('%d (mean, std) pairs for %d models' % (len(stats), len(models)))
    for mdl, wid, (mean, std) in zip(models, wids, stats):
        if not mdl._loaded:
            mdl._upload()
        eng.set_stats(np.asarray(mean), np.asarray(std), wid)
    res = int(dataset.dataset_info['resolution']) if dataset.dataset_info is not None else IMAGE_SIZE
    if res != IMAGE_SIZE:
        raise NotImplementedError('libse3tn is built for the reference resolution of 176 (dataset_info.yml:15)')
    files = list(dataset.rgbA_files)
    cap = eng.max_batch
    steps = batch_plan(len(files), batch_size, cap, drop_last)
    if not steps:
        raise ValueError('no validation batch: %d pairs under %r' % (len(files), dataset.root))
    dev = eng.device
    img = (IMAGE_SIZE, IMAGE_SIZE)
    variants = [(i, m) for i in range(len(models)) for m in modes]

    # the pinned sets decode step k+1 while step k runs; the one device set is what the steps read (uploads ordered on the stream)
    augment = getattr(dataset, 'augment', None)
    planes = dict(rgbA=((cap,) + img + (3,), torch.uint8), depthA=((cap,) + img, torch.uint16),
                  rgbB=((cap,) + img + (3,), torch.uint8), depthB=((cap,) + img, torch.uint16), poses=((cap, 2, 4, 4), torch.float64))
    if augment is not None:                                 # BlackCover's maskB: segB, or depthB > 100 where a pair has none
        planes['segB'] = ((cap,) + img, torch.uint8)
    ring = StagingRing(planes, 2, dev)
    d = ring.dev
    A_in_cam, B_in_cam = torch.empty(cap, 4, 4, dtype=torch.float64, device=dev), torch.empty(cap, 4, 4, dtype=torch.float64, device=dev)
    out_trans, out_rot = torch.empty(cap, 3, dtype=torch.float32, device=dev), torch.empty(cap, 3, dtype=torch.float32, device=dev)
    out_sums = torch.empty(2, dtype=torch.float32, device=dev)
    all_sums = {v: torch.empty(len(steps), 2, dtype=torch.float32, device=dev) for v in variants}
    preds = {v: torch.empty(len(files), 6, dtype=torch.float32, device=dev) for v in variants} if keep_predictions else None
    ids_host = [np.full(cap, w, dtype=np.int32) if w != 0 else None for w in wids]
    ids_dev = [torch.from_numpy(h).to(dev) if h is not None else None for h in ids_host]
    tn, rn = dataset.trans_normalizer, dataset.rot_normalizer
    if augment is not None:                                 # input B augmented once per step, read by every variant
        all_index = torch.arange(len(files), dtype=torch.int64, device=dev)
        aug_rgbB, aug_depthB = torch.empty((cap,) + img + (3,), dtype=torch.uint8, device=dev), torch.empty((cap,) + img, dtype=torch.uint16, device=dev)

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
        if augment is not None:
            h['segB'].numpy()[j] = segB_plane(maskB)
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
                if augment is not None:
                    if seg is not None and seg.dtype != torch.uint8:
                        raise ValueError('%s: augmentation needs segB as an 8-bit image, not %s' % (files[s + j], seg.dtype))
                    d['segB'][j].copy_(seg if seg is not None else (dB.to(torch.int32) > 100).to(torch.uint8))
            rB, dB = d['rgbB'][:n], d['depthB'][:n]
            if augment is not None:                         # what se3tn_eval_pairs_augmented evaluates, formed once
                rB, dB = eng.augment_crops(augment, rB, dB, all_index[s:e], segB=d['segB'][:n], out_rgbB=aug_rgbB[:n],
                                           out_depthB=aug_depthB[:n])
            for i, m in variants:
                wh = ids_host[i][:n] if ids_host[i] is not None else None
                if m == 'fp8' and k == 0:                   # the set's activation scales from the first batch, as the steps see it
                    eng.calibrate_fp8_pairs(d['rgbA'][:n], d['depthA'][:n], rB, dB, A_in_cam[:n], wh)
                eng.eval_pairs(d['rgbA'][:n], d['depthA'][:n], rB, dB, A_in_cam[:n], B_in_cam[:n], tn, rn, weight_ids_host=wh,
                               weight_ids_dev=ids_dev[i][:n] if ids_dev[i] is not None else None, precision=m,
                               out_trans=out_trans[:n], out_rot=out_rot[:n], out_sums=out_sums)
                all_sums[i, m][k].copy_(out_sums)
                if preds is not None:
                    preds[i, m][s:e, :3].copy_(out_trans[:n]); preds[i, m][s:e, 3:].copy_(out_rot[:n])
    out = {}
    for v in variants:
        bt, br = batch_means(all_sums[v].cpu().numpy(), steps)
        out[v] = dict(trans=_mean_over_batches(bt), rot=_mean_over_batches(br), batch_trans=bt, batch_rot=br,
                      predictions=preds[v].cpu().numpy() if preds is not None else None)
    return out if many else out[0, modes[0]]


# ----------------------------------------------------------------------------------------------------
# One pass over perturbed YCB-Video key frames: the pairs `produce_train_pair_data --mode ycbv` would write, scored as
# `evaluate` scores each class's folder, without the files.
# ----------------------------------------------------------------------------------------------------
class PairQueues:
    """Per-class device queues of kept pairs and the validation steps that drain them.

    add() takes one frame's pair steps and appends each kept row to its class's queue on the device (Engine.append_pairs: one
    launch per step, slots and tails computed there).  Before that it drains every queue the earlier frames filled: each full
    batch (rows [0, batch_size)) runs in every mode, cut into steps as batch_plan cuts it, and the remaining rows move to the
    front, so a class's full batches always read the same addresses and replay their CUDA graphs.  finish() drains the full
    batches left and then each class's partial last batch, and returns the results.  A class's batches are thus the loader's
    batches over its pairs in count order, and its step sums are added exactly as `evaluate` adds them.

    With `augment` (a se3tn_augment, as data_augmentation.chain_config builds it) the queues also carry each row's segB, and a
    batch's input B is augmented once, before any variant runs (se3tn_augment_crops in steps of at most max_batch rows, BlackCover's
    mask the queued segB), into a batch-sized buffer that every variant and fp8 calibration then reads.  Row r of a class's batch
    is keyed by its index in the class's count order, the index of its file in the folder `--mode ycbv` writes, so the draws are
    those `evaluate` makes on that folder.  The buffer is allocated once: later batches keep its addresses and their graphs.

    The tails come back through a pinned copy queued after each append and waited for at the next add(); the frame loop's
    visibility call has synchronised the stream by then, so the wait costs nothing.  Device memory: the queues hold
    len(class_ids) x (batch_size + rows_per_frame) pairs of 176 x 176 x 10 bytes (11 with augment) plus two float64 poses each,
    e.g. about 1.4 GB (1.5 GB) for 21 classes, batch_size 200 and 10 samples per class and frame; augment adds
    batch_size x 176 x 176 x 5 bytes for the augmented batch."""

    PLANES = (('rgbA', torch.uint8, (IMAGE_SIZE, IMAGE_SIZE, 3)), ('depthA', torch.uint16, (IMAGE_SIZE, IMAGE_SIZE)),
              ('rgbB', torch.uint8, (IMAGE_SIZE, IMAGE_SIZE, 3)), ('depthB', torch.uint16, (IMAGE_SIZE, IMAGE_SIZE)),
              ('A_in_cam', torch.float64, (4, 4)), ('B_in_cam', torch.float64, (4, 4)))

    def __init__(self, eng, normalizers, modes, batch_size, max_batch, rows_per_frame, keep_predictions=False, ckpts=1, augment=None):
        """normalizers: {class id (the weight set and mesh id): (trans_normalizer, rot_normalizer)}.  rows_per_frame: the most
        rows one frame sends to one class (num_sample).  max_batch: the most pairs per validation step.  ckpts: the number of
        checkpoints; checkpoint i's set of class c is weight id c + CKPT_ID_STRIDE * i, and every batch runs once per checkpoint
        and mode.  augment: the se3tn_augment applied to input B of every pair, or None."""
        if batch_size <= 0 or max_batch <= 0 or rows_per_frame <= 0:
            raise ValueError('batch_size, max_batch and rows_per_frame must be positive')
        self.eng = eng
        self.ids = sorted(normalizers)
        self.qid = {c: q for q, c in enumerate(self.ids)}
        self.normalizers = dict(normalizers)
        self.modes = list(modes)
        self.batch_size = int(batch_size)
        self.step = min(int(max_batch), self.batch_size)
        if self.step > eng.max_batch:
            raise ValueError('validation steps of %d pairs need an Engine of max_batch >= %d (it has %d)' % (self.step, self.step, eng.max_batch))
        self.cap = self.batch_size + int(rows_per_frame)
        self.keep_predictions = keep_predictions
        dev = eng.device
        Q = len(self.ids)
        self.augment = augment
        planes = self.PLANES + ((('segB', torch.uint8, (IMAGE_SIZE, IMAGE_SIZE)),) if augment is not None else ())
        self.queues = {k: torch.empty((Q, self.cap) + shape, dtype=dt, device=dev) for k, dt, shape in planes}
        if augment is not None:                             # one batch's augmented input B, read by every variant
            self.aug_rgbB = torch.empty((self.batch_size, IMAGE_SIZE, IMAGE_SIZE, 3), dtype=torch.uint8, device=dev)
            self.aug_depthB = torch.empty((self.batch_size, IMAGE_SIZE, IMAGE_SIZE), dtype=torch.uint16, device=dev)
        self.tails = np.zeros(Q, dtype=np.int32)            # host: exact after a read-back, then a bound as rows are sent
        self.tails_dev = torch.zeros(Q, dtype=torch.int32, device=dev)
        on_cuda = torch.device(dev).type == 'cuda'
        self._tails_back = torch.zeros(Q, dtype=torch.int32, pin_memory=on_cuda)
        self._back_done = torch.cuda.Event() if on_cuda else None
        self._sent = False                                  # rows appended since the tails were last read back
        self.out_trans = torch.empty(self.step, 3, dtype=torch.float32, device=dev)
        self.out_rot = torch.empty(self.step, 3, dtype=torch.float32, device=dev)
        self.out_sums = torch.empty(2, dtype=torch.float32, device=dev)
        self.variants = [(i, m) for i in range(int(ckpts)) for m in self.modes]
        wids = [c + CKPT_ID_STRIDE * i for c in self.ids for i in range(int(ckpts))]
        self.ids_host = {w: np.full(self.step, w, dtype=np.int32) for w in wids}
        self.ids_dev = {w: torch.from_numpy(self.ids_host[w]).to(dev) for w in wids}
        self.pairs = {c: 0 for c in self.ids}
        self.sums = {c: {v: [] for v in self.variants} for c in self.ids}
        self.preds = {c: {v: [] for v in self.variants} for c in self.ids}
        self.calibrated = set()

    def add(self, owners, chunks):
        """One frame: owners [(class id, B_in_cam, [A_in_cam of its rows], first row)], chunks [(first row, perturb_pairs dict with
        A_in_cam)] as produce_train_pair_data.ycbv_pair_steps yields them with on_device."""
        self._drain(final=False)
        row_q, row_B = [], []
        for c, B, inside, _ in owners:
            row_q += [self.qid[c]] * len(inside)
            row_B += [B] * len(inside)
        for i0, res in chunks:
            n = int(res['A_in_cam'].shape[0])
            qids = np.array(row_q[i0:i0 + n], dtype=np.int32)
            B = torch.from_numpy(np.ascontiguousarray(np.stack(row_B[i0:i0 + n]), dtype=np.float64)).to(self.eng.device)
            self.eng.append_pairs(res, res['A_in_cam'], B, qids, self.tails, self.tails_dev, self.queues)
            self.tails += np.bincount(qids, minlength=len(self.ids)).astype(np.int32)
            self._sent = True
        if self._sent:
            self._tails_back.copy_(self.tails_dev, non_blocking=True)
            if self._back_done is not None:
                self._back_done.record(torch.cuda.current_stream(self.eng.device))

    def finish(self):
        """Drain every queue, the partial last batches included -> {class id: {mode: dict}}: `evaluate`'s dict plus 'pairs'; with
        several checkpoints {checkpoint index: that}.  A class without a kept pair has pairs 0, trans / rot None, empty batch
        losses and predictions None."""
        self._drain(final=True)
        out = {}
        for c in self.ids:
            n = self.pairs[c]
            for i, m in self.variants:
                o = out.setdefault(i, {}).setdefault(c, {})
                if n == 0:
                    o[m] = dict(pairs=0, trans=None, rot=None, batch_trans=np.zeros(0, np.float32), batch_rot=np.zeros(0, np.float32),
                                     predictions=None)
                    continue
                steps = batch_plan(n, self.batch_size, self.step)
                assert len(steps) == len(self.sums[c][i, m])
                bt, br = batch_means(torch.stack(self.sums[c][i, m]).cpu().numpy(), steps)
                preds = torch.cat(self.preds[c][i, m]).cpu().numpy() if self.keep_predictions else None
                o[m] = dict(pairs=n, trans=_mean_over_batches(bt), rot=_mean_over_batches(br), batch_trans=bt, batch_rot=br,
                                 predictions=preds)
        return out if len(out) > 1 else out[0]

    def _drain(self, final):
        """Read the tails back, run every full batch (and with `final` every partial one), move the remainders to the front."""
        if self._sent:
            if self._back_done is not None:
                self._back_done.synchronize()
            self.tails[:] = self._tails_back.numpy()
            self._sent = False
            if (self.tails > self.cap).any():
                raise RuntimeError('a pair queue overflowed: tails %s, capacity %d' % (self.tails.tolist(), self.cap))
        moved = False
        for q, c in enumerate(self.ids):
            while self.tails[q] >= self.batch_size or (final and self.tails[q] > 0):
                n = min(int(self.tails[q]), self.batch_size)
                self._eval_batch(q, c, n)
                rest = int(self.tails[q]) - n
                for k in self.queues:
                    if rest:
                        self.queues[k][q, :rest].copy_(self.queues[k][q, n:n + rest].clone())
                self.tails[q] = rest
                moved = True
        if moved:
            self.tails_dev.copy_(torch.from_numpy(self.tails))

    def _eval_batch(self, q, c, n_rows):
        """Rows [0, n_rows) of queue q as one loader batch, in every checkpoint and mode."""
        tn, rn = self.normalizers[c]
        d = self.queues
        plan = batch_plan(n_rows, self.batch_size, self.step)
        rgbB, depthB = d['rgbB'][q], d['depthB'][q]
        if self.augment is not None:                        # evaluate's augmented input B, formed once for every variant
            first = self.pairs[c]
            for _, s, e in plan:
                index = torch.arange(first + s, first + e, dtype=torch.int64, device=self.eng.device)
                self.eng.augment_crops(self.augment, rgbB[s:e], depthB[s:e], index, segB=d['segB'][q, s:e],
                                       out_rgbB=self.aug_rgbB[s:e], out_depthB=self.aug_depthB[s:e])
            rgbB, depthB = self.aug_rgbB, self.aug_depthB
        for i, m in self.variants:
            w = c + CKPT_ID_STRIDE * i
            for _, s, e in plan:
                n = e - s
                pairs = [d['rgbA'][q, s:e], d['depthA'][q, s:e], rgbB[s:e], depthB[s:e]]
                if m == 'fp8' and w not in self.calibrated:      # the set's scales from its first step, as evaluate's k == 0
                    self.eng.calibrate_fp8_pairs(*pairs, d['A_in_cam'][q, s:e], self.ids_host[w][:n])
                    self.calibrated.add(w)
                self.eng.eval_pairs(*pairs, d['A_in_cam'][q, s:e], d['B_in_cam'][q, s:e], tn, rn, weight_ids_host=self.ids_host[w][:n],
                                    weight_ids_dev=self.ids_dev[w][:n], precision=m, out_trans=self.out_trans[:n],
                                    out_rot=self.out_rot[:n], out_sums=self.out_sums)
                self.sums[c][i, m].append(self.out_sums.clone())
                if self.keep_predictions:
                    self.preds[c][i, m].append(torch.cat((self.out_trans[:n], self.out_rot[:n]), 1))
        self.pairs[c] += n_rows


def validate_ycbv(ycb_dir, class_ids, templates, num_sample=10, seed=0, batch_size=200, max_batch=200, precisions=('bf16x3',),
                  keep_predictions=False, decode_ahead=4, workers=None, engine=None, augmentations=None, augment_seed=None):
    """Problem.validate of every class on the perturbed pairs of the YCB-Video key frames, in one pass and without pair files.

    For each class and mode the result is bit-identical to `produce_train_pair_data --mode ycbv` with the same seed and
    num_sample followed by `evaluate` on that class's folder with the same batch_size and max_batch: the same pair count, per-batch
    MSEs, means over batches and (keep_predictions) per-pair outputs.  The frame loop is the writer's own
    (produce_train_pair_data.ycbv_pair_steps: the same draws in the same order, so random / np.random end in the same state),
    and a class's kept pairs are batched in the order the writer numbers them; see PairQueues.

    templates: ckpt_dir, mean_std_path, train_data_path and model_path with {class_id} / {class_name} placeholders, as
    `predict --mode ycbv_all` takes them.  One Engine (engine, or one of max(min(max_batch, batch_size), classes x num_sample)
    rows) holds every class's weights, statistics and mesh under id = class id.  Each class's loss uses its dataset_info.yml's
    max_translation and max_rotation * pi / 180, as the loader's labels do.  fp8 calibrates each class on its first step.

    templates may give ckpt_dir (and mean_std_path) as lists, one entry per checkpoint (mean_std_path: one shared, or one per
    checkpoint): checkpoint i's set of class c is weight id c + 32 i.  The pairs are cut and queued once per class, and every
    batch runs once per checkpoint and mode, so each checkpoint's result is what a run of it alone returns.

    augmentations: train.py:85-92's chain (a Utils.Compose, as data_augmentation.from_config builds it), applied to input B of
    every pair with draws keyed by (augment_seed, default seed, the pair's index in its class's count order).  Each class's
    result is then bit-identical to `evaluate` on its folder through TrackDataset(augmentations=..., augment_seed=...).

    -> {class id: {mode: evaluate's dict plus 'pairs'}}; with several checkpoints {checkpoint index: that}.  A class without a kept pair is reported with 0 pairs and no loss
    (trans / rot None), where `evaluate` on its empty folder raises ValueError.  The queues take
    classes x (batch_size + num_sample) x 176 x 176 x 10 bytes of device memory (about 1.4 GB for 21 classes at 200 and 10);
    with augmentations 11 bytes (about 1.5 GB) plus batch_size x 176 x 176 x 5 bytes for the augmented batch."""
    from .engine import Engine
    from .predict import ycb_classes, expand_class_paths, _load_run_files, checkpoint_configs, _check_checkpoint_ids
    from .produce_train_pair_data import ycbv_producers, ycbv_pair_steps, ycbv_keyframe_jobs
    from .data_augmentation import chain_config
    modes = list(precisions)
    augment = chain_config(augmentations, seed if augment_seed is None else augment_seed) if augmentations is not None else None
    for m in modes:
        PREC[m]                                             # an unknown mode fails here
    configs = checkpoint_configs(templates)
    classes = ycb_classes(ycb_dir, class_ids)
    if not classes:
        raise ValueError('no class ids given')
    ids = [c for c, _ in classes]
    _check_checkpoint_ids(ids, len(configs), 'class')
    runs = {}
    for i, cfg in enumerate(configs):
        for c, name in classes:
            runs[c, i] = _load_run_files('class %d (%s)' % (c, name), expand_class_paths(cfg, c, name))
            if int(runs[c, i]['dataset_info']['resolution']) != IMAGE_SIZE:
                raise NotImplementedError('libse3tn is built for the reference resolution of 176 (dataset_info.yml:15)')
    if len(configs) > 1:
        check_weight_sets_fit(len(runs), what='weight sets (checkpoints x classes)')
    step = min(int(max_batch), int(batch_size))
    eng = engine if engine is not None else Engine(max_batch=max(step, len(ids) * int(num_sample)))
    normalizers = {}
    for (c, i), run in runs.items():
        info = runs[c, 0]['dataset_info']
        ckpt = torch.load(run['ckpt_dir'], map_location='cpu')
        eng.load_state_dict(ckpt['state_dict'] if 'state_dict' in ckpt else ckpt, c + CKPT_ID_STRIDE * i)
        eng.set_stats(np.asarray(run['mean']), np.asarray(run['std']), c + CKPT_ID_STRIDE * i)
        normalizers[c] = (info['max_translation'], info['max_rotation'] * np.pi / 180)
    _, producers = ycbv_producers(ycb_dir, ids, configs[0], eng, workers)
    queues = PairQueues(eng, normalizers, modes, batch_size, step, num_sample, keep_predictions, len(configs), augment)
    random.seed(seed); np.random.seed(seed)
    jobs = ycbv_keyframe_jobs(ycb_dir, ids)
    for owners, chunks in ycbv_pair_steps(eng, producers, jobs, num_sample, decode_ahead, workers, on_device=True):
        queues.add(owners, chunks)
    return queues.finish()


ALL_MODES = ['fp32', 'bf16x3', 'tf32', 'bf16']          # --precision all, fp32 first: the reference of "max |d6|"


def _print_modes(modes, losses, w):
    """The per-mode table: losses(m) -> evaluate's dict (with predictions when there is more than one mode)."""
    print('%-8s %14s %14s %14s %s' % ('mode', 'trans loss', 'rot loss', 'total', 'max |d6| vs fp32' if len(modes) > 1 else ''))
    ref = None
    for m in modes:
        r = losses(m)
        dev6 = ''
        if len(modes) > 1:
            if ref is None:
                ref = r['predictions']
            dev6 = '%.3e' % float(np.abs(r['predictions'] - ref).max())
        print('%-8s %14.8g %14.8g %14.8g %s' % (m, r['trans'], r['rot'], r['trans'] * w['trans'] + r['rot'] * w['rot'], dev6))


def main(argv=None):
    ap = argparse.ArgumentParser(description="Validation loss of a se(3)-TrackNet checkpoint on a folder of training pairs "
                                             "(the reference's Problem.validate), per precision mode; or of every class's checkpoint "
                                             "on the perturbed pairs of the YCB-Video key frames, in one pass without pair files")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument('--val_dir', help='folder of *rgbA.png / rgbB / depthA / depthB / [segB] / meta.npz pairs')
    src.add_argument('--ycb_dir', help='YCB-Video root (data_organized/, image_sets/keyframe.txt, CADmodels/): score the pairs '
                                       '`produce_train_pair_data --mode ycbv` would write, class by class, without writing them')
    ap.add_argument('--ckpt', help="--val_dir: checkpoint with a 'state_dict' (e.g. model_best_val.pth.tar)")
    ap.add_argument('--mean_std_path', help='folder holding mean.npy and std.npy (train.py:124-125); --ycb_dir: its path template')
    ap.add_argument('--dataset_info', help='--val_dir: dataset_info.yml (resolution, max_translation, max_rotation)')
    ap.add_argument('--class_ids', help='--ycb_dir: comma-separated class ids, or all')
    ap.add_argument('--ckpt_dir', help='--ycb_dir: path template ({class_id}, {class_name}) of each class\'s checkpoint')
    ap.add_argument('--train_data_path', help='--ycb_dir: path template; dataset_info.yml is read from its ../')
    ap.add_argument('--model_path', help='--ycb_dir: path template of each class\'s mesh')
    ap.add_argument('--num_sample', type=int, default=10, help='--ycb_dir: perturbations drawn per annotated class and key frame')
    ap.add_argument('--seed', type=int, default=0, help='--ycb_dir: seed of random and np.random before the first draw; '
                                                        '--augment: the seed of every pair\'s augmentation draws')
    ap.add_argument('--augment', help="the reference's config.yml; its data_augmentation block builds train.py:85-92's chain, "
                                      "applied to input B of every pair before the validation step")
    ap.add_argument('--precision', default='bf16x3', choices=sorted(PREC) + ['all'])
    ap.add_argument('--batch_size', type=int, default=200, help='the validation loader batch size (train.py:146)')
    ap.add_argument('--max_batch', type=int, default=200, help='pairs per device step (a larger batch runs as several steps)')
    args = ap.parse_args(argv)
    modes = ALL_MODES if args.precision == 'all' else [args.precision]
    if args.ycb_dir:
        return _main_ycbv(ap, args, modes)
    if not (args.ckpt and args.mean_std_path and args.dataset_info):
        ap.error('--val_dir needs --ckpt, --mean_std_path and --dataset_info')
    import yaml
    from .se3_tracknet import Se3TrackNet
    from .predict import checkpoint_list
    try:
        runs = checkpoint_list(args.ckpt.split(','), args.mean_std_path.split(','), '--ckpt', '--mean_std_path')
    except ValueError as e:
        ap.error(str(e))
    if len(runs) > 1:
        check_weight_sets_fit(len(runs), what='checkpoints')
    with open(args.dataset_info) as f:
        info = yaml.safe_load(f)
    stats = [(np.load(os.path.join(d, 'mean.npy')), np.load(os.path.join(d, 'std.npy'))) for _, d in runs]
    augmentations = _augmentations(args.augment)
    ds = TrackDataset(args.val_dir, 'val', stats[0][0], stats[0][1], None, augmentations, None, dataset_info=info,
                      trans_normalizer=info['max_translation'], rot_normalizer=info['max_rotation'] * np.pi / 180, augment_seed=args.seed)
    models = []
    for i, (path, _) in enumerate(runs):
        ckpt = torch.load(path, map_location='cpu')
        models.append(Se3TrackNet(image_size=int(info['resolution']), max_batch=min(args.max_batch, args.batch_size),
                                  engine=models[0].engine if models else None, weight_id=i))
        models[-1].load_state_dict(ckpt['state_dict'] if 'state_dict' in ckpt else ckpt)
    w = {'trans': 1, 'rot': 1}                                                          # config.yml:13-15
    print('%d pairs, batch %d, %s%s' % (len(ds), args.batch_size, torch.cuda.get_device_name(models[0].engine.device),
                                        ", augmented (train.py's chain, seed %d)" % args.seed if args.augment else ''))
    res = evaluate(models, ds, args.batch_size, False, modes, keep_predictions=len(modes) > 1, stats=stats)
    _print_checkpoints([p for p, _ in runs], modes, res, w)
    return res


def _augmentations(path):
    """--augment: train.py:85-92's chain from config.yml, or None without the option."""
    if not path:
        return None
    import yaml
    from .data_augmentation import from_config
    with open(path) as f:
        return from_config(yaml.safe_load(f))


def best_checkpoint(totals):
    """The index of the lowest of `totals`, the first listed among equals: Problem.loop keeps a checkpoint only when its
    validation loss is strictly below the best so far (problems.py:146-151)."""
    best = 0
    for i, t in enumerate(totals):
        if t < totals[best]:
            best = i
    return best


def _print_checkpoints(names, modes, res, w):
    """The table of one pass over several checkpoints (res: {(checkpoint index, mode): evaluate's dict}): one row per checkpoint
    and mode as _print_modes lays them out, max |d6| measured within each checkpoint from its first mode; then per mode the
    checkpoint Problem.loop would keep (best_checkpoint).  A single checkpoint prints _print_modes' table alone."""
    if len(names) == 1:
        _print_modes(modes, lambda m: res[0, m], w)
        return
    total = lambda r: r['trans'] * w['trans'] + r['rot'] * w['rot']
    print('%-5s %-8s %14s %14s %14s %s' % ('ckpt', 'mode', 'trans loss', 'rot loss', 'total', 'max |d6| vs %s' % modes[0] if len(modes) > 1 else ''))
    for i in range(len(names)):
        for m in modes:
            r = res[i, m]
            dev6 = '%.3e' % float(np.abs(r['predictions'] - res[i, modes[0]]['predictions']).max()) if len(modes) > 1 else ''
            print('%-5d %-8s %14.8g %14.8g %14.8g %s' % (i, m, r['trans'], r['rot'], total(r), dev6))
    for m in modes:
        b = best_checkpoint([total(res[i, m]) for i in range(len(names))])
        print('best %s: checkpoint %d (%s), total %.8g' % (m, b, names[b], total(res[b, m])))


def _main_ycbv(ap, args, modes):
    """--ycb_dir: validate_ycbv, then per class the table --val_dir prints."""
    from .predict import ycb_class_names, YCB_ALL_TEMPLATES, checkpoint_configs
    if args.ckpt or args.dataset_info:
        ap.error('--ycb_dir takes --ckpt_dir and --train_data_path templates, not --ckpt / --dataset_info')
    if not args.class_ids or not all(getattr(args, k) for k in YCB_ALL_TEMPLATES):
        need = '--ycb_dir needs --class_ids, --ckpt_dir, --mean_std_path, --train_data_path and --model_path'
        ap.error('--augment works with --val_dir only or with a whole --ycb_dir run: ' + need if args.augment else need)
    names = ycb_class_names(args.ycb_dir)
    if args.class_ids == 'all':
        ids = list(range(1, len(names) + 1))
    else:
        try:
            ids = sorted(set(int(c) for c in args.class_ids.split(',')))
        except ValueError:
            ap.error('--class_ids must be comma-separated integers or all, not %r' % args.class_ids)
    templates = {k: getattr(args, k) for k in YCB_ALL_TEMPLATES}
    for key in ('ckpt_dir', 'mean_std_path'):                   # template lists: one pass over several checkpoints
        if ',' in templates[key]:
            templates[key] = templates[key].split(',')
    try:
        ckpts = [cfg['ckpt_dir'] for cfg in checkpoint_configs(templates)]
    except ValueError as e:
        ap.error(str(e))
    augmentations = _augmentations(args.augment)
    res = validate_ycbv(args.ycb_dir, ids, templates, num_sample=args.num_sample, seed=args.seed, batch_size=args.batch_size,
                        max_batch=args.max_batch, precisions=modes, keep_predictions=len(modes) > 1, augmentations=augmentations,
                        augment_seed=args.seed)
    per_ckpt = [res[i] for i in range(len(ckpts))] if len(ckpts) > 1 else [res]
    device = torch.cuda.get_device_name(torch.cuda.current_device())
    for c in ids:
        n = per_ckpt[0][c][modes[0]]['pairs']
        print('class %d (%s): %d pairs, batch %d, %s%s' % (c, names[c - 1], n, args.batch_size, device,
                                                        ", augmented (train.py's chain, seed %d)" % args.seed if args.augment else ''))
        if n == 0:
            print('no kept pair: no loss')
            continue
        _print_checkpoints(ckpts, modes, {(i, m): r[c][m] for i, r in enumerate(per_ckpt) for m in modes},
                           {'trans': 1, 'rot': 1})                                      # config.yml:13-15
    return res


if __name__ == '__main__':
    main()
