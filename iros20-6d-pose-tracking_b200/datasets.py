"""Drop-in for the reference's datasets.py: TrackDataset's file list, __len__ / __getitem__ (reference datasets.py:50-112),
processData and processPredict (datasets.py:115-175) with the same signatures and return structure, executed by libse3tn
kernels (K0 normalisation, K5 so(3) log, K6 pose update, the crop kernel's nearest-neighbour resize).

pretransforms must be None, as Tracker passes them (predict.py:191).  augmentations may be None or a Utils.Compose of
data_augmentation's classes in train.py:85-92's order (the reference builds its validation set with that chain, train.py:132):
input B is then augmented on the device, every draw keyed by (augment_seed, the pair's index in the sorted file list), so the
augmented loss is reproducible where the reference's is a random variable (DESIGN §9).

One deliberate difference: the reference derives a pair's other file names by str.replace on the WHOLE path of its rgbA file
(``path.replace('A', 'B')`` for rgbB, datasets.py:76), which also rewrites every 'A' in the directory names.  Here every
replacement applies to the file's basename only, so a folder such as /data/A_set/ works.
"""
import os
import glob
import cv2
import numpy as np
import torch


class TrackDataset:
    def __init__(self, root, mode, images_mean, images_std, pretransforms=None, augmentations=None,
                 posttransforms=None, dataset_info=None, trans_normalizer=0.03, rot_normalizer=5 * np.pi / 180,
                 engine=None, weight_id=0, precision='bf16x3', augment_seed=0):
        if pretransforms is not None:
            raise NotImplementedError('pretransforms are out of scope (inference passes None, predict.py:191)')
        from .data_augmentation import chain_config
        self.augment_seed = int(augment_seed)
        self.augment = chain_config(augmentations, self.augment_seed) if augmentations is not None else None
        self.root = root
        self.mode = mode
        self.images_mean = np.asarray(images_mean)
        self.images_std = np.asarray(images_std)
        self.pretransforms = None
        self.augmentations = augmentations
        # The reference composes OffsetDepth -> NormalizeChannels -> ToTensor here; that chain is
        # what the K0 kernel implements, so the object passed in is only kept for introspection.
        self.posttransforms = posttransforms
        self.dataset_info = dataset_info
        if dataset_info is not None:
            cam = dataset_info['camera']
            self.cam_K = np.array([[cam['focalX'], 0, cam['centerX']], [0, cam['focalY'], cam['centerY']], [0, 0, 1]])
        self.trans_normalizer = trans_normalizer
        self.rot_normalizer = rot_normalizer
        self.weight_id = weight_id
        self.precision = precision
        self._engine = engine
        self._stats_set = False
        self.rgbA_files = sorted(glob.glob(self.root + '/*rgbA.png')) if root else []

    def __len__(self):
        return len(self.rgbA_files)

    def __getitem__(self, index):
        """-> (data=[dataA, dataB], target=[trans_label, rot_label], A_in_cam, B_in_cam, rgbA, rgbB, maskA, maskB), reference
        datasets.py:70-112.  Crops that are not `resolution` x `resolution` are resized with cv2.INTER_NEAREST's mapping by the
        crop kernel on the device.  One pair at a time, as a DataLoader would ask for it; Problem.validate reads the same files
        and runs whole batches in one step instead."""
        if torch.utils.data.get_worker_info() is not None:
            raise RuntimeError('TrackDataset.__getitem__ runs CUDA kernels and cannot be called in a DataLoader worker process '
                               '(CUDA does not survive fork): use num_workers=0, or Problem.validate / Engine.eval_pairs, which '
                               'decode the pairs in threads and evaluate whole batches on the device')
        p = read_pair(self.rgbA_files[index])
        res = int(self.dataset_info['resolution'])
        rgbA, depthA, rgbB, depthB, maskB = p['rgbA'], p['depthA'], p['rgbB'], p['depthB'], p['segB']
        if rgbB.shape[0] != res:
            rs = [t.cpu().numpy() if t is not None else None for t in resize_pair(self.engine, p, res)]
            rgbA, depthA, rgbB, depthB, maskB = rs
        if maskB is None:
            maskB = (depthB > 100).astype(np.uint8)
        assert np.sum(maskB) > 0, 'index={}'.format(index)
        if self.augment is not None:
            rgbB, depthB, maskB = self._augment_item(index, rgbB, depthB, maskB)
        data, target, rgbA, rgbB, maskA, maskB = self.processData(rgbA, depthA, p['A_in_cam'], rgbB, depthB, p['B_in_cam'], maskB)
        return data, target, p['A_in_cam'], p['B_in_cam'], rgbA, rgbB, maskA, maskB

    def _augment_item(self, index, rgbB, depthB, maskB):
        """The augmentation chain on one pair's B on the device (se3tn_augment_crops), BlackCover's corner applied to maskB too."""
        eng = self.engine
        dev = eng.device
        seg = torch.from_numpy(segB_plane(maskB)[None]).to(dev)
        dB, idx = self._u16(depthB, dev), torch.tensor([index], dtype=torch.int64, device=dev)
        r, d = eng.augment_crops(self.augment, self._u8(rgbB, dev), dB, idx, segB=seg)
        params, _, _ = eng.augment_draws(self.augment, dB, idx, segB=seg)
        p = params[0].cpu().numpy()
        maskB = np.array(maskB, copy=True)
        if p[17] and p[20] >= 0:                         # the accepted cover: the quadrant of corner (u, v), include/se3tn.h
            u, v, q = int(p[18]), int(p[19]), int(p[20])
            maskB[(slice(None, v) if q < 2 else slice(v, None)), (slice(None, u) if q % 2 == 0 else slice(u, None))] = 0
        return r[0].cpu().numpy(), d[0].cpu().numpy(), maskB

    @property
    def engine(self):
        if self._engine is None:
            from .engine import Engine
            self._engine = Engine(max_batch=1)
        if not self._stats_set:
            self._engine.set_stats(self.images_mean, self.images_std, self.weight_id)
            self._stats_set = True
        return self._engine

    def processData(self, rgbA, depthA, A_in_cam, rgbB, depthB, B_in_cam, maskB=None, original_size=None):
        """-> (sample=[dataA, dataB] float32 CPU tensors (4,H,W), [trans_label, rot_label],
               rgbA_viz, rgbB_viz, maskA, maskB)   -- reference datasets.py:115-156."""
        eng = self.engine
        dev = eng.device
        maskA = (depthA > 100).astype(np.uint8)
        if maskB is None:
            maskB = (depthB > 100).astype(np.uint8)
        A_pose = torch.from_numpy(np.ascontiguousarray(A_in_cam, dtype=np.float64).reshape(1, 4, 4)).to(dev)
        B_pose = torch.from_numpy(np.ascontiguousarray(B_in_cam, dtype=np.float64).reshape(1, 4, 4)).to(dev)
        wid = torch.tensor([self.weight_id], dtype=torch.int32, device=dev)
        tA, tB = eng.normalize(self._u8(rgbA, dev), self._u16(depthA, dev), self._u8(rgbB, dev), self._u16(depthB, dev),
                               A_pose, weight_ids=wid, precision=self.precision, want_tensors=True)
        tl, rl = eng.so3_log(A_pose, B_pose, self.trans_normalizer, self.rot_normalizer)
        sample = [tA[0].cpu(), tB[0].cpu()]
        trans_label, rot_label = tl[0].cpu().numpy(), rl[0].cpu().numpy()
        if self.mode == 'train':
            assert (trans_label <= 1).all() and (trans_label >= -1).all()
            assert (rot_label >= -1).all() and (rot_label <= 1).all()
        return sample, [trans_label, rot_label], rgbA.astype(np.uint8), rgbB.astype(np.uint8), maskA, maskB

    def processPredict(self, A_in_cam, predB, original_size=None):
        """-> 4x4 float64 object pose in the camera frame -- reference datasets.py:159-175."""
        eng = self.engine
        dev = eng.device
        poses = torch.from_numpy(np.ascontiguousarray(A_in_cam, dtype=np.float64).reshape(1, 4, 4)).to(dev)
        trans = torch.as_tensor(np.asarray(predB[0], dtype=np.float32).reshape(1, 3)).to(dev)
        rot = torch.as_tensor(np.asarray(predB[1], dtype=np.float32).reshape(1, 3)).to(dev)
        return eng.pose_update(poses, trans, rot, self.trans_normalizer, self.rot_normalizer)[0].cpu().numpy()

    @staticmethod
    def _u8(a, dev):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint8)[None]).to(dev)

    @staticmethod
    def _u16(a, dev):
        return torch.from_numpy(np.ascontiguousarray(a).astype(np.uint16)[None]).to(dev)


def segB_plane(maskB):
    """BlackCover's maskB as the device takes it: a uint8 image (segB, or depthB > 100 as uint8).  A 16-bit segB is refused: the
    reference's cover test would compare its values before and after a uint8 cast."""
    m = np.asarray(maskB)
    if m.dtype == np.bool_:
        m = m.astype(np.uint8)
    if m.dtype != np.uint8 or m.shape != (176, 176):
        raise ValueError('augmentation needs maskB as a uint8 176 x 176 image (segB or depthB > 100), not %s %s' % (m.dtype, m.shape))
    return np.ascontiguousarray(m)


def pair_paths(rgbA_path):
    """The files of one training pair (reference datasets.py:76-82), named from its rgbA file; the replacements touch the basename
    only (see the module docstring)."""
    d, b = os.path.split(rgbA_path)
    j = lambda name: os.path.join(d, name)
    return dict(rgbA=rgbA_path, rgbB=j(b.replace('A', 'B')), depthA=j(b.replace('rgbA', 'depthA')), depthB=j(b.replace('rgbA', 'depthB')),
                segB=j(b.replace('rgbA', 'segB')), meta=j(b.replace('rgbA.png', 'meta.npz')))


def read_pair(rgbA_path):
    """Decode one pair from disk: rgb uint8 (h,w,3) in RGB order (what PIL gives the reference), depth uint16 mm, segB as stored or
    None when the file is missing, A_in_cam / B_in_cam float64 (4,4) from meta.npz.  Host only (cv2 releases the GIL), so it may
    run in threads.  The rgb crops must be 8-bit three-channel images, what the reference's data generator writes and what
    processData takes: an RGBA, grayscale or 16-bit rgb file is an error (PIL would hand the reference an array of another
    shape or depth, which its pipeline does not handle either)."""
    f = pair_paths(rgbA_path)

    def rgb(path):
        im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if im is None:
            raise FileNotFoundError(path)
        if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
            raise ValueError('%s: rgb crops must be 8-bit three-channel images, got %s %s' % (path, im.dtype, im.shape))
        return cv2.cvtColor(im, cv2.COLOR_BGR2RGB)

    def raw(path, required=True):
        if not required and not os.path.exists(path):
            return None
        im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if im is None:
            raise FileNotFoundError(path)
        return im

    meta = np.load(f['meta'])
    return dict(rgbA=rgb(f['rgbA']), rgbB=rgb(f['rgbB']), depthA=raw(f['depthA']), depthB=raw(f['depthB']), segB=raw(f['segB'], False),
                A_in_cam=np.asarray(meta['A_in_cam'], dtype=np.float64), B_in_cam=np.asarray(meta['B_in_cam'], dtype=np.float64))


def resize_nearest(engine, rgb, depth, size):
    """cv2.resize(..., (size, size), interpolation=cv2.INTER_NEAREST) of an rgb uint8 (h,w,3) and a uint16 (h,w) image, on the
    device: the crop kernel over a window that is the whole image uses the same floor(dst * src / dst_size) source index.
    Host or CUDA arrays in, CUDA tensors (size,size,3), (size,size) out."""
    dev = engine.device
    rgb = torch.as_tensor(np.ascontiguousarray(rgb) if isinstance(rgb, np.ndarray) else rgb).to(dev).contiguous()
    depth = torch.as_tensor(np.ascontiguousarray(depth) if isinstance(depth, np.ndarray) else depth).to(dev).contiguous()
    h, w = depth.shape
    window = torch.tensor([[[0, 0], [h, 0], [0, w], [h, w]]], dtype=torch.int32, device=dev)   # rows (v, u): the whole image
    r, d = engine.crop_bbox(rgb, depth, window, (size, size))
    return r[0], d[0]


def resize_pair(engine, pair, size):
    """datasets.py:95-101 on the device: rgbA / depthA, rgbB / depthB and segB (when present) resized to size x size.
    -> CUDA tensors rgbA, depthA, rgbB, depthB, segB (segB None when the pair has none)."""
    rgbA, depthA = resize_nearest(engine, pair['rgbA'], pair['depthA'], size)
    rgbB, depthB = resize_nearest(engine, pair['rgbB'], pair['depthB'], size)
    segB = None
    if pair['segB'] is not None:
        seg = pair['segB']
        if seg.ndim != 2 or seg.dtype not in (np.uint8, np.uint16):
            raise ValueError('segB must be a single-channel 8- or 16-bit image')
        _, s16 = resize_nearest(engine, pair['rgbB'], seg.astype(np.uint16), size)   # the mask rides in the depth plane
        segB = s16.to(torch.uint8) if seg.dtype == np.uint8 else s16
    return rgbA, depthA, rgbB, depthB, segB
