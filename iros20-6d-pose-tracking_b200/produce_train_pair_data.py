"""Drop-in for the reference's produce_train_pair_data.py: ProducerPurturb (reference produce_train_pair_data.py:58-141), which cuts
perturbed (A, B) pairs out of annotated frames, completeBlender (:145-226), its driver over a Blender data set, and a YCB-Video
mode that builds held-out pair folders from real key frames.  The folders are what TrackDataset and Problem.validate read
(`python -m <package>.problems --val_dir ...`); `problems --ycb_dir` scores the same pairs in one pass without writing them,
on the key-frame loop both share (ycbv_pair_steps).

What runs where:
  * host (numpy, the reference's own arithmetic): the perturbations B_in_A (Utils.random_gaussian_magnitude, in the reference's
    RNG draw order), A_in_cam = B_in_cam . inv(B_in_A), the projection-centre test with the float32 cam_K, and the thresholds of
    the visibility and segmentation checks;
  * device, one step per frame (Engine.perturb_pairs -> se3tn_perturb_pairs): compute_bbox of every A_in_cam, the model rendered
    at it in the pyrender mode over the whole camera image and cropped (what the reference's pyrender Renderer + crop_bbox
    give), and B, its depth and its segmentation cropped through the same window with each sample's segB pixel count;
  * device, the visibility check (Engine.visibility -> se3tn_visibility): #(seg == class id) and the covered pixels of the
    model's full-image render;
  * PNG / npz writes on a thread pool, finished before generate returns.

All num_sample offsets of a generate call are drawn before the device step; no check after the draws stops one, so the RNG
advances exactly as in the reference's loop.  A frame the visibility check rejects draws nothing, as in the reference.

Differences from the reference, on purpose:
  * current_seg=None is a ValueError (the reference fails later with UnboundLocalError, produce_train_pair_data.py:128);
  * the seg plane must be uint8 labels (the reference copies it into a uint8 canvas) and the depth is taken as uint16 mm;
  * textured .obj models: per-fragment texture lookups are replaced by per-vertex colours, the rasteriser's documented
    substitution (mesh_io.load_obj_mesh), as in tracking;
  * completeBlender's pair-name replacements touch basenames only (datasets.pair_paths), and its paths are arguments.

    python -m <package>.produce_train_pair_data --mode blender --data_folder OUT/ --dataset_info dataset_info.yml [--generated_data DIR]
    python -m <package>.produce_train_pair_data --mode ycbv --ycb_dir YCB --class_ids 1,2|all --train_data_path TPL --model_path TPL
                                                --outdir OUT [--num_sample 10] [--seed 0]
"""
import argparse
import glob
import os
import random
import shutil
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

from . import Utils
from .engine import Engine, IMAGE_SIZE
from .mesh_io import load_mesh

GLCAM_IN_CVCAM = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])


def _cam_K32(dataset_info):
    """produce_train_pair_data.py:69-74: float32, which the centre test, compute_bbox and the render all see."""
    K = np.zeros((3, 3)).astype(np.float32)
    cam = dataset_info['camera']
    K[0, 0] = cam['focalX']; K[1, 1] = cam['focalY']; K[0, 2] = cam['centerX']; K[1, 2] = cam['centerY']; K[2, 2] = 1
    return K


def visible_enough(num_visible, covered):
    """produce_train_pair_data.py:99-104 in float64: num_visible <= 100 or num_visible / covered < 0.1 rejects.  covered == 0 gives
    inf (numpy scalar division), which is kept, as in the reference."""
    if num_visible <= 100:
        return False
    with np.errstate(divide='ignore', invalid='ignore'):
        ratio = np.int64(num_visible) / np.float64(covered)
    return not (ratio < 0.1)


def frame_to_device(engine, rgb, depth, seg):
    """The three planes of one annotated frame as contiguous CUDA tensors (uint8 rgb, uint16 mm depth, uint8 labels)."""
    seg = np.asarray(seg)
    if seg.dtype != np.uint8 or seg.ndim != 2:
        raise ValueError('current_seg must be a uint8 (H, W) label image')
    dev = engine.device
    return (torch.from_numpy(np.ascontiguousarray(rgb, dtype=np.uint8)).to(dev),
            torch.from_numpy(np.ascontiguousarray(np.asarray(depth).astype(np.uint16))).to(dev),
            torch.from_numpy(np.ascontiguousarray(seg)).to(dev))


def visibility(engine, seg_dev, K32, rows):
    """rows: [(B_in_cam, mesh id, class id)] of one frame -> (visible, covered) int64 numpy arrays, max_batch rows per call."""
    vis, cov = [], []
    for i0 in range(0, len(rows), engine.max_batch):
        chunk = rows[i0:i0 + engine.max_batch]
        poses = torch.from_numpy(np.ascontiguousarray(np.stack([r[0] for r in chunk]), dtype=np.float64)).to(engine.device)
        v, c = engine.visibility(seg_dev, K32.astype(np.float64), poses, np.array([r[2] for r in chunk], np.int32),
                                 mesh_ids=np.array([r[1] for r in chunk], np.int32))
        vis.append(v.cpu().numpy()); cov.append(c.cpu().numpy())
    return np.concatenate(vis).astype(np.int64), np.concatenate(cov).astype(np.int64)


def pair_step(engine, frame_dev, K32, rows, on_device=False):
    """rows: [(A_in_cam, object width, mesh id, class id)] of one frame -> dict of host arrays rgbA, depthA, rgbB, depthB, segB,
    count (one row each), through Engine.perturb_pairs in chunks of max_batch.  on_device: nothing is copied back; -> a list of
    (first row, the chunk's perturb_pairs dict with its A_in_cam CUDA tensor added), one per chunk."""
    out = {k: [] for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'segB', 'count')}
    chunks = []
    rgb, depth, seg = frame_dev
    dev = engine.device
    for i0 in range(0, len(rows), engine.max_batch):
        chunk = rows[i0:i0 + engine.max_batch]
        A = torch.from_numpy(np.ascontiguousarray(np.stack([r[0] for r in chunk]), dtype=np.float64)).to(dev)
        ow = torch.tensor([float(r[1]) for r in chunk], dtype=torch.float64, device=dev)
        cid = torch.tensor([int(r[3]) for r in chunk], dtype=torch.int32, device=dev)
        res = engine.perturb_pairs(rgb, depth, seg, K32.astype(np.float64), A, ow, cid, mesh_ids=np.array([r[2] for r in chunk], np.int32))
        if on_device:
            chunks.append((i0, dict(res, A_in_cam=A)))
            continue
        for k in out:
            out[k].append(res[k].cpu().numpy())
    if on_device:
        return chunks
    return {k: np.concatenate(v) if v else None for k, v in out.items()}


def write_pair(out_dir, index, rgbA, rgbB, depthA, depthB, segB, A_in_cam, B_in_cam):
    """produce_train_pair_data.py:132-139: the files of pair `index` (%07d) under out_dir (a prefix, as the reference concatenates)."""
    from PIL import Image
    Image.fromarray(rgbA).save(out_dir + '%07drgbA.png' % index, optimize=True)
    Image.fromarray(rgbB).save(out_dir + '%07drgbB.png' % index, optimize=True)
    cv2.imwrite(out_dir + '%07ddepthA.png' % index, depthA)
    cv2.imwrite(out_dir + '%07ddepthB.png' % index, depthB)
    np.savez(out_dir + '%07dmeta.npz' % index, A_in_cam=A_in_cam, B_in_cam=B_in_cam)
    cv2.imwrite(out_dir + '%07dsegB.png' % index, segB)


class ProducerPurturb:
    """This can be used both as eval or purturb on training data to get large training set (produce_train_pair_data.py:58-59)."""

    def __init__(self, dataset_info, check_vis=False, engine=None, model=None, mesh_id=0, max_batch=64, workers=None):
        """model: the CAD model (a path or a mesh dict); default dataset_info['models'][0]['model_path'] with .ply -> .obj, as the
        reference loads it (:76).  engine: an Engine to share (one of max_batch rows per step is made otherwise)."""
        self.count = 0
        self.check_vis = check_vis
        self.dataset_info = dataset_info
        self.image_size = (self.dataset_info['resolution'], self.dataset_info['resolution'])
        if tuple(self.image_size) != (IMAGE_SIZE, IMAGE_SIZE):
            raise NotImplementedError('libse3tn is built for the reference resolution of 176 (dataset_info.yml:15)')
        self.object_width = dataset_info['object_width']
        self.cam_K = _cam_K32(dataset_info)
        if model is None:
            model = self.dataset_info['models'][0]['model_path'].replace('.ply', '.obj')
        self.mesh = load_mesh(model) if isinstance(model, str) else model
        self.engine = engine if engine is not None else Engine(max_batch=max_batch)
        self.mesh_id = int(mesh_id)
        self.engine.set_mesh(self.mesh, self.mesh_id)
        self.workers = workers or min(16, os.cpu_count() or 4)
        self.glcam_in_cvcam = GLCAM_IN_CVCAM

    # -- the host half, shared with the YCB-Video mode --------------------------------------------------------------------------
    def draw(self, B_in_cam, num_sample):
        """All num_sample offsets of one generate call (:108-116) -> [(A_in_cam, centre inside the image)], in draw order."""
        max_trans = self.dataset_info['max_translation']
        max_rot = self.dataset_info['max_rotation']
        H = self.dataset_info['camera']['height']
        W = self.dataset_info['camera']['width']
        out = []
        for _ in range(num_sample):
            B_in_A = Utils.random_gaussian_magnitude(max_trans, max_rot)
            A_in_cam = B_in_cam.dot(np.linalg.inv(B_in_A))
            projected = self.cam_K.dot(A_in_cam[:3, 3].reshape(3, 1)).reshape(-1)
            u = projected[0] / projected[2]
            v = projected[1] / projected[2]
            out.append((A_in_cam, not (u < 0 or u >= W or v < 0 or v >= H)))
        return out

    def keep(self, out_dir, B_in_cam, A_in_cams, res, first, class_id, pool, futures):
        """Queue the writes of the rows [first, first + len(A_in_cams)) of a pair step whose segB count reaches 100 (:128-141)."""
        for j, A_in_cam in enumerate(A_in_cams):
            k = first + j
            if res['count'][k] < 100:
                continue
            futures.append(pool.submit(write_pair, out_dir, self.count, res['rgbA'][k], res['rgbB'][k], res['depthA'][k], res['depthB'][k],
                                       res['segB'][k], A_in_cam, B_in_cam))
            self.count += 1

    def generate(self, out_dir, B_in_cam, current_rgb, current_depth, num_sample, class_id, current_seg=None, debug=False):
        """Take one real image and sample various purturbation around for evaluating the mean error (:86-141)."""
        if current_seg is None:
            raise ValueError('generate needs current_seg: the kept pairs are those whose B crop shows the object (:124-129)')
        H = self.dataset_info['camera']['height']
        W = self.dataset_info['camera']['width']
        if np.asarray(current_seg).shape != (H, W):
            raise ValueError('the frame must be the camera image of dataset_info (%d x %d)' % (H, W))
        B_in_cam = np.asarray(B_in_cam, dtype=np.float64)
        frame = frame_to_device(self.engine, current_rgb, current_depth, current_seg)
        if self.check_vis:
            vis, cov = visibility(self.engine, frame[2], self.cam_K, [(B_in_cam, self.mesh_id, class_id)])
            if not visible_enough(vis[0], cov[0]):
                return
        inside = [A for A, ok in self.draw(B_in_cam, num_sample) if ok]
        if not inside:
            return
        res = pair_step(self.engine, frame, self.cam_K, [(A, self.object_width, self.mesh_id, class_id) for A in inside])
        with ThreadPoolExecutor(max_workers=self.workers) as pool:
            futures = []
            self.keep(out_dir, B_in_cam, inside, res, 0, class_id, pool, futures)
            for f in futures:
                f.result()


def _blender_B_in_cam(meta, class_id):
    """produce_train_pair_data.py:196-200."""
    pos = np.where(meta['class_ids'] == class_id)
    return np.linalg.inv(GLCAM_IN_CVCAM).dot(np.linalg.inv(meta['blendercam_in_world']).dot(meta['poses_in_world'][pos, :, :].reshape(4, 4)))


def _sub(path, old, new):
    """str.replace on the basename only (see datasets.pair_paths)."""
    d, b = os.path.split(path)
    return os.path.join(d, b.replace(old, new))


def completeBlender(data_folder, dataset_info_path, generated_data=None, engine=None):
    """Domain Randomization (:145-226): one perturbed pair per Blender frame of class 0 into <data_folder>/train_data_blender_DR/,
    then the dataset's val_samples last pairs (in reverse name order) moved to <data_folder>/validation_data_blender_DR/ as %07d.
    generated_data: the Blender renders (*rgb.png, *depth.png, *seg.png, *poses_in_world.npz); default <data_folder>/../generated_data,
    where the reference keeps both next to its code.  data_folder is emptied first, as the reference does."""
    import yaml
    from PIL import Image
    class_id = 0
    data_folder = os.path.join(data_folder, '')
    if generated_data is None:
        generated_data = os.path.join(os.path.dirname(os.path.dirname(data_folder)), 'generated_data')
    shutil.rmtree(data_folder, ignore_errors=True)
    os.makedirs(data_folder)
    with open(dataset_info_path, 'r') as ff:
        dataset_info = yaml.safe_load(ff)
    if 'object_width' not in dataset_info:
        from .predict import compute_obj_max_width
        object_max_width = compute_obj_max_width(load_mesh(dataset_info['models'][0]['model_path'])['pos'].astype(np.float64))
        dataset_info['object_width'] = float(object_max_width + dataset_info['boundingbox'] / 100 * object_max_width)
        with open(os.path.join(data_folder, 'dataset_info.yml'), 'w') as ff:
            yaml.dump(dataset_info, ff)
    num_val = dataset_info['val_samples']
    out_train_path = data_folder + 'train_data_blender_DR/'
    out_val_path = data_folder + 'validation_data_blender_DR/'
    os.makedirs(out_train_path)
    os.makedirs(out_val_path)
    producer = ProducerPurturb(dataset_info, engine=engine)
    rgb_files = sorted(glob.glob(os.path.join(generated_data, '*rgb.png')))
    if not rgb_files:
        raise FileNotFoundError('no *rgb.png under %s' % generated_data)
    for rgb_file in rgb_files:
        meta = np.load(_sub(rgb_file, 'rgb.png', 'poses_in_world.npz'))
        B_in_cam = _blender_B_in_cam(meta, class_id)
        current_depth = cv2.imread(_sub(rgb_file, 'rgb', 'depth'), cv2.IMREAD_UNCHANGED)
        current_seg = cv2.imread(_sub(rgb_file, 'rgb', 'seg'), cv2.IMREAD_UNCHANGED).astype(np.uint8)
        if len(current_seg.shape) == 3:
            current_seg = current_seg[:, :, 0]
        if np.sum(current_seg == class_id) < 100:
            continue
        current_rgb = np.array(Image.open(rgb_file))[:, :, :3]
        producer.generate(out_train_path, B_in_cam, current_rgb, current_depth, num_sample=1, class_id=class_id,
                          current_seg=np.ascontiguousarray(current_seg))
    split_validation(out_train_path, out_val_path, num_val)
    return producer.count


def split_validation(out_train_path, out_val_path, num_val):
    """:215-226: the num_val last pairs in name order (newest first) moved to out_val_path as %07d, 0 upwards."""
    rgbA_files = sorted(glob.glob(out_train_path + '*rgbA.png'))
    rgbA_files.reverse()
    if num_val > len(rgbA_files):
        raise ValueError('val_samples = %d, but only %d pairs were produced' % (num_val, len(rgbA_files)))
    for i in range(num_val):
        f = rgbA_files[i]
        for old, new in (('rgbA', 'rgbA'), ('rgbA', 'rgbB'), ('rgbA', 'depthA'), ('rgbA', 'depthB'), ('rgbA.png', 'meta.npz'), ('rgbA', 'segB')):
            src = _sub(f, old, new)
            shutil.move(src, out_val_path + '%07d' % i + os.path.basename(src)[7:])


# ----------------------------------------------------------------------------------------------------
# YCB-Video: held-out pairs from the real key frames (image_sets/keyframe.txt), check_vis=True since real frames are occluded.
# Per frame: one visibility call for all its classes, then one pair step for every kept (class, sample) row.  Frames decode
# ahead through a StagingRing.  Output: <outdir>/<CADmodels folder of the class>/%07d*, one ProducerPurturb count per class.
# ----------------------------------------------------------------------------------------------------
def _by_frame(files):
    """{'%06d' frame number: path} of a sorted file list named <frame>... ('000001-color.png', '000001.txt')."""
    return {os.path.basename(f)[:6]: f for f in files}


def ycbv_keyframe_jobs(ycb_dir, class_ids):
    """[(rgb path, depth path, seg path, [(class id, B_in_cam)])] for every key frame with at least one requested class in its
    pose_gt/, in keyframe.txt order."""
    from .predict import read_keyframes
    jobs = []
    seq_files = {}
    for kf in read_keyframes(ycb_dir):
        if not kf:
            continue
        seq, frame = kf.split('/')
        base = os.path.join(ycb_dir, 'data_organized', seq)
        if not os.path.isdir(base):
            continue
        if seq not in seq_files:
            seq_files[seq] = dict(color=_by_frame(sorted(glob.glob(os.path.join(base, 'color', '*')))),
                                  depth=_by_frame(sorted(glob.glob(os.path.join(base, 'depth_filled', '*')))),
                                  seg=_by_frame(sorted(glob.glob(os.path.join(base, 'seg', '*')))),
                                  gt={c: _by_frame(sorted(glob.glob(os.path.join(base, 'pose_gt', str(c), '*')))) for c in class_ids})
        sf = seq_files[seq]
        rows = [(c, np.loadtxt(sf['gt'][c][frame]).reshape(4, 4)) for c in class_ids if frame in sf['gt'][c]]
        if not rows:
            continue
        for what in ('color', 'depth', 'seg'):
            if frame not in sf[what]:
                raise FileNotFoundError('key frame %s: no %s file under %s' % (kf, what, base))
        jobs.append((sf['color'][frame], sf['depth'][frame], sf['seg'][frame], rows))
    return jobs


def ycbv_producers(ycb_dir, class_ids, templates, eng, workers=None, mesh_base=0):
    """One check_vis ProducerPurturb per class on `eng`, its mesh under id = mesh_base + class id (mesh_base > 0 keeps the
    producers' meshes apart from the tracking meshes a step draws under the weight ids).  templates: {'train_data_path',
    'model_path'} with {class_id} / {class_name} placeholders, as --mode ycbv_all takes them; dataset_info.yml is read from
    <train_data_path>/../.  The classes of a frame share one step, so they must share the camera.  -> (CADmodels folder names,
    {class id: producer})."""
    import yaml
    from .predict import ycb_class_names, ycb_classes
    names = ycb_class_names(ycb_dir)
    producers = {}
    for c, name in ycb_classes(ycb_dir, class_ids):
        paths = {k: str(templates[k]).format(class_id=c, class_name=name) for k in ('train_data_path', 'model_path')}
        with open(os.path.join(paths['train_data_path'], '../dataset_info.yml'), 'r') as ff:
            info = yaml.safe_load(ff)
        producers[c] = ProducerPurturb(info, check_vis=True, engine=eng, model=paths['model_path'], mesh_id=mesh_base + c, workers=workers)
    first_id = min(producers)
    for c, p in producers.items():
        if p.dataset_info['camera'] != producers[first_id].dataset_info['camera']:
            raise ValueError('class %d: its camera differs from class %d\'s; the classes of a frame share one step' % (c, first_id))
    return names, producers


def ycbv_pair_steps(eng, producers, jobs, num_sample, decode_ahead=4, workers=None, on_device=False, with_frame=False):
    """The key-frame loop of the YCB-Video mode, shared by produce_ycbv (which writes the kept pairs) and problems.validate_ycbv
    (which scores them).  jobs: ycbv_keyframe_jobs.  Per frame, decoded ahead through a StagingRing: one visibility call for all
    its classes (it synchronises), then, per visible class in class order, `draw` of num_sample offsets, then one pair step for
    every sample inside the image.  Yields, per frame with such a sample, (owners, res): owners [(class id, B_in_cam, [A_in_cam
    of its rows], first row)] and res pair_step's result for the frame's rows (a list of device chunks with on_device).  A frame's
    device buffers are refilled once the loop resumes, so what res holds is consumed (or queued on the stream) before that.
    with_frame: yields (owners, res, (rgb, depth)) instead, the frame's device planes (the ring's: the same tensors every frame)."""
    from .predict import read_rgb, read_depth
    from .staging import StagingRing
    first = producers[min(producers)]
    H, W = int(first.dataset_info['camera']['height']), int(first.dataset_info['camera']['width'])
    K32 = first.cam_K

    def seg_into(h, path):
        s = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if s is None:
            raise FileNotFoundError(path)
        h['seg'].numpy()[...] = s if s.ndim == 2 else s[:, :, 0]

    def into(h, name, read, path):
        h[name].numpy()[...] = read(path)

    ring = StagingRing(dict(rgb=((H, W, 3), torch.uint8), depth=((H, W), torch.uint16), seg=((H, W), torch.uint8)), decode_ahead, eng.device)
    items = [[(into, 'rgb', read_rgb, j[0]), (into, 'depth', read_depth, j[1]), (seg_into, j[2])] for j in jobs]
    frame = (ring.dev['rgb'], ring.dev['depth'], ring.dev['seg'])
    for k, _ in enumerate(ring.uploads(items, workers or min(16, os.cpu_count() or 4))):
        rows = jobs[k][3]
        vis, cov = visibility(eng, frame[2], K32, [(B, producers[c].mesh_id, c) for c, B in rows])
        step, owners = [], []
        for (c, B), v, cv in zip(rows, vis, cov):
            if not visible_enough(v, cv):
                continue
            inside = [A for A, ok in producers[c].draw(B, num_sample) if ok]
            owners.append((c, B, inside, len(step)))
            step += [(A, producers[c].object_width, producers[c].mesh_id, c) for A in inside]
        if not step:
            continue
        res = pair_step(eng, frame, K32, step, on_device)
        yield (owners, res, frame[:2]) if with_frame else (owners, res)


def produce_ycbv(ycb_dir, class_ids, templates, outdir, num_sample=10, seed=0, max_batch=64, decode_ahead=4, workers=None):
    """The YCB-Video mode (see above).  templates: {'train_data_path', 'model_path'} with {class_id} / {class_name} placeholders, as
    --mode ycbv_all takes them; dataset_info.yml is read from <train_data_path>/../.  -> {class id: pairs written}."""
    class_ids = sorted(set(int(c) for c in class_ids))
    eng = Engine(max_batch=max_batch)
    names, producers = ycbv_producers(ycb_dir, class_ids, templates, eng, workers)
    outs = {}
    for c in class_ids:
        outs[c] = os.path.join(outdir, names[c - 1], '')
        os.makedirs(outs[c], exist_ok=True)
    random.seed(seed); np.random.seed(seed)
    jobs = ycbv_keyframe_jobs(ycb_dir, class_ids)
    with ThreadPoolExecutor(max_workers=workers or min(16, os.cpu_count() or 4)) as pool:
        futures = []
        for owners, res in ycbv_pair_steps(eng, producers, jobs, num_sample, decode_ahead, workers):
            for c, B, inside, at in owners:
                producers[c].keep(outs[c], B, inside, res, at, c, pool, futures)
            done = [f for f in futures if f.done()]
            for f in done:
                f.result()
            futures = [f for f in futures if not f.done()]
        for f in futures:
            f.result()
    return {c: producers[c].count for c in class_ids}


def main(argv=None):
    ap = argparse.ArgumentParser(description='Perturbed (A, B) training / validation pairs from annotated frames (the reference\'s '
                                             'produce_train_pair_data.py)')
    ap.add_argument('--mode', default='blender', choices=('blender', 'ycbv'))
    ap.add_argument('--data_folder', help='blender: output folder (emptied first)')
    ap.add_argument('--dataset_info', help='blender: dataset_info.yml')
    ap.add_argument('--generated_data', default=None, help='blender: the Blender renders (default <data_folder>/../generated_data)')
    ap.add_argument('--ycb_dir', help='ycbv: the YCB-Video root (data_organized/, image_sets/keyframe.txt, CADmodels/)')
    ap.add_argument('--class_ids', help='ycbv: comma-separated class ids, or all')
    ap.add_argument('--train_data_path', help='ycbv: path template ({class_id}, {class_name}); dataset_info.yml is read from its ../')
    ap.add_argument('--model_path', help='ycbv: path template of each class\'s mesh')
    ap.add_argument('--outdir', help='ycbv: output root; pairs go to <outdir>/<CADmodels folder>/')
    ap.add_argument('--num_sample', type=int, default=10)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--max_batch', type=int, default=64, help='samples per device step')
    args = ap.parse_args(argv)
    if args.mode == 'blender':
        if not args.data_folder or not args.dataset_info:
            raise SystemExit('--mode blender needs --data_folder and --dataset_info')
        n = completeBlender(args.data_folder, args.dataset_info, args.generated_data)
        print('%d pairs -> %s' % (n, args.data_folder))
        return n
    if not (args.ycb_dir and args.class_ids and args.train_data_path and args.model_path and args.outdir):
        raise SystemExit('--mode ycbv needs --ycb_dir, --class_ids, --train_data_path, --model_path and --outdir')
    from .predict import ycb_class_names
    ids = list(range(1, len(ycb_class_names(args.ycb_dir)) + 1)) if args.class_ids == 'all' else \
        [int(c) for c in args.class_ids.split(',')]
    counts = produce_ycbv(args.ycb_dir, ids, {'train_data_path': args.train_data_path, 'model_path': args.model_path}, args.outdir,
                          num_sample=args.num_sample, seed=args.seed, max_batch=args.max_batch)
    for c, n in sorted(counts.items()):
        print('class %d: %d pairs' % (c, n))
    return counts


if __name__ == '__main__':
    main()
