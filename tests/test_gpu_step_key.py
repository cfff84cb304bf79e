"""The CUDA graph key of a step (se3tn.cu StepKey): a call that differs from a captured step in any one value the step's kernels
are given must not replay that step's graph.  After a base call has been replayed, every keyed field is changed on its own, and
the result must equal, bit for bit, the same call on a context without graphs (SE3TN_GRAPH=0, read when a context is created)."""
import importlib
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TN, RN = 0.03, 5 * np.pi / 180
HW = (480, 640)
K = importlib.import_module('iros20-6d-pose-tracking_b200.synth').CAMERA_K
N = 5
IDS = (np.arange(N) % 2).astype(np.int32)


def _make_engine(pkg, synth):
    e = pkg.Engine(max_batch=64)
    mean, std = synth.default_mean_std()
    for wid in (0, 1):
        e.load_state_dict(synth.make_state_dict(wid), wid)
        e.set_mesh(synth.mesh(2 - wid, seed=wid), wid)
    e.set_stats(mean, std, 0)
    e.set_stats(mean + 1.5, std * 1.25, 1)
    return e


@pytest.fixture(scope='module')
def engines(pkg, synth):
    eng = _make_engine(pkg, synth)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv('SE3TN_GRAPH', '0')
        plain = _make_engine(pkg, synth)
    yield eng, plain
    eng.close()
    plain.close()


def _dev(e, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(e.device)


def _frame(synth, poses, seed):
    """synth.raw_frame with holes inside the tracks' windows, so that the depth fill changes what K0 reads."""
    rgb, depth = synth.raw_frame(seed)
    for p in poses:
        v, u = int(round(K[1, 1] * p[1, 3] / p[2, 3] + K[1, 2])), int(round(K[0, 0] * p[0, 3] / p[2, 3] + K[0, 2]))
        if 6 <= v < depth.shape[0] and 6 <= u < depth.shape[1]:
            depth[v - 6:v - 2, u - 6:u - 2] = 0
            depth[v:v + 24, u:u + 24] = 0
    return rgb, depth


def _nan_like(t):
    return torch.full_like(t, float('nan'))


def _roll(t):
    """t's tracks in another order, in a new tensor (through the host: torch has no CUDA roll for uint16)."""
    return torch.from_numpy(np.roll(t.cpu().numpy(), 1, 0)).to(t.device)


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


class Steps:
    """One kind of step run on the graph context (with the case's output tensors, so their addresses stay) and on the plain one
    (fresh outputs) with the same inputs.  `args` is the base call; check() changes some of its entries."""

    def __init__(self, engines, run, args):
        self.eng, self.plain = engines
        self.run, self.args = run, args
        for _ in range(2):
            run(self.eng, args, args['outs'])
        assert self.eng.last_step_was_graph()
        self.want_base = [x.clone() for x in run(self.plain, args, {})]

    def check(self, name, differs=True, **changes):
        a = dict(self.args, **changes)
        got = [x.clone() for x in self.run(self.eng, a, a['outs'])]
        want = self.run(self.plain, a, {})
        assert _equal(got, want), name
        assert self.eng.last_launch_count() == self.plain.last_launch_count(), name
        if differs:                                # or a step replayed with the old value would pass unnoticed
            assert not _equal(want, self.want_base), name + ': the change leaves the result as it was'

    def moved_outputs(self):
        for k in self.args['outs']:
            self.check('%s at a new address' % k, differs=False, outs=dict(self.args['outs'], **{k: _nan_like(self.args['outs'][k])}))

    def moved_ids(self):
        """wid_dev at a new address with the same ids; the old buffer then holds other ids, which a stale step would read."""
        old = self.args['wid_dev']
        new = old.clone()
        old.copy_(1 - old)
        try:
            self.check('wid_dev at a new address', differs=False, wid_dev=new)
        finally:
            old.copy_(new)

    def mixed_then_first_id(self):
        """The same wid_dev buffer with single-set ids: first the same first id (only the mix changes), then another one."""
        ids = self.args['wid_dev']
        try:
            for w, name in ((0, 'single ids against mixed'), (1, 'first weight id of a single set')):
                ids.fill_(w)
                self.check(name, wid=np.full(N, w, np.int32))
        finally:
            ids.copy_(_dev(self.eng, IDS))


def _track(e, a, outs):
    n = a['n']
    kw = dict(weight_ids_host=a['wid'][:n], weight_ids_dev=a['wid_dev'][:n], precision=a['prec'], fill_depth=a['fill'],
              **{k: v[:n] for k, v in outs.items()})
    if a['mode'] is None:
        return e.track_batch(a['R'], a['D'], a['K'], a['P'][:n], a['ow'][:n], a['ra'][:n], a['da'][:n], a['tn'], a['rn'], **kw)
    return e.track_render(a['R'], a['D'], a['K'], a['P'][:n], a['ow'][:n], a['tn'], a['rn'], mode=a['mode'], image_hw=a['hw'], **kw)


def _track_args(engines, synth, seed, **kw):
    eng = engines[0]
    poses = synth.raw_poses(N, seed=seed)
    rgb, depth = _frame(synth, poses, seed)
    P, ow, wid_dev = _dev(eng, poses), torch.full((N,), 200.0, dtype=torch.float64, device=eng.device), _dev(eng, IDS)
    ra, da = eng.render(K, P, ow, wid_dev)
    outs = dict(out_poses=torch.empty_like(P), out_trans=torch.empty(N, 3, device=eng.device), out_rot=torch.empty(N, 3, device=eng.device))
    a = dict(R=_dev(eng, rgb), D=_dev(eng, depth), K=K.copy(), P=P, ow=ow, ra=ra, da=da, wid=IDS.copy(), wid_dev=wid_dev, tn=TN, rn=RN,
             prec='bf16x3', mode=None, hw=None, fill=None, n=N, outs=outs)
    a.update(kw)
    return a


def test_track_batch_key(engines, synth):
    s = Steps(engines, _track, _track_args(engines, synth, seed=3))
    a, eng = s.args, s.eng
    for i, (r, c) in enumerate(((0, 0), (1, 1), (0, 2), (1, 2))):
        k = K.copy()
        k[r, c] += 9.0
        s.check('K[%d]' % i, K=k)
    s.check('tn', tn=TN * 1.5)
    s.check('rn', rn=RN * 1.5)
    s.check('n', n=N - 1)
    s.check('precision', prec='tf32')
    s.mixed_then_first_id()
    s.moved_outputs()
    rgb2, depth2 = _frame(synth, synth.raw_poses(N, seed=4), 4)
    s.check('frame rgb', R=_dev(eng, rgb2))
    s.check('frame depth', D=_dev(eng, depth2))
    s.check('poses', P=_dev(eng, synth.raw_poses(N, seed=4)))
    s.check('object_width', ow=torch.full_like(a['ow'], 230.0))
    s.check('rgbA', ra=_roll(a['ra']))
    s.check('depthA', da=_roll(a['da']))
    s.moved_ids()
    s.check('host ids at a new address', differs=False, wid=a['wid'].copy())


def test_track_render_key(engines, synth):
    s = Steps(engines, _track, _track_args(engines, synth, seed=5, mode='vispy'))
    s.check('render mode', mode='pyrender', hw=HW)
    s.check('render_H', mode='pyrender', hw=(HW[0] // 2, HW[1]))
    s.check('render_W', mode='pyrender', hw=(HW[0], HW[1] // 2))


def test_fill_key(engines, synth):
    s = Steps(engines, _track, _track_args(engines, synth, seed=6, fill=True))
    s.check('fill off', fill=None)
    s.check('max_depth', fill=dict(max_depth=1.5))
    s.check('extrapolate', fill=dict(extrapolate=True))
    s.check('blur_type', fill=dict(blur_type='gaussian'))


def _eval(e, a, outs):
    n = a['n']
    r = e.eval_pairs(*(a[k][:n] for k in ('rgbA', 'depthA', 'rgbB', 'depthB', 'A', 'B')), a['tn'], a['rn'],
                     weight_ids_host=a['wid'][:n], weight_ids_dev=a['wid_dev'][:n], precision=a['prec'], want_terms=True, want_labels=True,
                     **{k: (v if k == 'out_sums' else v[:n]) for k, v in outs.items()})
    return list(r)


def test_eval_pairs_key(engines, synth):
    eng = engines[0]
    a = synth.raw_poses(N, seed=7)
    b, c, s3 = a.copy(), np.cos(0.05), np.sin(0.05)
    b[:, :3, :3] = np.array([[c, -s3, 0], [s3, c, 0], [0, 0, 1]]) @ a[:, :3, :3]      # B: turned and moved, so both labels are non-zero
    b[:, :3, 3] += (0.004, -0.003, 0.006)
    A, B = _dev(eng, a), _dev(eng, b)
    ow, wid_dev = torch.full((N,), 200.0, dtype=torch.float64, device=eng.device), _dev(eng, IDS)
    rgbA, depthA = eng.render(K, A, ow, wid_dev)
    rgbB, depthB = eng.render(K, B, ow, wid_dev)
    outs = dict(out_trans=torch.empty(N, 3, device=eng.device), out_rot=torch.empty(N, 3, device=eng.device),
                out_sums=torch.empty(2, device=eng.device), out_sq=torch.empty(N, 6, device=eng.device),
                out_labels=torch.empty(N, 6, dtype=torch.float64, device=eng.device))
    s = Steps(engines, _eval, dict(rgbA=rgbA, depthA=depthA, rgbB=rgbB, depthB=depthB, A=A, B=B, wid=IDS.copy(), wid_dev=wid_dev,
                                   tn=TN, rn=RN, prec='bf16x3', n=N, outs=outs))
    s.check('tn', tn=TN * 1.5)
    s.check('rn', rn=RN * 1.5)
    s.check('n', n=N - 1)
    s.check('precision', prec='tf32')
    s.mixed_then_first_id()
    s.moved_outputs()
    for k in ('rgbA', 'depthA', 'rgbB', 'depthB'):
        s.check(k, **{k: _roll(s.args[k])})
    s.check('A_in_cam', A=_roll(A))
    s.check('B_in_cam', B=_roll(B))
    s.moved_ids()
    s.check('host ids at a new address', differs=False, wid=IDS.copy())


def test_host_entry(engines, synth):
    eng, plain = engines
    poses = synth.raw_poses(N, seed=8)
    rgb, depth = _frame(synth, poses, 8)
    ra, da = (x.cpu().numpy() for x in eng.render(K, _dev(eng, poses), torch.full((N,), 200.0, dtype=torch.float64, device=eng.device), _dev(eng, IDS)))
    ow = np.full(N, 200.0)

    def run(e, p, tn, wid):
        return e.track_host(rgb, depth, K, p, ow, ra, da, tn, RN, weight_ids=wid, want_residuals=True)

    for _ in range(2):
        run(eng, poses, TN, IDS)
    assert eng.last_step_was_graph()
    moved = poses.copy()
    moved[:, :3, 3] += (0.003, -0.002, 0.004)
    for name, p, tn, wid in (('new pose values', moved, TN, IDS), ('host ids at a new address', poses, TN, IDS.copy()),
                             ('tn', poses, TN * 1.5, IDS), ('single ids', poses, TN, np.zeros(N, np.int32))):
        got = run(eng, p, tn, wid)
        assert eng.last_step_was_graph(), name
        want = run(plain, p, tn, wid)
        assert all(np.array_equal(x, y) for x, y in zip(got, want)), name
