"""Drop-in for the reference's train-time augmentations (data_augmentation.py:48-121, 217-267): HSVJitter, ChangeBright,
GaussianNoise, GaussianBlur and BlackCover with the reference's constructor arguments, and a refusing DepthMissing.

These objects describe a chain; they do not run on arrays.  A Utils.Compose of them in train.py:85-92's order (any subset) is
what TrackDataset(augmentations=...) and `problems --augment` take: the chain then runs on the device inside the validation step
(se3tn_eval_pairs_augmented), every random value drawn from Philox keyed by (seed, pair index), so a pair's augmentation depends
on the seed and its position in the dataset alone.  Given the draws, the arithmetic is the reference classes' bit for bit.
"""
from .engine import Engine

_DIRECT = ('%s is not applied to arrays here: pass a Utils.Compose of the augmentations to TrackDataset(augmentations=...), '
           'which runs them on the device inside the validation step')


class _Augmentation:
    def __call__(self, data):
        raise NotImplementedError(_DIRECT % type(self).__name__)


class HSVJitter(_Augmentation):
    def __init__(self, h_noise, s_noise, v_noise, prob=0.5):
        self.prob = prob
        self.h_noise = h_noise
        self.s_noise = s_noise
        self.v_noise = v_noise


class ChangeBright(_Augmentation):
    def __init__(self, prob=0.5, mag=[0.5, 1.5]):
        self.mag = mag                      # always applied: the reference ignores prob (data_augmentation.py:74-81)


class GaussianNoise(_Augmentation):
    def __init__(self, rgb_noise, depth_noise, prob=0.5):
        self.rgb_noise = rgb_noise
        self.depth_noise = depth_noise
        self.prob = prob


class GaussianBlur(_Augmentation):
    def __init__(self, max_kernel_size, min_kernel_size=3, prob=0.4):
        self.prob = prob
        self.max_kernel_size = max_kernel_size
        self.min_kernel_size = 3            # the reference ignores the argument (data_augmentation.py:109)


class BlackCover(_Augmentation):
    def __init__(self, prob=0.3):
        self.prob = prob


class DepthMissing(_Augmentation):
    """Commented out of the reference's chain (train.py:91): not supported."""
    def __init__(self, prob=0.5, missing_percent=0.5):
        raise NotImplementedError('DepthMissing is not supported: the reference trains without it (train.py:91 comments it out)')


ORDER = (HSVJitter, ChangeBright, GaussianNoise, GaussianBlur, BlackCover)   # train.py:85-92


def chain_config(augmentations, seed=0):
    """The se3tn_augment of a Utils.Compose (or a list) of the classes above, in train.py's order -> Engine.augment_config's
    structure, or None for an empty chain (the pairs are evaluated as they are).  Another order, a repeated or an unknown
    transform is a ValueError."""
    ts = list(getattr(augmentations, 'transforms', augmentations))
    pos = []
    for t in ts:
        if type(t) not in ORDER:
            raise ValueError('augmentations: %r is not one of %s' % (t, ', '.join(c.__name__ for c in ORDER)))
        pos.append(ORDER.index(type(t)))
    if pos != sorted(set(pos)):
        raise ValueError('augmentations must follow train.py:85-92, each at most once: %s'
                         % ' -> '.join(c.__name__ for c in ORDER))
    kw = {}
    for t in ts:
        if isinstance(t, HSVJitter):
            kw['hsv'] = dict(h=float(t.h_noise), s=float(t.s_noise), v=float(t.v_noise), prob=float(t.prob))
        elif isinstance(t, ChangeBright):
            kw['bright'] = dict(lo=float(t.mag[0]), hi=float(t.mag[1]))
        elif isinstance(t, GaussianNoise):
            kw['noise'] = dict(rgb=float(t.rgb_noise), depth=float(t.depth_noise), prob=float(t.prob))
        elif isinstance(t, GaussianBlur):
            kw['blur'] = dict(max_kernel=int(t.max_kernel_size), prob=float(t.prob))
        else:
            kw['cover'] = dict(prob=float(t.prob))
    return Engine.augment_config(seed=seed, **kw) if kw else None


def from_config(config):
    """train.py:85-92's chain from config.yml's data_augmentation block (a dict of the whole config or of the block)."""
    from .Utils import Compose
    c = config.get('data_augmentation', config)
    hsv = c['hsv_noise']
    return Compose([HSVJitter(hsv[0], hsv[1], hsv[2]),
                    ChangeBright(prob=0.5, mag=[c['bright_mag'][0], c['bright_mag'][1]]),
                    GaussianNoise(c['gaussian_noise']['rgb'], c['gaussian_noise']['depth']),
                    GaussianBlur(c['gaussian_blur_kernel']),
                    BlackCover(prob=0.2)])
