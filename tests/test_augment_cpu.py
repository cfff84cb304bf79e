"""CPU: the augmentation header (csrc/augment.cuh) built for the host against cv2 / numpy, the oracle's store semantics, and the
Python-side parsing and refusals of the augmentation chain.  The device build of the same header is checked in
test_gpu_augment.py against oracle/augment_ref.py."""
import ctypes as C
import importlib
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

import augment_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = 'iros20-6d-pose-tracking_b200'
CSRC = os.path.join(ROOT, PKG, 'csrc')

SHIM = r'''
#include "augment.cuh"
using namespace se3tn::aug;
extern "C" {
void rgb2hsv_img(const uint8_t* in, uint8_t* out, long rows) {
    for (long i = 0; i < rows * kImg; ++i) rgb2hsv(in[3 * i], in[3 * i + 1], in[3 * i + 2], out + 3 * i);
}
void hsv2rgb_img(const uint8_t* in, uint8_t* out, long rows) {
    for (long i = 0; i < rows * kImg; ++i) hsv2rgb(in[3 * i], in[3 * i + 1], in[3 * i + 2], out + 3 * i, static_cast<int>(i % kImg));
}
void blur8(const uint8_t* in, uint8_t* out, int k) {      // one 176 x 176 x 3 image, the separable fixed-point passes
    static uint32_t h[kImg * kImg * 3];
    for (int r = 0; r < kImg; ++r) for (int c = 0; c < kImg; ++c) for (int ch = 0; ch < 3; ++ch) {
        uint32_t a = 0;
        for (int j = 0; j < k; ++j) a += blur_tap8(k, j) * in[(r * kImg + reflect101(c + j - k / 2, kImg)) * 3 + ch];
        h[(r * kImg + c) * 3 + ch] = a;
    }
    for (int r = 0; r < kImg; ++r) for (int c = 0; c < kImg; ++c) for (int ch = 0; ch < 3; ++ch) {
        uint32_t a = 0;
        for (int j = 0; j < k; ++j) a += blur_tap8(k, j) * h[(reflect101(r + j - k / 2, kImg) * kImg + c) * 3 + ch];
        out[(r * kImg + c) * 3 + ch] = blur_round8(a);
    }
}
void blur16(const uint16_t* in, uint16_t* out, int k) {
    static uint32_t h[kImg * kImg];
    for (int r = 0; r < kImg; ++r) for (int c = 0; c < kImg; ++c) {
        uint32_t a = 0;
        for (int j = 0; j < k; ++j) a += blur_tap16(k, j) * in[r * kImg + reflect101(c + j - k / 2, kImg)];
        h[r * kImg + c] = a;
    }
    for (int r = 0; r < kImg; ++r) for (int c = 0; c < kImg; ++c) {
        uint64_t a = 0;
        for (int j = 0; j < k; ++j) a += static_cast<uint64_t>(blur_tap16(k, j)) * h[reflect101(r + j - k / 2, kImg) * kImg + c];
        out[r * kImg + c] = blur_round16(a);
    }
}
void store(const double* x, uint8_t* u8, uint16_t* u16, long n) { for (long i = 0; i < n; ++i) { u8[i] = store_u8(x[i]); u16[i] = store_u16(x[i]); } }
void philox_words(const uint32_t* c, const uint32_t* k, uint32_t* out) {
    const U4 r = philox({c[0], c[1], c[2], c[3]}, k[0], k[1]);
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}
}
'''


@pytest.fixture(scope='module')
def shim(tmp_path_factory):
    cxx = shutil.which('g++') or shutil.which('c++')
    if cxx is None:
        pytest.fail('a host C++ compiler is needed to build the augmentation header for the host')
    d = tmp_path_factory.mktemp('augshim')
    src, so = d / 'shim.cpp', d / 'shim.so'
    src.write_text(SHIM)
    subprocess.run([cxx, '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-I' + CSRC, str(src), '-o', str(so)], check=True)
    lib = C.CDLL(str(so))
    for name in ('rgb2hsv_img', 'hsv2rgb_img'):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_long]
    lib.blur8.argtypes = lib.blur16.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.store.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long]
    lib.philox_words.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def all_triples():
    """every uint8 triple, as images 176 pixels wide (the crops' width: cv2 treats the last 16 pixels of a row apart)"""
    a = np.arange(1 << 24, dtype=np.uint32)
    t = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8)
    rows = -(-len(t) // 176)
    img = np.zeros((rows * 176, 3), np.uint8)
    img[:len(t)] = t
    return img.reshape(rows, 176, 3), t


def test_rgb2hsv_all_triples(shim):
    img, _ = all_triples()
    out = np.empty_like(img)
    shim.rgb2hsv_img(_p(img), _p(out), img.shape[0])
    assert np.array_equal(out, cv2.cvtColor(img, cv2.COLOR_RGB2HSV))


def test_hsv2rgb_all_stored_triples_every_column(shim):
    img, _ = all_triples()
    out = np.empty_like(img)
    for src in (img, np.ascontiguousarray(np.roll(img, 160, axis=1)), np.ascontiguousarray(np.roll(img, 16, axis=1))):
        shim.hsv2rgb_img(_p(src), _p(out), src.shape[0])
        ref = cv2.cvtColor(src, cv2.COLOR_HSV2RGB)
        assert np.array_equal(out, ref), int((out != ref).any(-1).sum())


@pytest.mark.parametrize('k', [3, 5, 7])
def test_gaussian_blur_bit_exact(shim, k):
    rng = np.random.default_rng(k)
    imgs8 = [rng.integers(0, 256, (176, 176, 3), dtype=np.uint8), np.full((176, 176, 3), 255, np.uint8),
             (rng.integers(0, 2, (176, 176, 3)) * 255).astype(np.uint8), np.zeros((176, 176, 3), np.uint8)]
    imgs8[3][0, :] = 255; imgs8[3][:, -1] = 255
    for im in imgs8:
        out = np.empty_like(im)
        shim.blur8(_p(im), _p(out), k)
        assert np.array_equal(out, cv2.GaussianBlur(im, (k, k), sigmaX=2))
    imgs16 = [rng.integers(0, 65536, (176, 176), dtype=np.uint16), np.full((176, 176), 65535, np.uint16),
              (rng.integers(0, 2, (176, 176)) * 65535).astype(np.uint16), rng.integers(0, 3000, (176, 176)).astype(np.uint16)]
    for im in imgs16:
        out = np.empty_like(im)
        shim.blur16(_p(im), _p(out), k)
        assert np.array_equal(out, cv2.GaussianBlur(im, (k, k), sigmaX=2))


def test_float64_store_semantics(shim):
    """numpy's x86-64 store of float64 into uint8 / uint16 arrays (GaussianNoise's rgbB[mask] = rgbB[mask] + noise[mask]) is
    the header's store_u8 / store_u16 and the oracle's store()."""
    x = np.concatenate([np.arange(-70000, 70000, 0.25), [255.9, 256.0, 256.4, -0.5, -1.5, 65535.7, 65536.2, -9999.0, 511.0, -257.2]])
    u8, u16 = np.empty(len(x), np.uint8), np.empty(len(x), np.uint16)
    shim.store(_p(x), _p(u8), _p(u16), len(x))
    a8, a16 = np.zeros(len(x), np.uint8), np.zeros(len(x), np.uint16)
    with np.errstate(invalid='ignore', over='ignore'):
        a8[np.ones(len(x), bool)] = x
        a16[np.ones(len(x), bool)] = x
    assert np.array_equal(u8, a8) and np.array_equal(u16, a16)
    assert np.array_equal(R.store(x, np.uint8), a8) and np.array_equal(R.store(x, np.uint16), a16)
    assert a8[-8] == 0 and a8[-6] == 255 and a16[-3] == R.DEPTH_COVER        # 256.4 -> 0, -1.5 -> 255, -9999 -> 55537


def test_philox_known_answers(shim):
    """Philox4x32-10's known-answer vectors (Random123)."""
    out = np.zeros(4, np.uint32)
    for ctr, key, want in (([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
                           ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
                           ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
                            [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])):
        shim.philox_words(_p(np.array(ctr, np.uint32)), _p(np.array(key, np.uint32)), _p(out))
        assert out.tolist() == want


def test_cover_search_restates_the_reference_loop():
    m = np.zeros((176, 176), np.uint8)
    m[100:150, 100:150] = 1
    # the object sits bottom right of (105, 105): covering quadrant 3 there leaves too little, quadrant 0 (next cyclically) is kept
    assert R.cover_search(m, [(105, 105, 3)]) == (105, 105, 0, 1)
    # segB values of 255: no pixel equals 1, so no cover is ever kept (the reference loops forever)
    assert R.cover_search(m * 255, [(120, 120, 3), (5, 5, 0)]) is None


def _da():
    return importlib.import_module(PKG + '.data_augmentation')


def test_chain_parsing_and_refusals():
    A = _da()
    U = importlib.import_module(PKG + '.Utils')
    import yaml
    cfg = {'data_augmentation': {'hsv_noise': [15, 15, 15], 'bright_mag': [0.5, 1.5], 'gaussian_noise': {'rgb': 2, 'depth': 5},
                                 'gaussian_blur_kernel': 6, 'depth_missing_percent': 0.4}}
    c = A.chain_config(A.from_config(yaml.safe_load(yaml.safe_dump(cfg))), seed=7)
    assert (c.hsv_jitter, c.change_bright, c.gaussian_noise, c.gaussian_blur, c.black_cover, c.depth_missing) == (1, 1, 1, 1, 1, 0)
    assert list(c.hsv_noise) == [15, 15, 15] and c.hsv_prob == 0.5 and list(c.bright_mag) == [0.5, 1.5]
    assert (c.noise_rgb, c.noise_depth, c.noise_prob, c.blur_max_kernel, c.blur_prob, c.cover_prob, c.seed) == (2, 5, 0.5, 6, 0.4, 0.2, 7)
    sub = A.chain_config(U.Compose([A.ChangeBright(mag=[0.8, 1.2]), A.BlackCover(prob=0.2)]))
    assert (sub.hsv_jitter, sub.change_bright, sub.black_cover) == (0, 1, 1)
    with pytest.raises(ValueError, match='train.py'):
        A.chain_config(U.Compose([A.BlackCover(), A.HSVJitter(15, 15, 15)]))
    with pytest.raises(ValueError, match='train.py'):
        A.chain_config(U.Compose([A.BlackCover(), A.BlackCover()]))
    with pytest.raises(ValueError, match='not one of'):
        A.chain_config(U.Compose([A.HSVJitter(15, 15, 15), object()]))
    with pytest.raises(NotImplementedError, match='DepthMissing'):
        A.DepthMissing(prob=0.5, missing_percent=0.4)
    with pytest.raises(NotImplementedError, match='TrackDataset'):
        A.HSVJitter(15, 15, 15)([None] * 7)
    with pytest.raises(NotImplementedError, match='TrackDataset'):
        U.Compose([A.GaussianBlur(6)])([None] * 7)


def test_trackdataset_takes_the_chain(tmp_path):
    A = _da()
    D = importlib.import_module(PKG + '.datasets')
    U = importlib.import_module(PKG + '.Utils')
    ds = D.TrackDataset(str(tmp_path), 'val', np.zeros(8), np.ones(8), None, U.Compose([A.HSVJitter(15, 15, 15)]), None, augment_seed=3)
    assert ds.augment.hsv_jitter == 1 and ds.augment.seed == 3
    with pytest.raises(NotImplementedError):
        D.TrackDataset(str(tmp_path), 'val', np.zeros(8), np.ones(8), pretransforms=U.Compose([]))
    with pytest.raises(ValueError):
        D.segB_plane(np.ones((176, 176), np.uint16))


def test_cli_refuses_augment_with_ycb_dir(capsys):
    P = importlib.import_module(PKG + '.problems')
    with pytest.raises(SystemExit):
        P.main(['--ycb_dir', '/nonexistent', '--augment', 'config.yml'])
    assert '--augment works with --val_dir only' in capsys.readouterr().err


def test_oracle_equals_the_reference_classes():
    """oracle/augment_ref.py against the reference's own data_augmentation classes run on recorded draws
    (tests/golden/golden_augment.npz, made by oracle/make_golden_augment.py): every branch, BlackCover retrying within a corner
    and across corners, wrapping noise, pairs without segB, and BlackCover's -9999 stored as numpy 1.x stores it."""
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'golden_augment.npz'))
    kinds = ('seg', 'none', 'two')
    retried = 0
    for i in range(int(g['n_cases'])):
        rgbB, depthB, maskB, _ = R.case_inputs(int(g['seed_%d' % i]), kinds[int(g['kind_%d' % i])])
        p = g['params_%d' % i].copy()
        rng = np.random.default_rng(int(g['noise_seed_%d' % i]))
        noise_rgb = rng.standard_normal((176, 176, 3)) * p[R.NOISE_RGB_STD]
        noise_depth = rng.standard_normal((176, 176)) * p[R.NOISE_DEPTH_STD]
        if p[R.COVER_BRANCH]:
            u, v, q, used = R.cover_search(maskB, [tuple(c) for c in g['corners_%d' % i]])
            assert used == int(g['corners_used_%d' % i])
            p[R.COVER_U], p[R.COVER_V], p[R.COVER_QUADRANT] = u, v, q
            retried += used > 1 or q != g['corners_%d' % i][0][2]
        out = R.augment(rgbB, depthB, maskB, p, noise_rgb, noise_depth)
        for got, k in zip(out, ('rgbB', 'depthB', 'maskB')):
            assert np.array_equal(got, g['%s_%d' % (k, i)]), (i, k)
    assert retried >= 3


def test_philox_restatement_equals_the_header(shim):
    """augment_ref.philox (which replays the device's BlackCover corners in the GPU tests) is the header's Philox."""
    rng = np.random.default_rng(0)
    out = np.zeros(4, np.uint32)
    for _ in range(200):
        ctr = rng.integers(0, 1 << 32, 4, dtype=np.uint64).astype(np.uint32)
        key = rng.integers(0, 1 << 32, 2, dtype=np.uint64).astype(np.uint32)
        shim.philox_words(_p(ctr), _p(key), _p(out))
        assert list(R.philox(tuple(int(x) for x in ctr), tuple(int(x) for x in key))) == out.tolist()


def test_an_empty_chain_is_no_augmentation(tmp_path):
    A = _da()
    D = importlib.import_module(PKG + '.datasets')
    U = importlib.import_module(PKG + '.Utils')
    assert A.chain_config(U.Compose([])) is None
    assert D.TrackDataset(str(tmp_path), 'val', np.zeros(8), np.ones(8), None, U.Compose([]), None).augment is None
