"""Restatement of multi-hypothesis tracking (csrc/hypotheses.cu) in numpy / cv2: the start poses a hypothesis step draws around
each track's previous pose, and the rule that keeps one hypothesis per track.

The draws are the reference's random_gaussian_magnitude (Utils.py:372-404) with every uniform taken from Philox4x32-10
(augment_ref.philox): key = the seed, counter = (draw key low word, high word, h, slot).  Slot 0 holds the translation's
direction (U_theta from words x, y; U_phi from z, w), slot 1 the rotation axis', slots 2 + j and 66 + j the j-th N(0, max) draw of
the translation and rotation magnitudes (Box-Muller's first normal: sqrt(-2 ln(1 - u53(x, y))) cos(2 pi u53(z, w))).  The device
forms log, sqrt and sincospi with CUDA's functions, which may differ from numpy's in the last bits: the magnitudes agree to a few
ulps, the uniforms and try counts exactly.
"""
import math

import cv2
import numpy as np

from augment_ref import MASK32, philox

MAX_TRIES = 64
SLOT_DIR_T, SLOT_DIR_R, SLOT_MAG_T, SLOT_MAG_R = 0, 1, 2, 2 + MAX_TRIES
FIT_MODEL, FIT_INLIER, FIT_RESIDUAL = 0, 2, 5


def words(seed, key, h, slot):
    """The four Philox words of draw `slot` of hypothesis h of the track whose draw key is `key`."""
    key &= (1 << 64) - 1
    seed &= (1 << 64) - 1
    return philox((key & MASK32, key >> 32, h, slot), (seed & MASK32, seed >> 32))


def u53(a, b):
    return ((a >> 5) * 67108864.0 + (b >> 6)) * (1.0 / 9007199254740992.0)


def normal(w):
    """Box-Muller's first normal of one block of words."""
    u1 = 1.0 - u53(w[0], w[1])
    u2 = u53(w[2], w[3])
    return math.sqrt(-2.0 * math.log(u1)) * math.cos(2.0 * math.pi * u2)


def magnitude(seed, key, h, slot0, max_value):
    """np.random.normal(0, max) until |m| <= max, at most MAX_TRIES draws, then clamped -> (m, tries)."""
    m = 0.0
    for j in range(MAX_TRIES):
        m = max_value * normal(words(seed, key, h, slot0 + j))
        if abs(m) <= max_value:
            return m, j + 1
    return math.copysign(max_value, m), MAX_TRIES


def direction(u_theta, u_phi):
    """random_direction (Utils.py:393-404) of its two uniforms."""
    theta = u_theta * math.pi * 2
    phi = math.acos((2 * u_phi) - 1)
    return np.array([math.sin(phi) * math.cos(theta), math.sin(phi) * math.sin(theta), math.cos(phi)])


def draws(seed, key, h, max_t, max_r):
    """(U_theta_T, U_phi_T, U_theta_R, U_phi_R, m_T, m_R, tries_T, tries_R) of hypothesis h >= 1."""
    wt, wr = words(seed, key, h, SLOT_DIR_T), words(seed, key, h, SLOT_DIR_R)
    mt, tt = magnitude(seed, key, h, SLOT_MAG_T, max_t)
    mr, tr = magnitude(seed, key, h, SLOT_MAG_R, max_r)
    return (u53(wt[0], wt[1]), u53(wt[2], wt[3]), u53(wr[0], wr[1]), u53(wr[2], wr[3]), mt, mr, tt, tr)


def delta(d):
    """random_gaussian_magnitude's pose from its draws: translation direction * m_T, Rodrigues(axis / |axis| * m_R / 180 * pi)."""
    T = direction(d[0], d[1]) * d[4]
    axis = direction(d[2], d[3])
    axis = axis / np.linalg.norm(axis)
    rod = axis * d[5] / 180.0 * np.pi
    pose = np.eye(4)
    pose[:3, :3] = cv2.Rodrigues(rod)[0].reshape(3, 3)
    pose[:3, 3] = T
    return pose


def compose(P, D):
    """produce_train_pair_data.py:110: A_in_cam = B_in_cam . inv(B_in_A)."""
    return P.dot(np.linalg.inv(D))


def expand(poses, keys, S, seed, max_t, max_r):
    """(n,4,4) previous poses and n draw keys -> (n,S,4,4) starts and (n,S,8) draws; hypothesis 0 is the pose itself."""
    n = len(poses)
    out = np.zeros((n, S, 4, 4))
    dr = np.zeros((n, S, 8))
    for i in range(n):
        out[i, 0] = poses[i]
        for h in range(1, S):
            dr[i, h] = draws(seed, int(keys[i]), h, max_t, max_r)
            out[i, h] = compose(poses[i], delta(dr[i, h]))
    return out, dr


def better(x, y):
    """True when fit row x ranks strictly above row y: higher inlier / model (model = 0 last), then lower residual / inlier
    (inlier = 0 last), compared as exact integer cross products."""
    xm, ym, xi, yi, xr, yr = (int(v) for v in (x[FIT_MODEL], y[FIT_MODEL], x[FIT_INLIER], y[FIT_INLIER], x[FIT_RESIDUAL], y[FIT_RESIDUAL]))
    if (xm == 0) != (ym == 0):
        return ym == 0
    if xm and xi * ym != yi * xm:
        return xi * ym > yi * xm
    if (xi == 0) != (yi == 0):
        return yi == 0
    if xi and xr * yi != yr * xi:
        return xr * yi < yr * xi
    return False


def choose(rows):
    """rows (n,S,6) -> the kept hypothesis of each track; ties go to the lowest h."""
    rows = np.asarray(rows)
    out = np.zeros(len(rows), dtype=np.int32)
    for i, r in enumerate(rows):
        for h in range(1, len(r)):
            if better(r[h], r[out[i]]):
                out[i] = h
    return out
