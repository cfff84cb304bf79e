"""The fit check's rows (se3tn_track_opts.fit_tau_mm, include/se3tn.h) restated in numpy.

R: rendered depth of the model at the step's new pose, O: observed depth cropped at that pose's window (crop_bbox of the frame,
or of the filled frame), both uint16 mm of shape (..., 176, 176); tau: integer mm.  Per image, over the pixels with R > 0:
    model     #(R > 0)
    observed  #(R > 0, O > 0)
    inlier    #(R > 0, O > 0, |O - R| <= tau)
    front     #(R > 0, O > 0, O < R - tau)
    behind    #(R > 0, O > 0, O > R + tau)
    residual  sum of |O - R| over the inliers
-> int32 (..., 6) in that order."""
import numpy as np


def fit_rows(R, O, tau):
    R = np.asarray(R).astype(np.int64)
    O = np.asarray(O).astype(np.int64)
    if R.shape != O.shape:
        raise ValueError('R and O must have the same shape')
    tau = int(tau)
    m = R > 0
    ob = m & (O > 0)
    d = O - R
    inl = ob & (np.abs(d) <= tau)
    front = ob & (d < -tau)
    behind = ob & (d > tau)
    ax = (-2, -1)
    cols = [m.sum(ax), ob.sum(ax), inl.sum(ax), front.sum(ax), behind.sum(ax), np.where(inl, np.abs(d), 0).sum(ax)]
    return np.stack(cols, -1).astype(np.int32)
