"""Re-initialisation of lost tracks in numpy: the rules of se3tn_lost_tracks and se3tn_accept_starts (include/se3tn.h).

  Lost.    Track i is below in a step when 1000 * inlier < below_permille * model, compared as int64; model == 0 is below.  Its
           int32 streak becomes streak + 1 when below and 0 otherwise; the track is lost when the streak reaches `after`.
  Accept.  The start of a lost track replaces the tracked pose only when its init status is 0 and its fit row ranks strictly
           above the tracked row (better: inlier / model, then residual / inlier, int64 cross products; model = 0 and
           inlier = 0 rank last; a tie is not above).  The pose and the fit row are then both the start's.
  After an attempt the streak is 0 whatever the outcome.
  Events: 0 not below, 1 below and no attempt, 2 restarted, 3 no start (status != 0), 4 start rejected.
"""
import numpy as np

from hypotheses_ref import better   # the hypothesis choice's order: one definition, as in csrc/fit_rank.cuh

NONE, BELOW, RESTARTED, NO_START, REJECTED = 0, 1, 2, 3, 4


def below(rows, below_permille):
    """bool (n,): the tracks whose fit rows (n, 6) are below the threshold."""
    r = np.asarray(rows, dtype=np.int64)
    model, inlier = r[:, 0], r[:, 2]
    return (model == 0) | (1000 * inlier < np.int64(below_permille) * model)


def lost_tracks(rows, streak, below_permille, after):
    """-> (new streak int32 (n,), event int32 (n,) of 0 / 1, lost int64 (m,) ascending)."""
    b = below(rows, below_permille)
    streak = np.where(b, np.asarray(streak, dtype=np.int32) + 1, 0).astype(np.int32)
    event = b.astype(np.int32)
    lost = np.nonzero(b & (streak >= after))[0]
    return streak, event, lost


def accept_starts(lost, starts, init_rows, start_fit, poses, fit_rows, streak, event):
    """The accept rule over the starts of the tracks `lost` -> new (poses, fit_rows, streak, event); the inputs are not changed."""
    poses, fit_rows, streak, event = (np.array(a, copy=True) for a in (poses, fit_rows, streak, event))
    for k, i in enumerate(np.asarray(lost, dtype=np.int64)):
        if int(init_rows[k][0]) != 0:
            event[i] = NO_START
        elif better(start_fit[k], fit_rows[i]):
            event[i] = RESTARTED
            poses[i] = starts[k]
            fit_rows[i] = start_fit[k]
        else:
            event[i] = REJECTED
        streak[i] = 0
    return poses, fit_rows, streak, event

