"""The decode-ahead staging ring (staging.StagingRing) that validation and both one-pass drivers upload through.

  * items reach the device set in order and whole, for decode depths 1, 2 and 4, while the stream runs far behind the decoding
    (a host set rewritten before its last upload has left it would show up as a later item's index)
  * a job's exception is raised when its item is reached; no pool thread outlives the iteration, closed early or not
  * a row count uploads only those leading rows
"""
import contextlib, importlib, threading
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 24
SLEEP_CYCLES = 4_000_000                      # ~2 ms at the H100's 1.98 GHz: longer than a decode job by far


@pytest.fixture(scope='module')
def StagingRing():
    return importlib.import_module('iros20-6d-pose-tracking_b200.staging').StagingRing


def write(h, name, value):
    h[name].numpy()[...] = value
    return value


@pytest.mark.parametrize('depth', [1, 2, 4])
def test_every_item_reaches_the_device_in_order_while_uploads_lag(StagingRing, depth):
    dev = torch.device('cuda', torch.cuda.current_device())
    ring = StagingRing({'a': ((64, 3), torch.int32), 'b': ((64,), torch.int64)}, depth, dev)
    items = [[(write, 'a', k), (write, 'b', 1000 + k)] for k in range(N)]
    history_a = torch.empty((N, 64, 3), dtype=torch.int32, device=dev)
    history_b = torch.empty((N, 64), dtype=torch.int64, device=dev)
    got = []
    for k, values in enumerate(ring.uploads(items, 2 * depth)):
        got.append(values)
        history_a[k].copy_(ring.dev['a'])
        history_b[k].copy_(ring.dev['b'])
        torch.cuda._sleep(SLEEP_CYCLES)       # the next upload queues behind this: the host decodes far ahead of the stream
    torch.cuda.synchronize()
    assert got == [[k, 1000 + k] for k in range(N)]
    a, b = history_a.cpu().numpy(), history_b.cpu().numpy()
    assert (a == np.arange(N)[:, None, None]).all(), a[:, 0, 0]
    assert (b == 1000 + np.arange(N)[:, None]).all(), b[:, 0]


def test_a_job_error_is_raised_at_its_item_and_no_pool_thread_is_left(StagingRing):
    dev = torch.device('cuda', torch.cuda.current_device())
    ring = StagingRing({'x': ((4,), torch.int64)}, 2, dev)

    def job(h, k):
        if k == 3:
            raise ValueError('item 3 is unreadable')
        return write(h, 'x', k)
    before = set(threading.enumerate())
    got = []
    with pytest.raises(ValueError, match='item 3'):
        for values in ring.uploads([[(job, k)] for k in range(8)], 4):
            got.append(values[0])
    assert got == [0, 1, 2]
    assert [t for t in threading.enumerate() if t not in before] == []
    with contextlib.closing(ring.uploads([[(job, k)] for k in range(3)], 4)) as it:       # a consumer that stops early
        assert next(it) == [0]
    assert [t for t in threading.enumerate() if t not in before] == []


def test_a_row_count_uploads_only_those_rows(StagingRing):
    dev = torch.device('cuda', torch.cuda.current_device())
    ring = StagingRing({'x': ((6, 2), torch.float64)}, 2, dev)
    seen = []
    for _ in ring.uploads([[(write, 'x', 1.0)], [(write, 'x', 2.0)], [(write, 'x', 3.0)]], 2, rows=[6, 2, 4]):
        seen.append(ring.dev['x'][:, 0].cpu().tolist())
    assert seen == [[1.0] * 6, [2.0] * 2 + [1.0] * 4, [3.0] * 4 + [1.0] * 2]
