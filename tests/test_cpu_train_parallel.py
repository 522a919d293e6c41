"""Data-parallel training without a GPU: the reduction rule (tests/train_parallel_oracle.py) on hand cases, and train() in a
gloo world of 2 up to its first device call -- the divisibility check of the global batch and the broadcast of numpy's
random state."""
import os, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from train_parallel_oracle import replica_reduce_np, run_world

TINY = np.float32(2.0 ** -24)


def _rows(grads, skipped, n_out=4):
    """[W][P + n_out] rows: gradient values, then (loss, prob_loss, dist_loss, skipped) with loss = 10 r + 1 etc."""
    W, P = len(grads), len(grads[0])
    rows = np.zeros((W, P + n_out), np.float32)
    for r in range(W):
        rows[r, :P] = grads[r]
        rows[r, P:P + 3] = (10 * r + 1, 10 * r + 2, 10 * r + 3)
        rows[r, P + 3] = skipped[r]
        if n_out > 4:
            rows[r, P + 4:] = 10 * r + 5
    return rows


def test_sum_in_ascending_rank_order_then_one_division():
    """1 + 2^-24 rounds back to 1 (tie to even), so adding the two tiny values one by one to rank 0's 1 keeps 1; any other
    order, or a pairwise tree, gives 1 + 2^-23"""
    rows = _rows([[1.0, 3.0], [TINY, 3.0], [TINY, 3.0]], [0, 0, 0])
    g, out, st = replica_reduce_np(rows, 2, 4, (0, 0, 0))
    assert g.dtype == np.float32
    assert g[0] == np.float32(1) / np.float32(3) and g[0] != (np.float32(1) + np.float32(2 * TINY)) / np.float32(3)
    assert g[1] == np.float32(3)
    assert np.array_equal(out, np.float32([11 + 21 + 1, 12 + 22 + 2, 13 + 23 + 3, 0]) / np.float32(3))
    assert tuple(st) == (1, 0, 0)


def test_only_replicas_with_a_labelled_pixel_count():
    rows = _rows([[1.0, -2.0], [100.0, 100.0], [3.0, 4.0], [np.nan, np.inf]], [0, 1, 0, 1])
    g, out, st = replica_reduce_np(rows, 2, 4, (5, 2, 1))
    assert np.array_equal(g, np.float32([2.0, 1.0]))
    assert np.array_equal(out, np.float32([11.0, 12.0, 13.0, 0.0]))          # ranks 0 and 2: (1 + 21) / 2, ...
    assert tuple(st) == (6, 2, 0)                                            # one step, not skipped: t advances once


def test_one_replica_ok_is_its_row_exactly():
    g0 = np.float32([-0.0, 1e-38, 3.4e38, -7.25])
    rows = _rows([np.full(4, 9.0), g0], [1, 0], n_out=5)
    g, out, st = replica_reduce_np(rows, 4, 5, (0, 0, 0))
    assert np.array_equal(g.view(np.int32), g0.view(np.int32))               # x / 1, -0.0 kept
    assert np.array_equal(out, rows[1, 4:])
    assert tuple(st) == (1, 0, 0)


def test_no_replica_ok_is_a_skipped_step_over_all_rows():
    rows = _rows([[1.0], [2.0]], [1, 1])
    g, out, st = replica_reduce_np(rows, 1, 4, (3, 1, 0))
    assert g[0] == np.float32(1.5) and out[3] == 1
    assert tuple(st) == (3, 2, 1)                                            # t stays: Adam skips the step


def test_world_of_one_is_the_identity():
    rng = np.random.default_rng(0)
    for skipped in (0, 1):
        row = rng.standard_normal((1, 37 + 4)).astype(np.float32)
        row[0, 37 + 3] = skipped
        g, out, st = replica_reduce_np(row, 37, 4, (2, 0, 0))
        assert np.array_equal(g, row[0, :37]) and np.array_equal(out, row[0, 37:])
        assert tuple(st) == ((2, 1, 1) if skipped else (3, 0, 0))


# ------------------------------------------------------------------------------------------------ gloo world of 2
class _DeviceCall(Exception):
    pass


def _train_until_device(rank, world, batch_size, seed):
    """train() on a tiny 2-D model with the first device call (require_cuda) replaced by an exception: returns (what was
    raised, numpy's random state afterwards, whether CUDA was initialised)"""
    import torch
    from stardist_b200 import Config2D, StarDist2D, _lib
    def refuse():
        raise _DeviceCall()
    _lib.require_cuda = refuse
    np.random.seed(1000 + rank)                                  # the ranks start from different states
    rng = np.random.default_rng(3)
    X = [rng.uniform(0, 1, (64, 64)).astype(np.float32) for _ in range(2)]
    Y = [np.zeros((64, 64), np.int32) for _ in range(2)]
    for y in Y:
        y[10:20, 10:20] = 1
    config = Config2D(n_rays=8, unet_n_depth=1, grid=(1, 1), train_patch_size=(32, 32), train_batch_size=batch_size)
    model = StarDist2D(config, name=None, basedir=None)
    try:
        model.train(X, Y, validation_data=(X, Y), seed=seed, epochs=1, steps_per_epoch=1)
        raised = None
    except ValueError as e:
        raised = 'ValueError: %s' % e
    except _DeviceCall:
        raised = 'device'
    st = np.random.get_state()
    return raised, (st[0], st[1].tolist(), st[2], st[3], st[4]), torch.cuda.is_initialized()


def test_global_batch_not_divisible_by_the_world_raises_before_the_device(tmp_path):
    res = run_world(_train_until_device, 2, tmp_path, args=(3, None), timeout=300)
    for raised, _, cuda in res:
        assert raised is not None and raised.startswith('ValueError') and 'world size 2' in raised, raised
        assert not cuda


@pytest.mark.parametrize("seed", [None, 7])
def test_ranks_share_numpy_random_state_after_the_broadcast(tmp_path, seed):
    res = run_world(_train_until_device, 2, tmp_path, args=(2, seed), timeout=300)
    (r0, s0, c0), (r1, s1, c1) = res
    assert r0 == r1 == 'device' and not c0 and not c1
    assert s0 == s1
    # rank 0's own state without a seed (train() draws nothing before the device), else the seed's
    st = np.random.RandomState(1000 if seed is None else seed).get_state()
    assert s0 == (st[0], st[1].tolist(), st[2], st[3], st[4])
