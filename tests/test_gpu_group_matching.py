"""group_matching_labels on the device: the device back-end (sdb_stack_labels, sdb_stack_overlap, sdb_stack_group_remap, the
shared host chaining) equals the reference's group_matching_labels (tests/golden/group_matching.npz) bit for bit, for numpy
and CUDA-tensor input; the batched overlap tables equal sdb_label_overlap pair by pair, also through the capacity retry and
in chunks of pairs; and a 20-frame 1024^2 stack groups like the host back-end."""
import os, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))
import group_matching_cases as C

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return np.load(os.path.join(HERE, "golden", "group_matching.npz"))


def _cuda_stack(ys):
    import torch
    return torch.from_numpy(np.ascontiguousarray(np.stack([np.asarray(y).astype(np.int32) for y in ys]))).cuda()


@pytest.mark.parametrize("name", sorted(C.cases()))
def test_device_backend_equals_reference(name, golden):
    from stardist_b200.matching import group_matching_labels, _device_ready
    assert _device_ready()
    ys = C.cases()[name]
    arg = list(ys) if name.endswith('_list') else ys
    stack = _cuda_stack(ys)
    for crit, thr in C.RUNS:
        want = golden["out/%s/%s/%g" % (name, crit, thr)]
        got = group_matching_labels(arg, thresh=thr, criterion=crit)
        assert isinstance(got, np.ndarray) and got.dtype == np.int32 and np.array_equal(got, want), (name, crit, thr)
        got_d = group_matching_labels(stack, thresh=thr, criterion=crit)
        assert got_d.is_cuda and str(got_d.dtype) == "torch.int32"
        assert np.array_equal(got_d.cpu().numpy(), want), (name, crit, thr)


def test_reference_grouping_on_device_without_host_copy(golden, monkeypatch):
    """the reference's test_grouping (tests/test_matching.py:35-54): 6 frames, each the previous one shuffled and rolled by
    15; a CUDA stack is grouped without copying it to the host (only tables far smaller than the stack leave the device)"""
    import torch
    from stardist_b200.matching import group_matching_labels
    y0 = golden["grouping/mask"]
    frames = C.grouping_frames(y0)
    stack = _cuda_stack(frames)
    copied = []
    cpu = torch.Tensor.cpu
    monkeypatch.setattr(torch.Tensor, "cpu", lambda t, *a, **k: (copied.append(t.numel()), cpu(t, *a, **k))[1])
    got = group_matching_labels(stack)
    monkeypatch.undo()
    assert got.is_cuda and max(copied) * 100 < stack.numel()
    got = got.cpu().numpy()
    assert np.array_equal(got, golden["grouping/out"])
    assert got.max(axis=(1, 2)).tolist() == [183, 199, 215, 231, 247, 263]
    pair = group_matching_labels([y0, C.shuffle_labels(y0, np.random.default_rng(1))])
    assert np.array_equal(pair, golden["grouping/pair"]) and np.array_equal(pair[0], pair[1])


def _random_stack(rng, T, shape, n):
    """frames of random blobs with random ids, some up to 2^31 - 1, so that the compacted ids differ from the labels"""
    frames = []
    for t in range(T):
        y = C._blobs(rng, shape, n)
        frames.append(C._renumber(rng, y, hi=C.INT32_MAX if t % 2 else 5000))
    return _cuda_stack(frames)


@pytest.mark.parametrize("capacity,pairs_per_chunk", [(None, None), (1, None), (None, 2), (3, 1)])
def test_stack_overlap_equals_label_overlap_pair_by_pair(golden, capacity, pairs_per_chunk):
    """capacity 1 forces the retry with the reported bound; pairs_per_chunk splits the pairs into several calls, each with
    its own pair field in the key"""
    from stardist_b200.matching import stack_labels_device, stack_overlap_device, label_overlap_device
    rng = np.random.default_rng(3)
    stack = _random_stack(rng, 7, (96, 80), 40)
    ids, offsets = stack_labels_device(stack, capacity=1 if capacity == 1 else 1 << 16)
    for f in range(stack.shape[0]):
        y = stack[f].cpu().numpy()
        assert np.array_equal(ids[offsets[f]:offsets[f + 1]], np.unique(y[y > 0]))
    tables = stack_overlap_device(stack, ids, offsets, capacity=capacity, pairs_per_chunk=pairs_per_chunk)
    assert len(tables) == stack.shape[0] - 1
    for p, (a, b, c) in enumerate(tables):
        pairs, counts = label_overlap_device(stack[p].contiguous(), stack[p + 1].contiguous())
        pairs, counts = pairs.cpu().numpy(), counts.cpu().numpy()
        ia, ib = ids[offsets[p]:offsets[p + 1]], ids[offsets[p + 1]:offsets[p + 2]]
        lab_a = np.where(a > 0, ia[np.maximum(a - 1, 0)], 0)
        lab_b = np.where(b > 0, ib[np.maximum(b - 1, 0)], 0)
        assert np.array_equal(lab_a, pairs[:, 0]) and np.array_equal(lab_b, pairs[:, 1]) and np.array_equal(c, counts), p


def test_negative_labels_raise_on_device(golden):
    import torch
    from stardist_b200.matching import group_matching_labels
    s = torch.zeros((3, 16, 16), dtype=torch.int32, device="cuda")
    s[2, 3, 4] = -5
    with pytest.raises(ValueError, match="ys must be an array of non-negative integers."):
        group_matching_labels(s)


def test_twenty_frames_of_1024_device_equals_host(golden):
    """T = 20 frames of 1024^2 (bench_data.ellipse_labels, rolled and relabelled per frame): device == host back-end"""
    from bench_data import ellipse_labels
    from stardist_b200.matching import group_matching_labels, _group_host
    rng = np.random.default_rng(0)
    base = ellipse_labels((1024, 1024), seed=1)
    frames = []
    for t in range(20):
        y = np.roll(base, (3 * t, 2 * t), axis=(0, 1))
        frames.append(C._renumber(rng, y, hi=10 ** 6).astype(np.int32))
    stack = np.stack(frames)
    got = group_matching_labels(stack)
    want = _group_host(stack, 1e-10, 'iou')
    assert np.array_equal(got, want)
    assert got[0].max() == stack[0].max() and len(np.unique(got[-1])) == len(np.unique(stack[-1]))
