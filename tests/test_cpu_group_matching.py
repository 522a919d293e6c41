"""group_matching_labels and intersection_over_* without a device: the host back-end (numpy overlaps, the shared chaining)
equals the reference's group_matching_labels (tests/golden/group_matching.npz) bit for bit, the three criteria equal the
reference's arrays, and every argument error is raised before any device call."""
import os, sys
import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))
import group_matching_cases as C


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "group_matching.npz"))


def _no_device(monkeypatch):
    from stardist_b200 import _lib, matching
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))
    monkeypatch.setattr(matching, '_device_ready', lambda: False)


@pytest.mark.parametrize("name", sorted(C.cases()))
def test_host_backend_equals_reference(name, golden, monkeypatch):
    from stardist_b200.matching import group_matching_labels
    _no_device(monkeypatch)
    ys = C.cases()[name]
    arg = list(ys) if name.endswith('_list') else ys
    for crit, thr in C.RUNS:
        want = golden["out/%s/%s/%g" % (name, crit, thr)]
        got = group_matching_labels(arg, thresh=thr, criterion=crit)
        assert got.dtype == want.dtype == np.int32
        assert np.array_equal(got, want), (name, crit, thr)
        for k, f in enumerate(ys):                                            # the input is left as it was
            assert np.array_equal(f, golden["in/%s/%d" % (name, k)])


def test_host_backend_reference_grouping(golden, monkeypatch):
    """the reference's test_grouping (tests/test_matching.py:35-54) on the nuclei mask"""
    from stardist_b200.matching import group_matching_labels
    _no_device(monkeypatch)
    y0 = golden["grouping/mask"]
    got = group_matching_labels(C.grouping_frames(y0))
    assert np.array_equal(got, golden["grouping/out"])
    assert got.max(axis=(1, 2)).tolist() == [183, 199, 215, 231, 247, 263]
    pair = group_matching_labels([y0, C.shuffle_labels(y0, np.random.default_rng(1))])
    assert np.array_equal(pair, golden["grouping/pair"]) and np.array_equal(pair[0], pair[1])


def test_intersection_over_equals_reference(golden):
    from stardist_b200 import matching as M
    fns = dict(iou=M.intersection_over_union, iot=M.intersection_over_true, iop=M.intersection_over_pred)
    n = 0
    for key in golden.files:
        if not key.startswith("overlap/"):
            continue
        ov = golden[key]
        rest = key[len("overlap/"):]
        for crit, fn in fns.items():
            want, got = golden["%s/%s" % (crit, rest)], fn(ov)
            assert got.dtype == want.dtype and np.array_equal(got, want), (crit, rest)
            assert np.array_equal(M._criterion_scores(ov, crit), want)
            n += 1
    assert n > 50
    zero = np.zeros((3, 4), np.int64)
    for fn in fns.values():
        assert fn(zero) is zero                                               # returned as it is (matching.py:67)
        with pytest.raises(ValueError, match="overlap must be an array of non-negative integers."):
            fn(zero.astype(np.float32))
        with pytest.raises(ValueError, match="overlap must be an array of non-negative integers."):
            fn(zero - 1)


def _errors():
    y = np.zeros((8, 9), np.int32)
    return [
        ([y], "'ys' must have 2 or more entries"),
        (np.zeros((1, 8, 9), np.int32), "'ys' must have 2 or more entries"),
        (np.zeros((2, 8, 9), np.float32), "ys must be an array of non-negative integers."),
        (np.full((2, 8, 9), -1, np.int32), "ys must be an array of non-negative integers."),
        (np.zeros(5, np.int32), "'ys' must be at least 2-dimensional"),
        ([y, y.astype(np.float64)], "ys must be an array of non-negative integers."),
        ([y, [[1, 2]]], "ys must be an array of non-negative integers."),
        ([y, y - 1], "ys must be an array of non-negative integers."),
        ((y, np.zeros((8, 8), np.int32)), "all label images must have the same shape"),
        (np.full((2, 3, 3), 2 ** 31, np.int64), "labels must be below 2\\^31"),
        ([y.astype(np.uint32), np.full((8, 9), 2 ** 32 - 1, np.uint32)], "labels must be below 2\\^31"),
        ([y, np.full((8, 9), 2 ** 40, np.uint64)], "labels must be below 2\\^31"),
    ]


@pytest.mark.parametrize("i", range(len(_errors())))
def test_argument_errors_before_the_device(i, monkeypatch):
    from stardist_b200.matching import group_matching_labels
    from stardist_b200 import _lib, matching
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))
    monkeypatch.setattr(matching, '_group_device', lambda *a: pytest.fail("device back-end reached"))
    ys, msg = _errors()[i]
    with pytest.raises(ValueError, match=msg):
        group_matching_labels(ys)


def test_criterion_and_tensor_errors_before_the_device(monkeypatch):
    import torch
    from stardist_b200.matching import group_matching_labels
    from stardist_b200 import _lib, matching
    monkeypatch.setattr(_lib, 'require_cuda', lambda: pytest.fail("device touched"))
    monkeypatch.setattr(matching, '_group_device', lambda *a: pytest.fail("device back-end reached"))
    with pytest.raises(ValueError, match="Matching criterion 'dice' not supported."):
        group_matching_labels(np.zeros((2, 4, 4), np.int32), criterion='dice')
    with pytest.raises(ValueError, match="contiguous CUDA int32 tensor"):
        group_matching_labels(torch.zeros((2, 4, 4), dtype=torch.int32))
    with pytest.raises(ValueError, match="'ys' must be at least 2-dimensional"):
        group_matching_labels(torch.zeros(4, dtype=torch.int32))


def test_ids_beyond_int32_raise(monkeypatch):
    """the reference's next_id is an np.int32 that wraps past 2^31 - 1; here the grouping raises instead"""
    from stardist_b200.matching import group_matching_labels
    _no_device(monkeypatch)
    ys = np.zeros((2, 6, 6), np.int64)
    ys[0, 0, 0] = 2 ** 31 - 2
    ys[1, 3:, 3:] = 1; ys[1, 0, 5] = 2                                        # two new objects: ids 2^31 - 1 and 2^31
    with pytest.raises(ValueError, match="more than 2\\^31 - 1 label ids"):
        group_matching_labels(ys)
    ys[1, 0, 5] = 0                                                            # one new object still fits
    assert group_matching_labels(ys)[1].max() == 2 ** 31 - 1
