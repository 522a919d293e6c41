"""tests/golden/group_matching.npz: the reference's own group_matching_labels (stardist/matching.py:409-472) on the cases of
group_matching_cases.py under every (criterion, thresh) of RUNS, the reference's test_grouping data (the mask of
test_image_nuclei_2d, stardist/data/images/mask2d.tif, and its 6 shuffled / rolled frames), and intersection_over_union /
_true / _pred (:65-93) on overlap matrices of those cases -- run from /root/reference through tests/golden/_refpkg.py.
The regionprops stand-in is replaced by one that does not allocate per label value, so that ids up to 2^31 - 1 can be
painted.  Run in the build container: python tests/golden/make_group_matching.py"""
import os, sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import group_matching_cases as C


def _regionprops_sparse(label_image):
    """skimage.measure.regionprops restricted to label / slice, ascending label order"""
    from types import SimpleNamespace
    y = np.asarray(label_image)
    out = []
    for lab in np.unique(y[y > 0]):
        idx = np.nonzero(y == lab)
        sl = tuple(slice(int(i.min()), int(i.max()) + 1) for i in idx)
        out.append(SimpleNamespace(label=int(lab), slice=sl))
    return out


if __name__ == "__main__":
    import _refpkg
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from stardist_b200.io.tiff import imread
    rm = _refpkg.load("stardist.matching")
    rm.regionprops = _regionprops_sparse
    data = {}
    for name, ys in C.cases().items():
        arg = list(ys) if name.endswith('_list') else ys
        for k, f in enumerate(ys):
            data["in/%s/%d" % (name, k)] = np.asarray(f)
        for crit, thr in C.RUNS:
            data["out/%s/%s/%g" % (name, crit, thr)] = rm.group_matching_labels(arg, thresh=thr, criterion=crit)
        for p in range(len(ys) - 1):
            a, b = np.asarray(ys[p]).astype(np.int32), np.asarray(ys[p + 1]).astype(np.int32)
            ov = rm.label_overlap(rm.relabel_sequential(a)[0], rm.relabel_sequential(b)[0], check=False)
            data["overlap/%s/%d" % (name, p)] = ov
            for crit in ('iou', 'iot', 'iop'):
                data["%s/%s/%d" % (crit, name, p)] = rm.matching_criteria[crit](ov)
    y0 = imread("/root/reference/stardist/data/images/mask2d.tif")
    frames = C.grouping_frames(y0)
    data["grouping/mask"] = y0
    data["grouping/out"] = rm.group_matching_labels(frames)
    data["grouping/pair"] = rm.group_matching_labels([y0, C.shuffle_labels(y0, np.random.default_rng(1))])
    assert np.array_equal(data["grouping/out"].max(axis=(1, 2)), [183, 199, 215, 231, 247, 263])
    np.savez_compressed(os.path.join(HERE, "group_matching.npz"), **data)
    print("wrote group_matching.npz:", len(data), "arrays")
