"""tests/golden/matching.npz: the reference's own evaluation API -- stardist/matching.py matching (:109-230) with a tuple of
thresholds and report_matches, matching_dataset (:234-314) with by_image both ways, label_overlap (:38-52) -- for the three
criteria on the seeded label pairs of make_hostfuncs.label_pair, run from /root/reference through tests/golden/_refpkg.py.
Results are stored as JSON (field name -> value, float fields as float64) plus the dtype name of every scalar.
Run in the build container: python tests/golden/make_matching.py"""
import os, sys, json
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

SEEDS = (3, 4, 5)
THRESHS = (0.1, 0.3, 0.5, 0.7, 0.9)
CRITERIA = ('iou', 'iot', 'iop')


def pairs():
    from make_hostfuncs import label_pair
    out = [label_pair(s) for s in SEEDS]
    a, b = out[0]
    out.append((a, np.zeros_like(b)))                      # nothing predicted
    return out


def encode(t):
    """namedtuple -> {field: [value, type name]} (tuples of scores / pairs as lists)"""
    def one(v):
        if isinstance(v, tuple):
            return [one(x) for x in v]
        if isinstance(v, (np.floating, float)):
            return [float(v), type(v).__name__]
        if isinstance(v, (np.integer, int)) and not isinstance(v, bool):
            return [int(v), type(v).__name__]
        return [v, type(v).__name__]
    return {k: one(v) for k, v in t._asdict().items()}


if __name__ == "__main__":
    import _refpkg
    rm = _refpkg.load("stardist.matching")
    res = {}
    data = pairs()
    for crit in CRITERIA:
        for i, (a, b) in enumerate(data):
            res["matching/%s/%d" % (crit, i)] = [encode(m) for m in rm.matching(a, b, thresh=THRESHS, criterion=crit, report_matches=True)]
            res["matching_scalar/%s/%d" % (crit, i)] = encode(rm.matching(a, b, thresh=0.5, criterion=crit, report_matches=True))
        for by_image in (False, True):
            ys = [a for a, b in data]; ps = [b for a, b in data]
            res["dataset/%s/%d" % (crit, by_image)] = [encode(m) for m in rm.matching_dataset(ys, ps, thresh=THRESHS, criterion=crit,
                                                                                                 by_image=by_image, show_progress=False)]
    a, b = data[0]
    ov = rm.label_overlap(rm.relabel_sequential(a)[0], rm.relabel_sequential(b)[0])
    np.savez_compressed(os.path.join(HERE, "matching.npz"), results=np.frombuffer(json.dumps(res).encode(), np.uint8),
                        overlap=ov, overlap_dtype=np.frombuffer(str(ov.dtype).encode(), np.uint8))
    print("wrote matching.npz:", len(res), "entries")
