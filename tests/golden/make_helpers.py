"""tests/golden/helpers.npz: the reference's own mask_to_categorical and sample_points (stardist/utils.py:156-177, 318-380),
sample_patches / get_valid_inds (stardist/sample_patches.py) and the reference extension's c_dist_to_volume /
c_dist_to_centroid (stardist3d.cpp:146-234) on the cases of helpers_cases.py, run from /root/reference through
tests/golden/_refpkg.py with a seeded np.random; the np.random state after each draw is recorded.  csbdeep's `choice`, which
sample_patches imports, is csbdeep 0.8.1's, as restated in stardist_b200/models/data.py.
Run in the build container: python tests/golden/make_helpers.py"""
import json, os, sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import helpers_cases as C


def _state(data, key):
    _, k, pos, has_gauss, cached = np.random.get_state()
    data[key + "/key"], data[key + "/pos"] = k, np.int64(pos)
    data[key + "/gauss"] = np.array([has_gauss, cached], np.float64)


if __name__ == "__main__":
    import _refpkg
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    _refpkg.setup()
    from stardist_b200.models.data import choice
    sys.modules["csbdeep.utils"].choice = choice
    ru = _refpkg.load("stardist.utils")
    rs = _refpkg.load("stardist.sample_patches")
    ext = sys.modules["stardist.lib.stardist3d"]
    data = {}
    for name, (y, n, cls) in C.categorical_cases().items():
        m, d = ru.mask_to_categorical(y, n, cls, return_cls_dict=True)
        data["m2c/%s/out" % name] = m
        data["m2c/%s/cls_dict" % name] = np.array(json.dumps([[k, [int(l) for l in v]] for k, v in d.items()]))
    for name, (n, mask, prob, b, seed) in C.sample_points_cases().items():
        np.random.seed(seed)
        data["sp/%s/out" % name] = ru.sample_points(n, mask, prob=prob, b=b)
        _state(data, "sp/%s/state" % name)
    for name, (datas, ps, n, vi, seed) in C.sample_patches_cases().items():
        img = datas[0]
        if vi is not None:
            v = rs.get_valid_inds(img, ps, None if vi == 'plain' else C.FILTERS[vi])
            for a, va in enumerate(v):
                data["vi/%s/%d" % (name, a)] = va
            vi = v
        np.random.seed(seed)
        try:
            res = rs.sample_patches(datas, ps, n, valid_inds=vi)
            for k, r in enumerate(res):
                data["spa/%s/out/%d" % (name, k)] = r
        except ValueError as e:
            data["spa/%s/error" % name] = np.array(str(e))
        _state(data, "spa/%s/state" % name)
    for name, (d, rays) in C.dist_cases().items():
        v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
        data["dist/%s/verts" % name], data["dist/%s/faces" % name] = v, f
        data["dist/%s/volume" % name] = ext.c_dist_to_volume(d, v, f)
        data["dist/%s/centroid_abs" % name] = ext.c_dist_to_centroid(d, v, f, np.int32(1))
        data["dist/%s/centroid_rel" % name] = ext.c_dist_to_centroid(d, v, f, np.int32(0))
    np.savez_compressed(os.path.join(HERE, "helpers.npz"), **data)
    print("wrote helpers.npz:", len(data), "arrays")
