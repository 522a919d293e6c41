"""tests/golden/star_dist.npz: the reference's own star_dist (stardist/geometry/geom2d.py:80-92), star_dist3D (geom3d.py:87-97),
relabel_image_stardist (geom2d.py:200-211), relabel_image_stardist3D (geom3d.py:201-217) and calculate_extents
(utils.py:180-193) on the maps and ray sets of star_dist_cases.py, run from /root/reference through tests/golden/_refpkg.py
with the reference's compiled C++ from oracle/_ref; the regionprops stand-in is extended here with `centroid`.

Stored: sha256 of every dense distance array (key -> [sha, shape]) as JSON; for the 2-D relabel the (dist, points) the
reference hands to polygons_to_label (captured by wrapping that call); the 3-D relabel maps; calculate_extents results.
Run in the build container: python tests/golden/make_star_dist.py"""
import os, sys, json
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import star_dist_cases as C

RAYS_2D = {"demo": (32, 61, 96), "ellipses": (7, 32, 61), "big_labels": (32,), "int8_negative": (32,)}
RELABEL_2D = (("demo", 32, (1, 1)), ("ellipses", 32, (1, 1)), ("ellipses", 64, (1, 1)), ("ellipses_odd", 32, (2, 2)),
              ("border", 32, (1, 1)), ("singles", 16, (1, 1)), ("big_labels", 32, (1, 1)), ("empty", 32, (1, 1)))
RELABEL_3D = (("ellipsoids", "gs32"), ("ellipsoids", "gs96"), ("border", "gs32"), ("big_labels", "gs32"))


def dense_entries(g2, g3):
    """key -> reference result of every dense case (also used by the CPU test that re-derives a few of them)"""
    rays = C.ray_sets()
    out = {}
    for name, m in C.maps_2d().items():
        for R in RAYS_2D.get(name, (32,)):
            for grid in C.GRIDS_2D:
                out["s2/%s/%d/%d,%d" % ((name, R) + grid)] = lambda m=m, R=R, grid=grid: g2.star_dist(m, R, grid=grid)
    for name, m in C.maps_3d().items():
        for rname, r in rays.items():
            for grid in C.GRIDS_3D:
                out["s3/%s/%s/%d,%d,%d" % ((name, rname) + grid)] = lambda m=m, r=r, grid=grid: g3.star_dist3D(m, r, grid=grid)
    return out


def regionprops(label_image):
    """the regionprops stand-in of _refpkg.py plus skimage's `centroid`: the mean of the region's pixel coordinates,
    coords.mean(axis=0)"""
    import _refpkg

    class Region(_refpkg._Region):
        @property
        def centroid(self):
            coords = np.argwhere(self.image) + np.array([s.start for s in self.slice])
            return tuple(coords.mean(axis=0))
    regs = _refpkg._regionprops(label_image)
    for r in regs:
        r.__class__ = Region
    return regs


def reference_modules():
    """the reference's geom2d, geom3d and utils, reading regions through `regionprops` above"""
    import _refpkg
    _refpkg.setup()
    import importlib
    mods = tuple(importlib.import_module(m) for m in ("stardist.geometry.geom2d", "stardist.geometry.geom3d", "stardist.utils"))
    sys.modules["skimage.measure"].regionprops = regionprops
    for m in mods:
        m.regionprops = regionprops
    return mods


def main():
    g2, g3, ut = reference_modules()
    hashes = {}
    for key, fn in dense_entries(g2, g3).items():
        d = fn()
        assert d.dtype == np.float32
        hashes[key] = [C.sha(d), list(d.shape)]
    arrays = {}
    # 2-D relabel: capture what reaches polygons_to_label
    captured = []
    orig = g2.polygons_to_label
    g2.polygons_to_label = lambda dist, points, shape: captured.append((dist, points)) or np.zeros(shape, np.int32)
    m2 = C.maps_2d()
    for i, (name, R, grid) in enumerate(RELABEL_2D):
        captured.clear()
        try:
            g2.relabel_image_stardist(m2[name], R, grid=grid)
            dist, points = captured[0]
            arrays["relabel2d/%d/dist" % i] = np.asarray(dist, np.float32)
            arrays["relabel2d/%d/points" % i] = np.asarray(points, np.int64)
        except IndexError:
            arrays["relabel2d/%d/raises" % i] = np.array(1)
    g2.polygons_to_label = orig
    rays = C.ray_sets()
    m3 = C.maps_3d()
    for i, (name, rname) in enumerate(RELABEL_3D):
        lbl = g3.relabel_image_stardist3D(m3[name], rays[rname])
        arrays["relabel3d/%d" % i] = np.asarray(lbl, np.int32)
    e2, e3 = C.maps_2d(), C.maps_3d()
    ext = {"ellipses": e2["ellipses"], "demo": e2["demo"], "border": e2["border"], "empty": e2["empty"],
           "ellipsoids": e3["ellipsoids"], "border3d": e3["border"], "big_labels3d": e3["big_labels"]}
    for k, m in ext.items():
        for fname, f in (("median", np.median), ("max", np.max)):
            arrays["extents/%s/%s" % (k, fname)] = np.asarray(ut.calculate_extents(m, f))
    arrays["extents/list/median"] = np.asarray(ut.calculate_extents([e2["ellipses"], e2["border"], e2["singles"]]))
    arrays["extents/stack/median"] = np.asarray(ut.calculate_extents(np.stack([e3["ellipsoids"], e3["big_labels"]])))
    np.savez_compressed(os.path.join(HERE, "star_dist.npz"), hashes=np.frombuffer(json.dumps(hashes, sort_keys=True).encode(), np.uint8),
                        **arrays)
    print("wrote star_dist.npz: %d dense hashes, %d arrays" % (len(hashes), len(arrays)))


if __name__ == "__main__":
    main()
