"""Label maps, anisotropies and connectivities of the edt_prob / fill_label_holes fixture (tests/golden/label_prep.npz,
make_label_prep.py) and tests."""
import os, sys
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import star_dist_cases as S

ANISO_2D = {"none": None, "scalar2": 2.0, "2,1": (2, 1), "1.7,0.9": (1.7, 0.9)}
ANISO_3D = {"none": None, "scalar2": 2.0, "2,1,1": (2, 1, 1), "1.73,1,1": (1.73, 1, 1)}
NON_DYADIC = ("1.7,0.9", "1.73,1,1")


def hole_smaller():
    """ring of label 50 around background and a smaller id (7) with its own hole"""
    m = np.zeros((24, 26), np.int32)
    m[3:20, 4:22] = 50; m[6:17, 7:19] = 0; m[8:14, 9:15] = 7; m[10:12, 11:13] = 0
    m[18:, 22:] = 3
    return m


def hole_larger():
    """ring of label 5 around a larger id (90): 90 survives inside 5's filled region"""
    m = np.zeros((22, 25), np.int32)
    m[2:19, 3:21] = 5; m[5:16, 6:18] = 0; m[7:14, 8:16] = 90; m[9:11, 10:12] = 0; m[0:2, 0:4] = 2
    return m


def ring_border_hole():
    """a ring closed by the image border: its hole touches the border and is not filled; a diagonal gap that only
    connectivity 2 crosses"""
    m = np.zeros((18, 20), np.int32)
    m[0:10, 3] = 4; m[0:10, 12] = 4; m[9, 3:13] = 4            # U against the top border
    m[12:17, 14:19] = 6; m[13:16, 15:18] = 0; m[12, 14] = 0; m[13, 15] = 6   # hole reachable only diagonally
    return m


def whole_box():
    """an object whose bounding box is the whole image (a frame), holding background and two other labels"""
    m = np.full((16, 19), 8, np.int32)
    m[2:-2, 2:-2] = 0; m[4:8, 4:9] = 3; m[9:13, 10:16] = 12; m[5, 14] = 0
    return m


def shell_3d():
    """3-D shell with a cavity holding background and a smaller label; a second object with a diagonal-only hole"""
    m = np.zeros((14, 15, 16), np.int32)
    m[1:12, 2:13, 2:14] = 9; m[3:10, 4:11, 4:12] = 0; m[5:8, 6:9, 6:9] = 2
    m[10:14, 11:15, 0:4] = 1; m[11:13, 12:14, 1:3] = 0; m[11, 12, 1] = 1; m[10, 11, 0] = 0
    return m


def maps_2d():
    d = S.maps_2d()
    d.update({"hole_smaller": hole_smaller(), "hole_larger": hole_larger(), "ring_border_hole": ring_border_hole(),
              "whole_box": whole_box(), "row": (S.ellipses_2d((1, 57), 6, seed=5) + (np.arange(57) % 9 == 0)).astype(np.int32),
              "column": S.ellipses_2d((49, 1), 5, seed=6)})
    return d


def maps_3d():
    d = S.maps_3d()
    d.update({"shell": shell_3d(), "thin": S.ellipsoids_3d((1, 30, 33), 5, seed=7)})
    return d


def dtype_maps():
    """the ellipses relabelled 1..n in each integer input dtype"""
    e = S.ellipses_2d()
    seq = np.unique(e, return_inverse=True)[1].reshape(e.shape)
    return {dt: seq.astype(dt) for dt in ("uint8", "uint16", "int32", "int64")}


def edt_cases():
    """key -> (map, anisotropy)"""
    out = {}
    for nd, maps, aniso in ((2, maps_2d(), ANISO_2D), (3, maps_3d(), ANISO_3D)):
        for name, m in maps.items():
            for aname, a in aniso.items():
                out["edt%d/%s/%s" % (nd, name, aname)] = (m, a)
    for dt, m in dtype_maps().items():
        out["edt2/dtype_%s/none" % dt] = (m, None)
    return out


def fill_cases():
    """key -> (map, connectivity)"""
    out = {}
    for nd, maps in ((2, maps_2d()), (3, maps_3d())):
        for name, m in maps.items():
            for c in range(1, nd + 1):
                out["fill%d/%s/%d" % (nd, name, c)] = (m, c)
    for dt, m in dtype_maps().items():
        out["fill2/dtype_%s/1" % dt] = (m, 1)
    return out


def stored_as_array(key, a):
    """small results and non-dyadic anisotropies are stored whole (the latter may differ by an ulp), the rest as sha256"""
    return a.size <= 4096 or key.rsplit("/", 1)[1] in NON_DYADIC
