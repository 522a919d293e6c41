"""Host-side formats either side of the path: ImageJ ROI export, TIFF in/out, the command line parser."""
import hashlib, os, zipfile
import numpy as np
import pytest


def _golden():
    """seeded inputs and the reference's outputs on them (sha256), frozen by tests/golden/make_io_ref.py"""
    import json, sys
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, golden)
    import io_cases
    with open(os.path.join(golden, "io_ref.json")) as f:
        return io_cases, json.load(f)


def test_polyroi_bytes_golden_and_reference():
    from stardist_b200.io import rois
    x = np.array([10.2, 30.7, 25.1, 8.4]); y = np.array([5.5, 7.25, 40.0, 33.3])
    b = bytes(rois.polyroi_bytearray(x, y, pos=2, subpixel=True))
    assert len(b) == 112 and b[:4] == b"Iout"
    assert hashlib.sha256(b).hexdigest() == "9e394be9b5d3ae592c63d1bd595a585848eff9eca31af44bf83dc8026b2b4719"
    # the reference's own function on the seeded cases, frozen by tests/golden/make_io_ref.py
    cases, ref = _golden()
    got = [hashlib.sha256(bytes(rois.polyroi_bytearray(xs, ys, pos=pos, subpixel=sub))).hexdigest() for xs, ys, pos, sub in cases.roi_cases()]
    assert got == ref["polyroi_bytearray"]

def test_export_imagej_rois_and_tiff_roundtrip(tmp_path):
    from stardist_b200.io import rois, tiff
    rng = np.random.default_rng(1)
    coord = rng.uniform(0, 100, (5, 2, 32))
    rois.export_imagej_rois(tmp_path / "set.zip", coord)
    with zipfile.ZipFile(tmp_path / "set.zip") as z:
        names = sorted(z.namelist())
        assert names == ["001_%03d.roi" % i for i in range(1, 6)]
        assert z.read(names[0])[:4] == b"Iout"
    a = rng.integers(0, 5000, (7, 33, 21)).astype(np.int32)
    tiff.imwrite(tmp_path / "a.tif", a)
    assert np.array_equal(tiff.imread(tmp_path / "a.tif"), a)
    b = rng.integers(0, 60000, (40, 50)).astype(np.uint16)
    tiff.imwrite(tmp_path / "b.tif", b)
    assert np.array_equal(tiff.imread(tmp_path / "b.tif"), b)
    with pytest.raises(ValueError):
        tiff.imwrite(tmp_path / "c.tif", np.zeros(3))


def test_cli_parser():
    from stardist_b200.scripts.predict import build_parser
    a = build_parser().parse_args(["-i", "x.tif", "y.tif", "-m", "model", "--n_tiles", "2", "3", "--pnorm", "2", "99", "--rois"])
    assert a.input == ["x.tif", "y.tif"] and a.n_tiles == [2, 3] and a.pnorm == [2.0, 99.0] and a.rois and a.outname == "{img}.stardist.tif"


def test_export_to_obj_file3D(tmp_path):
    """text identical to stardist/geometry/geom3d.py:277-347 (its outputs frozen in tests/golden/io_ref.json)"""
    import stardist_b200 as sd
    from stardist_b200.io import obj
    rays = sd.Rays_GoldenSpiral(12)
    rng = np.random.default_rng(0)
    polys = dict(dist=rng.uniform(2, 6, (4, 12)).astype(np.float32), points=rng.integers(5, 40, (4, 3)),
                 rays_vertices=rays.vertices, rays_faces=rays.faces)
    text = obj.export_to_obj_file3D(polys, fname=str(tmp_path / "m.obj"))
    assert open(tmp_path / "m.obj").read() == text
    assert text.count("\nv ") + text.startswith("v ") == 4 * 12 and text.count("f ") == 4 * len(rays.faces) and text.startswith("o poly_0\n")
    with pytest.raises(ValueError):
        obj.export_to_obj_file3D(dict(dist=polys["dist"]))
    cases, ref = _golden()
    got = [hashlib.sha256(obj.export_to_obj_file3D(cases.obj_polys(), **kw).encode()).hexdigest() for kw in cases.OBJ_KWARGS]
    assert got == ref["export_to_obj_file3D"]
