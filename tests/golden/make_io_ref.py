"""Freeze the reference's ImageJ ROI and Wavefront OBJ writers into tests/golden/io_ref.json: sha256 of
stardist/utils.py::polyroi_bytearray and stardist/geometry/geom3d.py::export_to_obj_file3D on the seeded inputs of
tests/test_io_cpu.py (each function compiled in isolation: their modules import csbdeep / skimage).
Run where a reference checkout exists:  python tests/golden/make_io_ref.py /path/to/stardist"""
import ast, hashlib, json, os, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import io_cases


def load(src, names, ns):
    fns = [n for n in ast.parse(open(src).read()).body if isinstance(n, ast.FunctionDef) and n.name in names]
    exec(compile(ast.Module(body=fns, type_ignores=[]), src, "exec"), ns)
    return ns


def main(ref):
    sha = lambda b: hashlib.sha256(b).hexdigest()
    u = load(os.path.join(ref, "stardist", "utils.py"), ("polyroi_bytearray",), {"np": np})
    rois = [sha(bytes(u["polyroi_bytearray"](xs, ys, pos=pos, subpixel=sub))) for xs, ys, pos, sub in io_cases.roi_cases()]
    g = load(os.path.join(ref, "stardist", "geometry", "geom3d.py"), ("dist_to_coord3D", "export_to_obj_file3D"), {"np": np, "tqdm": (lambda x: x)})
    polys = io_cases.obj_polys()
    objs = [sha(g["export_to_obj_file3D"](dict(polys), **kw).encode()) for kw in io_cases.OBJ_KWARGS]
    with open(os.path.join(HERE, "io_ref.json"), "w") as f:
        json.dump(dict(polyroi_bytearray=rois, export_to_obj_file3D=objs), f, indent=0)


if __name__ == "__main__":
    main(sys.argv[1])
