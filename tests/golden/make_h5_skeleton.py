"""Freeze small stand-ins of the reference's shipped Keras checkpoints (models/examples/{2D,3D}_demo/weights_best.h5) for the
HDF5 reader and model-folder tests: the file byte for byte -- superblock, groups, object headers, attributes, every dataset --
except that the payload of each dataset larger than KEEP bytes is zeroed, then gzip-compressed (the zero runs vanish).
The kept datasets must read back bit-equal to the checkpoint frozen in demo2d.npz / demo3d.npz, the zeroed ones as zeros
of the right shape.  Run where a reference checkout exists:  python tests/golden/make_h5_skeleton.py /path/to/stardist"""
import gzip, os, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
KEEP = 16384


def skeleton(src, dst):
    from stardist_b200.io import h5lite
    raw = bytearray(open(src, "rb").read())
    for name, a in h5lite.read_datasets(src).items():
        b = np.ascontiguousarray(a).tobytes()
        if len(b) <= KEEP:
            continue
        at = raw.find(b)
        assert at >= 0 and raw.find(b, at + 1) < 0, name      # contiguous layout, one occurrence
        raw[at:at + len(b)] = bytes(len(b))
    with open(dst, "wb") as out, gzip.GzipFile(fileobj=out, mode="wb", compresslevel=9, mtime=0) as f:
        f.write(bytes(raw))


if __name__ == "__main__":
    for demo in ("2D_demo", "3D_demo"):
        skeleton(os.path.join(sys.argv[1], "models", "examples", demo, "weights_best.h5"),
                 os.path.join(HERE, "%s_weights_skeleton.h5.gz" % demo.split("_")[0].lower()))
