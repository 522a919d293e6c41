"""Command line prediction for a 2-D or 3-D model folder (stardist/scripts/predict2d.py, predict3d.py):

    python -m stardist_b200.scripts.predict -i input.tif [...] -m model_folder -o output_folder [--dim 3]

Same options as the reference's `stardist-predict2d` / `stardist-predict3d`; registered pretrained models need a download
and are not available on this path -- `-m` must be a model folder (config.json, thresholds.json, weights_best.h5 | weights.npz).
TIFF via Pillow (stardist_b200.io.tiff); `--rois` additionally writes the ImageJ ROI set of a 2-D prediction."""
import argparse
import pathlib
import sys
import numpy as np


def build_parser():
    p = argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter,
                                description="Prediction script for a stardist model folder on the H100 path")
    p.add_argument("-i", "--input", type=str, nargs="+", required=True, help="input file (tiff)")
    p.add_argument("-o", "--outdir", type=str, default=".", help="output directory")
    p.add_argument("--outname", type=str, default="{img}.stardist.tif", help="output file name (tiff)")
    p.add_argument("-m", "--model", type=str, required=True, help="model folder")
    p.add_argument("--dim", type=int, choices=(2, 3), default=None, help="2 or 3 (default: n_dim of the model's config.json)")
    p.add_argument("--axes", type=str, default=None, help="axes to use for the input, e.g. 'XYC'")
    p.add_argument("--n_tiles", type=int, nargs="+", default=None, help="number of tiles to use for prediction")
    p.add_argument("--pnorm", type=float, nargs=2, default=[1, 99.8], help="pmin/pmax to use for normalization")
    p.add_argument("--prob_thresh", type=float, default=None, help="prob_thresh for model (if not given use model default)")
    p.add_argument("--nms_thresh", type=float, default=None, help="nms_thresh for model (if not given use model default)")
    p.add_argument("--rois", action="store_true", help="2-D: also write <outname>.rois.zip (ImageJ polygon ROIs)")
    p.add_argument("-v", "--verbose", action="store_true")
    return p


def main(argv=None):
    args = build_parser().parse_args(argv)
    import json
    from ..utils import normalize
    from ..io.tiff import imread, imwrite
    from ..io.rois import export_imagej_rois
    from .. import StarDist2D, StarDist3D
    folder = pathlib.Path(args.model)
    if not folder.is_dir():
        raise ValueError("model folder not found: %s (pretrained model names need a download and are not supported)" % args.model)
    dim = args.dim
    if dim is None:
        with open(folder / "config.json") as f:
            dim = int(json.load(f).get("n_dim", 2))
    cls = StarDist2D if dim == 2 else StarDist3D
    model = cls(None, name=folder.name, basedir=str(folder.parent))
    out = pathlib.Path(args.outdir)
    out.mkdir(parents=True, exist_ok=True)
    written = []
    for fname in args.input:
        if args.verbose: print("reading image %s" % fname)
        img = imread(fname)
        axes = args.axes
        if axes is None:
            axes = {2: "YX", 3: "YXC"}.get(img.ndim) if dim == 2 else {3: "ZYX", 4: "ZYXC"}.get(img.ndim)
        if axes is None or len(axes) != img.ndim:
            raise ValueError("dimension of input (%d) not compatible with the axes (%s)" % (img.ndim, axes))
        if args.verbose: print("loaded image of size %s, normalizing..." % (img.shape,))
        # csbdeep.utils.normalize(img, pmin, pmax, axis=<all but C>) of the reference script (predict2d.py:77) as the model's
        # normalizer: same numbers, computed in HBM for single-channel images (stardist_b200/prep.py), on the host otherwise
        from ..models.base import PercentileNormalizer
        labels, res = model.predict_instances(img, axes=axes, normalizer=PercentileNormalizer(*args.pnorm), n_tiles=args.n_tiles,
                                              prob_thresh=args.prob_thresh, nms_thresh=args.nms_thresh)
        target = out / args.outname.format(img=pathlib.Path(fname).with_suffix("").name)
        imwrite(target, labels)
        written.append(str(target))
        if args.rois and dim == 2:
            export_imagej_rois(str(target.with_suffix("")) + ".rois", res["coord"])
        if args.verbose: print("%d instances -> %s" % (len(res["prob"]), target))
    return written


if __name__ == "__main__":
    main(sys.argv[1:])
