"""configs[2] at full size (SURVEY 8d: 128x512x512, Rays_GoldenSpiral n_rays = 96, default Config3D), one GPU.

R1 "network-real": the random-init 3-D U-Net (tensor-core 3x3x3 convolutions) on a synthetic volume, timed with CUDA events,
    then predict_instances end to end (host volume in, label volume out) with prob_thresh at a high quantile of its own
    prob map (a random-init dist head gives tiny polyhedra, so this exercises network + threshold/sort/gather + a trivial NMS).
R2 "post-proc-real": candidates (prob, dist rows, points) derived analytically from ground-truth ellipsoids generated for a
    base cell and replicated over the volume (objects keep a margin from the cell faces, so cells do not interact),
    through StarDist3D._instances_from_prediction(points=...) = sort + NMS3D + polyhedron_to_label + relabel.
Optionally (--cpu) the reference C++/OpenMP NMS (oracle/_ref) on the base cell's candidates, all host cores.

Usage: python tests/tools/run_3d_full.py [D H W] [--cell d h w] [--pthr 0.8] [--cpu] [--json out.json]"""
import os, sys, time, json, argparse
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch
import stardist_b200 as sd

ap = argparse.ArgumentParser()
ap.add_argument("shape", type=int, nargs="*", default=[128, 512, 512])
ap.add_argument("--cell", type=int, nargs=3, default=[64, 256, 256])
ap.add_argument("--n-rays", type=int, default=96)
ap.add_argument("--pthr", type=float, default=0.8)
ap.add_argument("--quantile", type=float, default=0.998)
ap.add_argument("--cpu", action="store_true")
ap.add_argument("--skip-r1", action="store_true")
ap.add_argument("--only-net", action="store_true", help="stop after the timed network passes (profiling)")
ap.add_argument("--json", default=None)
ap.add_argument("--nms3d-variant", type=int, default=0, help="sdb_nms3d_set_variant: 1 = S3/S4 volumes on pre-normalised planes")
args = ap.parse_args()
D, H, W = args.shape
cd, ch, cw = args.cell
assert D % cd == 0 and H % ch == 0 and W % cw == 0
n_rays = args.n_rays
out = dict(shape=[D, H, W], n_rays=n_rays, cell=[cd, ch, cw])

from stardist_b200 import _lib as _L
_L.require_cuda().sdb_nms3d_set_variant(args.nms3d_variant)
out['nms3d_variant'] = args.nms3d_variant
rng = np.random.default_rng(0)
rays = sd.Rays_GoldenSpiral(n_rays)
cfg = sd.Config3D(rays=rays)
model = sd.StarDist3D(cfg, name=None, basedir=None)
out['network_executor'] = type(model.net).__name__


def ev_time(fn, reps):
    ts = []
    for _ in range(reps):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record(); r = fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(ts)), r


# ---- R1: network pass + end-to-end predict_instances on the network's own output
if not args.skip_r1:
    from stardist_b200.models.weights import unet_layers
    flop = 0
    sp = np.array([D, H, W], dtype=np.float64)
    for l in unet_layers(cfg):
        if l['kind'] == 'pool': sp = sp / 2
        elif l['kind'] == 'up': sp = sp * 2
        elif l['kind'] == 'conv': flop += 2 * np.prod(sp) * l['cin'] * l['cout'] * 27
    vol = rng.uniform(0, 1, (D, H, W)).astype(np.float32)
    x = torch.from_numpy(vol[None, ..., None]).cuda()
    model.net.forward(x); torch.cuda.synchronize()
    t_net, (p, d) = ev_time(lambda: model.net.forward(x), 3)
    out.update(network_s=t_net, network_alg_flop=float(flop), network_alg_tflops=flop / t_net / 1e12,
               peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print("network %dx%dx%d (%s): %.4f s = %.1f algorithmic TFLOP/s (3x3x3 convs, %.3e FLOP), peak device memory %.1f GB"
          % (D, H, W, out['network_executor'], t_net, flop / t_net / 1e12, flop, out['peak_mem_gb']))
    if args.only_net:
        print(json.dumps(out)); sys.exit(0)
    # prob threshold at the given quantile of the (subsampled) prob map
    ps = p.flatten()[::37].float()
    k = max(1, int(round(args.quantile * ps.numel())))
    qthr = float(torch.kthvalue(ps, k).values)
    del p, d, x, ps
    torch.cuda.empty_cache()
    for rep in range(2):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        labels, res = model.predict_instances(vol, prob_thresh=qthr, nms_thresh=0.3)
        torch.cuda.synchronize(); t_e2e = time.perf_counter() - t0
    n1 = len(res['prob'])
    out.update(r1_prob_thresh=qthr, r1_e2e_s=t_e2e, r1_instances=n1, r1_stats={k: (float(v) if np.isscalar(v) else str(v)) for k, v in getattr(model, '_stats', {}).items()})
    print("R1 predict_instances host-to-host (prob_thresh = %.4f, the %.4f quantile): %.3f s, %d instances" % (qthr, args.quantile, t_e2e, n1))
    del labels, res

# ---- R2: ground-truth ellipsoids of one cell -> candidate rows (prob > pthr), replicated over the volume
pthr = args.pthr
verts = rays.vertices.astype(np.float64)
occ = np.zeros((cd, ch, cw), bool)
c_prob, c_dist, c_pts = [], [], []
n_obj = 0; filled = 0; target = 0.30 * cd * ch * cw
t_gen = time.perf_counter()
for _ in range(400000):
    if filled >= target: break
    r = rng.uniform(5, 9, 3) * np.array([0.6, 1, 1])
    m = np.ceil(r).astype(int) + 1
    c = np.array([rng.integers(m[0], cd - m[0]), rng.integers(m[1], ch - m[1]), rng.integers(m[2], cw - m[2])])
    sl = tuple(slice(c[i] - m[i], c[i] + m[i] + 1) for i in range(3))
    zz, yy, xx = np.mgrid[-m[0]:m[0] + 1, -m[1]:m[1] + 1, -m[2]:m[2] + 1]
    q = np.stack([zz / r[0], yy / r[1], xx / r[2]], -1)
    rn = np.sqrt((q ** 2).sum(-1))
    inside = rn <= 1
    if occ[sl][inside].any(): continue
    occ[sl] |= inside
    n_obj += 1; filled += inside.sum()
    sel = (1 - rn) > pthr                                            # candidate voxels of this object
    if not sel.any(): continue
    qs = q[sel]                                                      # [n, 3] offsets in the unit-sphere frame
    v = verts / r
    a = (v ** 2).sum(-1)
    b = 2 * qs @ v.T                                                 # [n, R]
    cc = (rn[sel] ** 2 - 1)[:, None]
    t = (-b + np.sqrt(np.maximum(b * b - 4 * a * cc, 0))) / (2 * a)
    c_prob.append((1 - rn[sel]).astype(np.float32))
    c_dist.append(np.maximum(t, 1e-3).astype(np.float32))
    c_pts.append(np.stack([zz[sel], yy[sel], xx[sel]], -1) + c)
cell_prob = np.concatenate(c_prob); cell_dist = np.concatenate(c_dist); cell_pts = np.concatenate(c_pts).astype(np.int64)
offs = [(z, y, x) for z in range(0, D, cd) for y in range(0, H, ch) for x in range(0, W, cw)]
prob = np.concatenate([cell_prob] * len(offs))
dist = np.concatenate([cell_dist] * len(offs))
pts = np.concatenate([cell_pts + np.array(o) for o in offs])
print("ground truth: %d ellipsoids per %dx%dx%d cell (fill %.2f, %.1f s to generate), %d cells -> %d objects, %d candidates (prob > %.2f)"
      % (n_obj, cd, ch, cw, filled / (cd * ch * cw), time.perf_counter() - t_gen, len(offs), n_obj * len(offs), len(prob), pthr))
out.update(r2_objects=n_obj * len(offs), r2_candidates=int(len(prob)))
for rep in range(3):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    labels, res = model._instances_from_prediction((D, H, W), prob, dist, points=pts, prob_thresh=pthr, nms_thresh=0.3)
    torch.cuda.synchronize(); t_post = time.perf_counter() - t0
    print("R2 sort + NMS3D + polyhedron_to_label + relabel (host candidate rows in, label volume out): %.3f s -> %d instances, %d labelled voxels"
          % (t_post, len(res['prob']), int((labels > 0).sum())))
nk = len(res['prob'])
out.update(r2_post_s=t_post, r2_instances=nk)
if 'network_s' in out:
    tot = out['network_s'] + t_post
    out.update(total_s=tot, instances_per_s=nk / tot)
    print("R1 network + R2 post-processing: %.3f s per volume -> %.0f instances/s" % (tot, nk / tot))

# ---- reference C++/OpenMP NMS on ONE cell's candidates (bounded CPU sample), all host cores
if args.cpu:
    from oracle import ref_ext
    ext = ref_ext.stardist3d() if ref_ext.available() else None
    if ext is None:
        print("oracle/_ref 3D extension not available")
    else:
        order = np.argsort(cell_prob, kind='stable')[::-1]
        dd = np.ascontiguousarray(cell_dist[order]); pp = np.ascontiguousarray(cell_pts[order].astype(np.float32)); ss = np.ascontiguousarray(cell_prob[order])
        v32 = np.ascontiguousarray(rays.vertices, np.float32); f32 = np.ascontiguousarray(rays.faces, np.int32)
        t0 = time.perf_counter()
        keep = ext.c_non_max_suppression_inds(dd, pp, v32, f32, ss, 1, 1, 0, np.float32(0.3))
        t_cpu = time.perf_counter() - t0
        print("reference C++/OpenMP NMS3D on one cell (%d candidates, %d cores): %.2f s -> %d kept" % (len(dd), os.cpu_count(), t_cpu, int(keep.sum())))
        out.update(cpu_ref_nms_cell_s=t_cpu, cpu_ref_nms_cell_candidates=int(len(dd)), cpu_cores=os.cpu_count(), cpu_ref_kept=int(keep.sum()))
if args.json:
    with open(args.json, "w") as f:
        json.dump(out, f)
print(json.dumps(out))
