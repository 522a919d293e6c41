"""Time the any-shape convolution of csrc/unet_any.cu (sdb_conv_any_nd):
  - against the tiled CUDA-core convolution sdb_conv3_nd on shapes both accept (3^d, cin = cout = 32 and 64, 2-D 1 x 1024^2,
    3-D 1 x 64 x 256^2), with the largest relative difference of their outputs (the two sum in different orders);
  - against torch's fp32 cuDNN convolution (TF32 off) on shapes only the new kernel takes;
  - one full predict_instances on a 1024^2 image for two 2-D configurations outside the default family.
Kernel times are CUDA events around `--steps` launches after `--warmup`.  Prints one JSON line per case, the first one with
the device name and power limit.

    python tests/tools/any_config_bench.py [--steps 20] [--warmup 3] [--out FILE]
"""
import argparse, json, os, subprocess, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
        return dict(device=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                       # the torch name is still reported
        import torch
        return dict(device=torch.cuda.get_device_name(), power_limit="unknown (%s)" % type(e).__name__)


def time_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def conv_call(lib, which, x, k, b, out, stride=(1, 1, 1)):
    """closure launching sdb_conv3_nd or sdb_conv_any_nd (ReLU) on x [1, (D,) H, W, cin]"""
    from stardist_b200 import _lib as L
    nd = x.dim() - 2
    d, h, w = ((1,) + tuple(x.shape[1:3])) if nd == 2 else tuple(x.shape[1:4])
    cin, cout = x.shape[-1], k.shape[-1]
    ks = ((1,) if nd == 2 else ()) + tuple(k.shape[:nd])
    st = L.stream_ptr()
    if which == 'conv3':
        return lambda: L.check(lib.sdb_conv3_nd(L.ptr(x), L.ptr(None), 1, d, h, w, cin, 0, 1, 1, 1, L.ptr(k), L.ptr(b), cout,
                                                1 if nd == 2 else 3, 1, L.ptr(out), st))
    return lambda: L.check(lib.sdb_conv_any_nd(L.ptr(x), L.ptr(None), 1, d, h, w, cin, 0, 1, 1, 1, L.ptr(k), L.ptr(b), cout,
                                               *ks, *stride, 1, L.ptr(out), st))


def tf_pad(size, k, s):
    out = -(-size // s)
    tot = max((out - 1) * s + k - size, 0)
    return tot // 2, tot - tot // 2


def torch_conv(x, k, b, stride):
    """closure: fp32 cuDNN convolution with TensorFlow 'same' padding, ReLU; x channels-last [1, *sp, cin]"""
    import torch
    import torch.nn.functional as F
    nd = x.dim() - 2
    xc = x.movedim(-1, 1).contiguous()
    wc = k.permute(nd + 1, nd, *range(nd)).contiguous()
    pads = []
    for ax in reversed(range(nd)):
        pads += list(tf_pad(x.shape[1 + ax], k.shape[ax], stride[ax]))
    conv = F.conv2d if nd == 2 else F.conv3d
    return lambda: torch.relu(conv(F.pad(xc, pads), wc, b, stride=stride))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from stardist_b200 import _lib as L
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    lib = L.require_cuda()
    rows = [gpu_info()]
    gen = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: (torch.rand(s, generator=gen, device="cuda") - 0.5)

    def flops(sp_out, k, cin, cout):
        return 2.0 * np.prod(sp_out) * np.prod(k) * cin * cout

    # 1. equal shapes: sdb_conv_any_nd against sdb_conv3_nd
    for nd, sp in ((2, (1024, 1024)), (3, (64, 256, 256))):
        for c in (32, 64):
            x = rnd(1, *sp, c).contiguous(); k = (rnd(*(3,) * nd, c, c) * 0.2).contiguous(); b = rnd(c).contiguous()
            o3 = torch.empty(1, *sp, c, device="cuda"); oa = torch.empty_like(o3)
            t3 = time_ms(conv_call(lib, 'conv3', x, k, b, o3), args.steps, args.warmup)
            ta = time_ms(conv_call(lib, 'any', x, k, b, oa, stride=(1, 1, 1)), args.steps, args.warmup)
            rel = float((oa - o3).abs().max() / o3.abs().max())
            fl = flops(sp, (3,) * nd, c, c)
            rows.append(dict(case="equal_shape", nd=nd, shape=list(sp), cin=c, cout=c, conv3_ms=round(t3, 4), any_ms=round(ta, 4),
                             ratio=round(ta / t3, 3), conv3_tflops=round(fl / t3 / 1e9, 2), any_tflops=round(fl / ta / 1e9, 2),
                             max_rel_diff=rel))
            print(json.dumps(rows[-1]), flush=True)

    # 2. new shapes: sdb_conv_any_nd against torch fp32 cuDNN (TF32 off)
    for nd, sp, kk, s, cin, cout in ((2, (1024, 1024), (5, 5), (1, 1), 16, 16), (2, (1024, 1024), (3, 3), (1, 1), 1, 16),
                                     (2, (1024, 1024), (3, 3), (1, 1), 24, 24), (2, (1024, 1024), (7, 7), (2, 2), 16, 32),
                                     (3, (64, 256, 256), (1, 3, 3), (1, 1, 1), 16, 16), (3, (64, 256, 256), (3, 3, 3), (1, 2, 2), 16, 32),
                                     (3, (64, 256, 256), (7, 7, 7), (1, 1, 1), 1, 16)):
        x = rnd(1, *sp, cin).contiguous(); k = (rnd(*kk, cin, cout) * 0.2).contiguous(); b = rnd(cout).contiguous()
        osp = tuple(-(-a // t) for a, t in zip(sp, s))
        oa = torch.empty(1, *osp, cout, device="cuda")
        s3 = ((1,) + tuple(s)) if nd == 2 else tuple(s)
        ta = time_ms(conv_call(lib, 'any', x, k, b, oa, stride=s3), args.steps, args.warmup)
        tc = torch_conv(x, k, b, s)
        tt = time_ms(tc, args.steps, args.warmup)
        rel = float((oa - tc().movedim(1, -1)).abs().max() / oa.abs().max())
        fl = flops(osp, kk, cin, cout)
        rows.append(dict(case="new_shape", nd=nd, shape=list(sp), k=list(kk), stride=list(s), cin=cin, cout=cout,
                         any_ms=round(ta, 4), cudnn_fp32_ms=round(tt, 4), ratio=round(ta / tt, 3),
                         any_tflops=round(fl / ta / 1e9, 2), max_rel_diff=rel))
        print(json.dumps(rows[-1]), flush=True)

    # 3. full predict_instances on a 1024^2 image
    import bench_data
    from stardist_b200 import Config2D, StarDist2D
    img, _ = bench_data.synthetic_image((1024, 1024), seed=0)
    for name, cfg in (("unet_n_filter_base=16", Config2D(unet_n_filter_base=16)),
                      ("unet_kernel_size=(5,5), elu", Config2D(unet_kernel_size=(5, 5), unet_activation='elu', unet_last_activation='linear'))):
        model = StarDist2D(cfg, name=None, basedir=None)
        k, bb = model.weights['dist']
        model.weights['dist'] = (k, bb + np.float32(4.0))
        prob, _ = model.predict(img)
        pthr = float(np.quantile(prob, 0.97))
        for _ in range(args.warmup):
            model.predict_instances(img, prob_thresh=pthr, nms_thresh=0.3)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            labels, res = model.predict_instances(img, prob_thresh=pthr, nms_thresh=0.3)
        torch.cuda.synchronize()
        ms = 1000 * (time.perf_counter() - t0) / args.steps
        x = torch.from_numpy(img[None, ..., None]).cuda()
        tf = time_ms(lambda: model.net.forward(x), args.steps, args.warmup)
        rows.append(dict(case="predict_instances_1024", config=name, ms=round(ms, 2), forward_ms=round(tf, 2), instances=len(res['prob'])))
        print(json.dumps(rows[-1]), flush=True)

    print(json.dumps(rows[0]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
