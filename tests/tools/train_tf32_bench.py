"""Training step time with the TF32 backward pass off and on (stardist_b200.enable_tensor_float_32_execution), for the 2-D
default (4 x 256^2, 32 rays), the 3-D default (1 x 128^3, 96 rays) and the 3-D notebook batch (2 x 48x96x96, 96 rays, grid
(1, 2, 2)); the same steps in torch autograd with cuDNN, allow_tf32 off and on; and per layer of the defaults the kernel time
and achieved TFLOP/s of the fp32 and TF32 weight-gradient (sdb_conv_wgrad_nd / _tf32_nd) and input-gradient (sdb_conv3_nd on
the flipped kernel / sdb_conv_dgrad_tf32_nd) kernels.  Finally a torch.profiler breakdown of the TF32 step by kernel.

Step times: CUDA events around each step after warm-up, median over --steps steps; the two modes are timed alternately in
rounds.  Kernel times: CUDA events around --reps launches after one warm-up launch.  The card's name, power limit and max SM
clock are read in the same call and printed with every result line.

    python tests/tools/train_tf32_bench.py [--steps 20] [--warmup 3] [--reps 10] [--case 2d|3d|3d_nb|all] [--out FILE]
"""
import argparse, json, os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_step_bench import step_flops, gpu_info, batch, time_it


def make_case(case):
    from stardist_b200 import Config2D, Config3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    if case == '2d':
        return Config2D(n_rays=32), (256, 256), 4
    if case == '3d':
        return Config3D(rays=Rays_GoldenSpiral(96)), (128, 128, 128), 1
    return Config3D(rays=Rays_GoldenSpiral(96), grid=(1, 2, 2)), (48, 96, 96), 2


def trainer(config, weights, on):
    import stardist_b200 as s
    from stardist_b200.models.train import UNetTrainer
    s.enable_tensor_float_32_execution(on)
    try:
        return UNetTrainer(config, weights)
    finally:
        s.enable_tensor_float_32_execution(False)


def torch_step_fn(config, weights, x, p, d):
    import torch
    import train_oracle as O
    from stardist_b200.models.weights import unet_layers
    P = O.params64(weights, [l['name'] for l in unet_layers(config) if l['kind'] in ('conv', 'head')])
    P = {n: (k.detach().float().cuda().requires_grad_(True), b.detach().float().cuda().requires_grad_(True)) for n, (k, b) in P.items()}
    opt = torch.optim.Adam([t for kb in P.values() for t in kb], lr=config.train_learning_rate, eps=1e-7)

    def step():
        opt.zero_grad(set_to_none=True)
        prob, dist = O.forward64(config, P, x)
        loss = O.loss64(prob, dist, p, d, dist_loss=config.train_dist_loss, lam=float(config.train_background_reg),
                        weights=tuple(float(v) for v in config.train_loss_weights))[0]
        loss.backward()
        opt.step()
    return step


def run_case(case, steps, warmup, rounds=2):
    import torch
    from stardist_b200.models.weights import glorot_uniform_weights
    config, spatial, B = make_case(case)
    weights = glorot_uniform_weights(config, seed=0)
    x, p, d = batch(config, spatial, B)
    flops = step_flops(config, spatial, B)
    trs = {on: trainer(config, weights, on) for on in (False, True)}
    ms = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            ms[on].append(time_it(lambda: trs[on].step(x, p, d), steps, warmup))
    del trs
    torch.cuda.empty_cache()
    torch.backends.cudnn.benchmark = True
    mt = {}
    for allow in (False, True):
        torch.backends.cudnn.allow_tf32 = allow
        torch.backends.cuda.matmul.allow_tf32 = allow
        mt[allow] = time_it(torch_step_fn(config, weights, x, p, d), steps, warmup)
    torch.cuda.empty_cache()
    off, on = float(np.median(ms[False])), float(np.median(ms[True]))
    return dict(case=case, batch=B, spatial=list(spatial), n_rays=config.n_rays, tflop_per_step=flops / 1e12,
                step_ms_fp32=off, step_ms_tf32=on, speedup=off / on, rounds_ms_fp32=ms[False], rounds_ms_tf32=ms[True],
                achieved_tflops_fp32=flops / (off * 1e-3) / 1e12, achieved_tflops_tf32=flops / (on * 1e-3) / 1e12,
                torch_cudnn_step_ms_fp32=mt[False], torch_cudnn_step_ms_tf32=mt[True], gpu=gpu_info())


def conv_layers(config, spatial, B):
    """(name, spatial size, cin_skip, cin_lo, up, cout, k, first) of every U-Net convolution, as the trainer's backward sees it"""
    from stardist_b200.models.weights import unet_layers
    size, out, first, up = np.array(spatial, np.int64), [], True, None
    for l in unet_layers(config):
        if l['kind'] == 'pool':
            size = size // np.array(l['pool'])
        elif l['kind'] == 'up':
            size = size * np.array(l['pool'])
            up = tuple(l['pool'])
        elif l['kind'] == 'conv':
            c_lo = l.get('cin_lo', 0)
            out.append((l['name'], tuple(int(s) for s in size), l['cin'] - c_lo, c_lo, up if c_lo else (1,) * config.n_dim,
                        l['cout'], tuple(l['k']), first))
            first = False
    return out


def time_kernel(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def layer_kernels(case, reps):
    """per convolution of the case: fp32 / TF32 weight- and input-gradient kernel times (ms) and achieved TFLOP/s"""
    import torch
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    config, spatial, B = make_case(case)
    nd, rows = config.n_dim, []
    st = L.stream_ptr()
    for name, size, c_skip, c_lo, up, cout, k, first in conv_layers(config, spatial, B):
        cin = c_skip + c_lo
        d, h, w = ((1,) + size) if nd == 2 else size
        npix = B * d * h * w
        kz, kyx = (1, 3) if nd == 2 else (3, 3)
        g = torch.randn((B,) + size + (cout,), device='cuda')
        xs = torch.randn((B,) + size + (c_skip,), device='cuda')
        lo = torch.randn((B,) + tuple(s // u for s, u in zip(size, up)) + (c_lo,), device='cuda') if c_lo else None
        uz, uy, ux = ((1,) + tuple(up)) if nd == 2 else tuple(up)
        need = int(lib.sdb_conv_wgrad_workspace(npix, 3 ** nd, cin, cout))
        work = torch.empty(need, device='cuda')
        dw = torch.empty((3 ** nd, cin, cout), device='cuda'); db = torch.empty(cout, device='cuda')
        flops = 2.0 * npix * 3 ** nd * cin * cout
        r = dict(case=case, layer=name, size=list(size), cin=cin, cout=cout, gflop=flops / 1e9)
        for tag, fn in (('wgrad_fp32', lib.sdb_conv_wgrad_nd), ('wgrad_tf32', lib.sdb_conv_wgrad_tf32_nd)):
            r[tag + '_ms'] = time_kernel(lambda: L.check(fn(L.ptr(xs), L.ptr(lo), B, d, h, w, c_skip, c_lo, uz, uy, ux, kz, kyx, L.ptr(g), cout,
                                                            cout, L.ptr(work), need, L.ptr(dw), L.ptr(db), st)), reps)
        if not first:
            from stardist_b200.models.unet_device import conv_dgrad3_accepts
            assert conv_dgrad3_accepts(nd, k, cin, cout)
            wf = torch.randn((3 ** nd, cout, cin), device='cuda')
            zb = torch.zeros(cin, device='cuda')
            gin = torch.empty((B,) + size + (cin,), device='cuda')
            r['dgrad_fp32_ms'] = time_kernel(lambda: L.check(lib.sdb_conv3_nd(L.ptr(g), None, B, d, h, w, cout, 0, 1, 1, 1, L.ptr(wf), L.ptr(zb),
                                                                             cin, kz, 0, L.ptr(gin), st)), reps)
            r['dgrad_tf32_ms'] = time_kernel(lambda: L.check(lib.sdb_conv_dgrad_tf32_nd(L.ptr(g), B, d, h, w, cout, L.ptr(wf), cin, kz, 3,
                                                                                        L.ptr(gin), st)), reps)
        for key in [k_ for k_ in r if k_.endswith('_ms')]:
            r[key.replace('_ms', '_tflops')] = flops / (r[key] * 1e-3) / 1e12
        rows.append(r)
        del g, xs, lo, work, dw
        torch.cuda.empty_cache()
    tot = {t: sum(r.get(t + '_ms', 0.0) for r in rows) for t in ('wgrad_fp32', 'wgrad_tf32', 'dgrad_fp32', 'dgrad_tf32')}
    return rows, dict(case=case, layer_totals_ms=tot, gpu=gpu_info())


def profile_tf32(case):
    import torch
    from torch.profiler import profile, ProfilerActivity
    from stardist_b200.models.weights import glorot_uniform_weights
    config, spatial, B = make_case(case)
    tr = trainer(config, glorot_uniform_weights(config, seed=0), True)
    x, p, d = batch(config, spatial, B)
    for _ in range(2):
        tr.step(x, p, d)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            tr.step(x, p, d)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = e.name.replace('(anonymous namespace)::', '')[:60]
            tot[k] = tot.get(k, 0.0) + e.device_time_total / 3e3
    return dict(case=case, tf32_ms_per_step_by_kernel={k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:10]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--case", default="all", choices=["2d", "3d", "3d_nb", "all"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_tf32_bench needs a CUDA device")
    cases = ["2d", "3d", "3d_nb"] if a.case == "all" else [a.case]
    res = []
    for c in cases:
        r = run_case(c, a.steps, a.warmup)
        print(json.dumps(r), flush=True)
        res.append(r)
    for c in [c for c in cases if c in ("2d", "3d")]:
        rows, tot = layer_kernels(c, a.reps)
        for r in rows:
            print(json.dumps(r), flush=True)
        print(json.dumps(tot), flush=True)
        res += rows + [tot]
    for c in [c for c in cases if c in ("2d", "3d")]:
        r = profile_tf32(c)
        print(json.dumps(r), flush=True)
        res.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
