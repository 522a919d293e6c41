"""Training step time and peak device memory under the three precision settings -- 'float32', 'float32' with the TF32
switch on, and the 'mixed_bfloat16' policy (stardist_b200.mixed_precision) -- for the 2-D default (4 x 256^2, 32 rays), the
3-D default (1 x 128^3, 96 rays) and the 3-D notebook batch (2 x 48x96x96, 96 rays, grid (1, 2, 2)); the same step in torch
autograd with cuDNN under bf16 autocast; per convolution of the defaults the time and achieved TFLOP/s of the bf16 forward,
input-gradient and weight-gradient kernels against the 989 TFLOP/s dense bf16 data-sheet figure; and a torch.profiler
breakdown of the bf16 step by kernel.

Step times: CUDA events around each step after warm-up, median over --steps steps (>= 10); the settings are timed alternately
in rounds.  Peak memory: torch.cuda.max_memory_allocated over one step after the trainer's buffers exist, above the memory
allocated before it.  Kernel times: CUDA events around --reps launches after one warm-up launch.  The card's name, power
limit and max SM clock are read in the same call and printed with every result line.

    python tests/tools/train_bf16_bench.py [--steps 20] [--warmup 3] [--reps 10] [--case 2d|3d|3d_nb|all] [--out FILE]
"""
import argparse, json, os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_step_bench import gpu_info, batch, time_it
from train_tf32_bench import make_case, conv_layers, time_kernel

PEAK_BF16_TFLOPS = 989.0
SETTINGS = ('float32', 'tf32', 'mixed_bfloat16')


def trainer(config, weights, setting):
    import stardist_b200 as s
    from stardist_b200 import mixed_precision as mp
    from stardist_b200.models.train import UNetTrainer
    s.enable_tensor_float_32_execution(setting == 'tf32')
    mp.set_global_policy('mixed_bfloat16' if setting == 'mixed_bfloat16' else 'float32')
    try:
        return UNetTrainer(config, weights)
    finally:
        s.enable_tensor_float_32_execution(False)
        mp.set_global_policy('float32')


def torch_autocast_step_fn(config, weights, x, p, d):
    """the step in torch autograd: fp32 parameters, convolutions under torch.autocast(bfloat16) on cuDNN, Adam"""
    import torch
    import train_oracle as O
    from stardist_b200.models.weights import unet_layers
    P = O.params64(weights, [l['name'] for l in unet_layers(config) if l['kind'] in ('conv', 'head')])
    P = {n: (k.detach().float().cuda().requires_grad_(True), b.detach().float().cuda().requires_grad_(True)) for n, (k, b) in P.items()}
    opt = torch.optim.Adam([t for kb in P.values() for t in kb], lr=config.train_learning_rate, eps=1e-7)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast('cuda', dtype=torch.bfloat16):
            prob, dist = O.forward64(config, P, x)
        loss = O.loss64(prob.float(), dist.float(), p, d, dist_loss=config.train_dist_loss, lam=float(config.train_background_reg),
                        weights=tuple(float(v) for v in config.train_loss_weights))[0]
        loss.backward()
        opt.step()
    return step


def peak_step_bytes(fn):
    import torch
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return int(torch.cuda.max_memory_allocated() - base)


def run_case(case, steps, warmup, rounds=2):
    import torch
    from stardist_b200.models.weights import glorot_uniform_weights
    config, spatial, B = make_case(case)
    weights = glorot_uniform_weights(config, seed=0)
    x, p, d = batch(config, spatial, B)
    res = dict(case=case, batch=B, spatial=list(spatial), n_rays=config.n_rays)
    ms = {s: [] for s in SETTINGS}
    trs = {s: trainer(config, weights, s) for s in SETTINGS}
    for _ in range(rounds):
        for s in SETTINGS:
            ms[s].append(time_it(lambda: trs[s].step(x, p, d), steps, warmup))
    for s in SETTINGS:
        res['step_ms_' + s] = float(np.median(ms[s]))
        res['peak_step_mib_' + s] = peak_step_bytes(lambda: trs[s].step(x, p, d)) / 2 ** 20
    for s in SETTINGS:
        trs[s].gradients(x, p, d)
        res['saved_activation_mib_' + s] = sum(t.numel() * t.element_size() for t in trs[s].saved_activations()) / 2 ** 20
    del trs
    torch.cuda.empty_cache()
    fn = torch_autocast_step_fn(config, weights, x, p, d)
    res['torch_cudnn_bf16_autocast_step_ms'] = time_it(fn, steps, warmup)
    res['torch_cudnn_bf16_autocast_peak_step_mib'] = peak_step_bytes(fn) / 2 ** 20
    res['gpu'] = gpu_info()
    return res


def layer_kernels(case, reps):
    """per 3^d convolution of the case: bf16 forward, input-gradient and weight-gradient kernel times (ms), TFLOP/s and share
    of the 989 TFLOP/s bf16 data-sheet figure"""
    import torch
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    config, spatial, B = make_case(case)
    nd, rows = config.n_dim, []
    st = L.stream_ptr()
    bf = torch.bfloat16
    for name, size, c_skip, c_lo, up, cout, k, first in conv_layers(config, spatial, B):
        cin = c_skip + c_lo
        d, h, w = ((1,) + size) if nd == 2 else size
        npix = B * d * h * w
        kz, kyx = (1, 3) if nd == 2 else (3, 3)
        taps = 3 ** nd
        g = torch.randn((B,) + size + (cout,), device='cuda').to(bf)
        xs = torch.randn((B,) + size + (c_skip,), device='cuda').to(bf)
        lo = torch.randn((B,) + tuple(s // u for s, u in zip(size, up)) + (c_lo,), device='cuda').to(bf) if c_lo else None
        uz, uy, ux = ((1,) + tuple(up)) if nd == 2 else tuple(up)
        wb = torch.randn(taps * cin * cout, device='cuda').to(bf)
        bias = torch.zeros(max(cin, cout), device='cuda')
        y = torch.empty((B,) + size + (max(cin, cout),), device='cuda', dtype=bf)
        need = int(lib.sdb_conv_wgrad_workspace(npix, taps, cin, cout))
        work = torch.empty(need, device='cuda')
        dw = torch.empty((taps, cin, cout), device='cuda'); db = torch.empty(cout, device='cuda')
        flops = 2.0 * npix * taps * cin * cout
        r = dict(case=case, layer=name, size=list(size), cin=cin, cout=cout, gflop=flops / 1e9)
        r['forward_ms'] = time_kernel(lambda: L.check(lib.sdb_conv_bf16_nd(L.ptr(xs), L.ptr(lo), B, d, h, w, c_skip, c_lo, uz, uy, ux, kz, kyx,
                                                                          kyx, L.ptr(wb), L.ptr(bias), cout, 1, 0, L.ptr(y), st)), reps)
        r['wgrad_ms'] = time_kernel(lambda: L.check(lib.sdb_conv_wgrad_bf16_nd(L.ptr(xs), L.ptr(lo), B, d, h, w, c_skip, c_lo, uz, uy, ux, kz,
                                                                              kyx, L.ptr(g), 1, cout, cout, L.ptr(work), need, L.ptr(dw),
                                                                              L.ptr(db), st)), reps)
        if not first:
            r['dgrad_ms'] = time_kernel(lambda: L.check(lib.sdb_conv_bf16_nd(L.ptr(g), None, B, d, h, w, cout, 0, 1, 1, 1, kz, kyx, kyx,
                                                                            L.ptr(wb), None, cin, 0, 0, L.ptr(y), st)), reps)
        for key in [k_ for k_ in r if k_.endswith('_ms')]:
            tf = flops / (r[key] * 1e-3) / 1e12
            r[key.replace('_ms', '_tflops')] = tf
            r[key.replace('_ms', '_share_of_989')] = tf / PEAK_BF16_TFLOPS
        rows.append(r)
        del g, xs, lo, work, dw, y, wb
        torch.cuda.empty_cache()
    tot = {t: sum(r.get(t + '_ms', 0.0) for r in rows) for t in ('forward', 'dgrad', 'wgrad')}
    return rows, dict(case=case, layer_totals_ms=tot, gpu=gpu_info())


def profile_bf16(case):
    import torch
    from torch.profiler import profile, ProfilerActivity
    from stardist_b200.models.weights import glorot_uniform_weights
    config, spatial, B = make_case(case)
    tr = trainer(config, glorot_uniform_weights(config, seed=0), 'mixed_bfloat16')
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
    return dict(case=case, bf16_ms_per_step_by_kernel={k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:12]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--case", default="all", choices=["2d", "3d", "3d_nb", "all"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.steps < 10:
        raise SystemExit("--steps must be at least 10")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_bf16_bench needs a CUDA device")
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
        r = profile_bf16(c)
        print(json.dumps(r), flush=True)
        res.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
