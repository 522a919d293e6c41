"""Time one training step (UNetTrainer.step: forward with saved activations, loss, backward, Adam) for the 2-D default
configuration (batch 4 x 256^2, 32 rays) and the 3-D U-Net default (1 x 128^3, 96 rays), and the same step in torch
autograd with cuDNN at fp32 (TF32 off) on the same GPU as a comparison point.  Prints one JSON line per case.

FLOPs are counted from the layer shapes: a step is 3 x the forward FLOPs (forward, input gradient, weight gradient) minus
the first convolution's input gradient, which is never computed.  Times: CUDA events around each step after warm-up,
median over --steps steps.

    python tests/tools/train_step_bench.py [--steps 20] [--warmup 3] [--case 2d|3d|all] [--out FILE]
"""
import argparse, json, os, sys, subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def step_flops(config, spatial, batch):
    from stardist_b200.models.weights import unet_layers
    size = np.array(spatial, np.int64)
    total, first = 0, None
    for l in unet_layers(config):
        if l['kind'] == 'pool':
            size = size // np.array(l['pool'])
        elif l['kind'] == 'up':
            size = size * np.array(l['pool'])
        elif l['kind'] in ('conv', 'head'):
            f = 2 * batch * int(np.prod(size)) * int(np.prod(l['k'])) * l['cin'] * l['cout']
            first = f if first is None else first
            total += f
    return 3 * total - first


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:           # the numbers stay meaningful only with this line; report why it is missing
        return "unavailable: %s" % e


def make_case(case):
    from stardist_b200 import Config2D, Config3D
    if case == '2d':
        return Config2D(n_rays=32), (256, 256), 4
    from stardist_b200.rays3d import Rays_GoldenSpiral
    return Config3D(rays=Rays_GoldenSpiral(96)), (128, 128, 128), 1


def batch(config, spatial, B, seed=0):
    import torch
    rng = np.random.default_rng(seed)
    R = config.n_rays
    pg = tuple(s // g for s, g in zip(spatial, config.grid))
    x = torch.from_numpy(rng.normal(0, 1, (B,) + tuple(spatial) + (1,)).astype(np.float32)).cuda()
    p = torch.from_numpy(rng.uniform(0, 1, (B,) + pg + (1,)).astype(np.float32)).cuda()
    dam = rng.uniform(0, 10, (B,) + pg + (R + 1,)).astype(np.float32)
    dam[..., R] = rng.uniform(0, 1, (B,) + pg) < 0.4
    return x, p, torch.from_numpy(dam).cuda()


def time_it(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def run_case(case, steps, warmup):
    import torch
    import train_oracle as O
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config, spatial, B = make_case(case)
    weights = glorot_uniform_weights(config, seed=0)
    x, p, d = batch(config, spatial, B)
    flops = step_flops(config, spatial, B)
    torch.cuda.reset_peak_memory_stats()
    tr = UNetTrainer(config, weights)
    ms = time_it(lambda: tr.step(x, p, d), steps, warmup)
    peak = torch.cuda.max_memory_allocated()
    del tr
    torch.cuda.empty_cache()
    # torch autograd comparison: the same walk, loss and Adam in fp32 with cuDNN, TF32 off
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    P = O.params64(weights, [l['name'] for l in __import__('stardist_b200.models.weights', fromlist=['x']).unet_layers(config)
                             if l['kind'] in ('conv', 'head')])
    P = {n: (k.detach().float().cuda().requires_grad_(True), b.detach().float().cuda().requires_grad_(True)) for n, (k, b) in P.items()}
    opt = torch.optim.Adam([t for kb in P.values() for t in kb], lr=config.train_learning_rate, eps=1e-7)

    def torch_step():
        opt.zero_grad(set_to_none=True)
        prob, dist = O.forward64(config, P, x)
        loss = O.loss64(prob, dist, p, d, dist_loss=config.train_dist_loss, lam=float(config.train_background_reg),
                        weights=tuple(float(v) for v in config.train_loss_weights))[0]
        loss.backward()
        opt.step()

    torch.cuda.reset_peak_memory_stats()
    ms_t = time_it(torch_step, steps, warmup)
    peak_t = torch.cuda.max_memory_allocated()
    return dict(case=case, batch=B, spatial=list(spatial), n_rays=config.n_rays, step_ms=ms, tflop_per_step=flops / 1e12,
                achieved_tflops=flops / (ms * 1e-3) / 1e12, peak_mem_gb=peak / 1e9, torch_cudnn_fp32_step_ms=ms_t,
                torch_achieved_tflops=flops / (ms_t * 1e-3) / 1e12, torch_peak_mem_gb=peak_t / 1e9, gpu=gpu_info())


def profile_case(case):
    import torch
    from torch.profiler import profile, ProfilerActivity
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config, spatial, B = make_case(case)
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=0))
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
    print(json.dumps(dict(case=case, ms_per_step_by_kernel={k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:12]})))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--case", default="all", choices=["2d", "3d", "all"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="instead: per-kernel device time of 3 steps (torch.profiler)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_step_bench needs a CUDA device")
    if a.profile:
        for c in (["2d", "3d"] if a.case == "all" else [a.case]):
            profile_case(c)
        return
    res = [run_case(c, a.steps, a.warmup) for c in (["2d", "3d"] if a.case == "all" else [a.case])]
    for r in res:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
