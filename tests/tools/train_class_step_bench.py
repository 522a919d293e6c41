"""Time one training step of a multi-class model (n_classes=3: the features_class / prob_class branch and its weighted
categorical cross-entropy) on the defaults of train_step_bench.py (2-D: batch 4 x 256^2, 32 rays; 3-D U-Net: 1 x 128^3,
96 rays), next to the single-class step of the same configuration timed in the same process, so the line reports the
class branch's overhead.  Also the multi-class step in torch autograd with cuDNN at fp32 (TF32 off) as a comparison point.
Prints one JSON line per case.

FLOPs are counted as in train_step_bench.py, with the features_class and prob_class layers included.  --profile prints
instead the per-kernel device time of 3 multi-class steps (torch.profiler).

    python tests/tools/train_class_step_bench.py [--steps 20] [--warmup 3] [--case 2d|3d|all] [--out FILE] [--profile]
"""
import argparse, json, os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_step_bench as B

N_CLASSES = 3


def step_flops(config, spatial, batch):
    from stardist_b200.models.weights import unet_layers
    size = np.array(spatial, np.int64)
    total, first = 0, None
    for l in unet_layers(config):
        if l['kind'] == 'pool':
            size = size // np.array(l['pool'])
        elif l['kind'] == 'up':
            size = size * np.array(l['pool'])
        elif l['kind'] in ('conv', 'head', 'conv_class', 'head_class'):
            f = 2 * batch * int(np.prod(size)) * int(np.prod(l['k'])) * l['cin'] * l['cout']
            first = f if first is None else first
            total += f
    return 3 * total - first


def make_case(case):
    """(single-class config, multi-class config, spatial, batch)"""
    from stardist_b200 import Config2D, Config3D
    single, spatial, bs = B.make_case(case)
    if case == '2d':
        return single, Config2D(n_rays=32, n_classes=N_CLASSES), spatial, bs
    from stardist_b200.rays3d import Rays_GoldenSpiral
    return single, Config3D(rays=Rays_GoldenSpiral(96), n_classes=N_CLASSES), spatial, bs


def class_target(config, spatial, batch, seed=1):
    """one-hot prob_class targets [B, *grid-spatial, n_classes + 1] on the device, 10 % of the pixels ignored (-1)"""
    import torch
    rng = np.random.default_rng(seed)
    pg = tuple(s // g for s, g in zip(spatial, config.grid))
    C = config.n_classes + 1
    pc = np.eye(C, dtype=np.float32)[rng.integers(0, C, (batch,) + pg)]
    pc[rng.uniform(0, 1, (batch,) + pg) < 0.1] = -1
    return torch.from_numpy(pc).cuda()


def run_case(case, steps, warmup):
    import torch
    import train_oracle as O
    import train_oracle_classes as OC
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    single, config, spatial, bs = make_case(case)
    x, p, d = B.batch(single, spatial, bs)
    pc = class_target(config, spatial, bs)
    tr1 = UNetTrainer(single, glorot_uniform_weights(single, seed=0))
    ms_single = B.time_it(lambda: tr1.step(x, p, d), steps, warmup)
    del tr1
    torch.cuda.empty_cache()
    weights = glorot_uniform_weights(config, seed=0)
    torch.cuda.reset_peak_memory_stats()
    tr = UNetTrainer(config, weights)
    ms = B.time_it(lambda: tr.step(x, p, d, pc), steps, warmup)
    peak = torch.cuda.max_memory_allocated()
    names = tr.names
    del tr
    torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    P = O.params64(weights, names)
    P = {n: (k.detach().float().cuda().requires_grad_(True), b.detach().float().cuda().requires_grad_(True)) for n, (k, b) in P.items()}
    opt = torch.optim.Adam([t for kb in P.values() for t in kb], lr=config.train_learning_rate, eps=1e-7)
    w = tuple(float(v) for v in config.train_loss_weights)

    def torch_step():
        opt.zero_grad(set_to_none=True)
        prob, dist, prob_class = OC.forward64_classes(config, P, x)
        loss = O.loss64(prob, dist, p, d, dist_loss=config.train_dist_loss, lam=float(config.train_background_reg), weights=w[:2])[0]
        loss = loss + w[2] * OC.class_loss64(prob_class, pc, config.train_class_weights)
        loss.backward()
        opt.step()

    ms_t = B.time_it(torch_step, steps, warmup)
    flops = step_flops(config, spatial, bs)
    return dict(case=case + "_classes", n_classes=N_CLASSES, batch=bs, spatial=list(spatial), n_rays=config.n_rays, step_ms=ms,
                single_class_step_ms=ms_single, class_overhead=ms / ms_single - 1, tflop_per_step=flops / 1e12,
                achieved_tflops=flops / (ms * 1e-3) / 1e12, peak_mem_gb=peak / 1e9, torch_cudnn_fp32_step_ms=ms_t, gpu=B.gpu_info())


def profile_case(case):
    import torch
    from torch.profiler import profile, ProfilerActivity
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    single, config, spatial, bs = make_case(case)
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=0))
    x, p, d = B.batch(single, spatial, bs)
    pc = class_target(config, spatial, bs)
    for _ in range(2):
        tr.step(x, p, d, pc)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            tr.step(x, p, d, pc)
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = e.name.replace('(anonymous namespace)::', '')[:60]
            tot[k] = tot.get(k, 0.0) + e.device_time_total / 3e3
    print(json.dumps(dict(case=case + "_classes", ms_per_step_by_kernel={k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:16]})))


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
        raise SystemExit("train_class_step_bench needs a CUDA device")
    cases = ["2d", "3d"] if a.case == "all" else [a.case]
    if a.profile:
        for c in cases:
            profile_case(c)
        return
    res = [run_case(c, a.steps, a.warmup) for c in cases]
    for r in res:
        print(json.dumps(r))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
