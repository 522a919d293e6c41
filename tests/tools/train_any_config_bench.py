"""Time one training step (UNetTrainer.step) of configurations outside the default architecture family at user sizes
(batch 4 x 256^2 in 2-D, 1 x 64x128^2 in 3-D), and in the same process the 3^d ReLU configuration of the same shape and
width, and the same step in torch autograd with cuDNN at fp32 (TF32 off).  Prints one JSON line per case, with the card's
name and power limit.

FLOPs as in train_step_bench.py: 3 x the forward FLOPs minus the first convolution's input gradient.  Times: CUDA events
around each step after warm-up, median over --steps steps.

    python tests/tools/train_any_config_bench.py [--steps 20] [--warmup 3] [--case NAME|all] [--out FILE]
"""
import argparse, json, os, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))

CASES = ['2d_k55_elu', '2d_k22_swish', '2d_base16_gelu_cin3', '3d_k133_pool122', '2d_classes_k55_selu']


def make_case(case, default=False):
    """(config, spatial, batch); default=True: the same shape and widths with 3^d kernels and ReLU"""
    from stardist_b200 import Config2D, Config3D
    from stardist_b200.rays3d import Rays_GoldenSpiral
    kw = {
        '2d_k55_elu': dict(unet_kernel_size=(5, 5), unet_activation='elu'),
        '2d_k22_swish': dict(unet_kernel_size=(2, 2), unet_activation='swish', unet_last_activation='softplus'),
        '2d_base16_gelu_cin3': dict(unet_n_filter_base=16, unet_activation='gelu', n_channel_in=3),
        '2d_classes_k55_selu': dict(unet_kernel_size=(5, 5), unet_activation='selu', n_classes=3),
        '3d_k133_pool122': dict(unet_kernel_size=(1, 3, 3), unet_pool=(1, 2, 2), grid=(1, 2, 2)),
    }[case]
    if default:
        kw = {k: v for k, v in kw.items() if k not in ('unet_kernel_size', 'unet_activation', 'unet_last_activation')}
    if case.startswith('3d'):
        return Config3D(rays=Rays_GoldenSpiral(96), **kw), (64, 128, 128), 1
    return Config2D(n_rays=32, **kw), (256, 256), 4


def batch(config, spatial, B, seed=0):
    import torch
    rng = np.random.default_rng(seed)
    R = config.n_rays
    pg = tuple(s // g for s, g in zip(spatial, config.grid))
    x = torch.from_numpy(rng.normal(0, 1, (B,) + tuple(spatial) + (config.n_channel_in,)).astype(np.float32)).cuda()
    p = torch.from_numpy(rng.uniform(0, 1, (B,) + pg).astype(np.float32)).cuda()
    dam = rng.uniform(0, 10, (B,) + pg + (R + 1,)).astype(np.float32)
    dam[..., R] = rng.uniform(0, 1, (B,) + pg) < 0.4
    out = [x, p, torch.from_numpy(dam).cuda()]
    if config.n_classes is not None:
        C = config.n_classes + 1
        out.append(torch.from_numpy(np.eye(C, dtype=np.float32)[rng.integers(0, C, (B,) + pg)]).cuda())
    return out


def torch_step_fn(config, weights, x, targets):
    """the same step in torch autograd (fp32, cuDNN, TF32 off): the any_config_oracle walk with TF 'same' padding, the
    float64 loss restatements evaluated in float32, Adam"""
    import torch
    import any_config_oracle as AO
    import train_oracle as O
    import train_oracle_classes as OC
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    W = {n: tuple(torch.from_numpy(np.asarray(a, np.float32)).cuda().requires_grad_(True) for a in kb) for n, kb in weights.items()}
    opt = torch.optim.Adam([t for kb in W.values() for t in kb], lr=config.train_learning_rate, eps=1e-7)
    w = tuple(float(v) for v in config.train_loss_weights)

    def step():
        opt.zero_grad(set_to_none=True)
        feat, base, act = AO._unet(config, W, x)
        prob, dist = AO._heads(W, feat, None)
        loss = O.loss64(prob, dist, targets[0], targets[1], dist_loss=config.train_dist_loss, lam=float(config.train_background_reg),
                        weights=w[:2])[0]
        if config.n_classes is not None:
            loss = loss + w[2] * OC.class_loss64(AO._class(config, W, base, act), targets[2], config.train_class_weights)
        loss.backward()
        opt.step()
    return step


def run_case(case, steps, warmup):
    import torch
    from train_step_bench import step_flops, gpu_info, time_it
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    res = dict(case=case)
    for tag, default in (('', False), ('default3_relu_', True)):
        config, spatial, B = make_case(case, default)
        weights = glorot_uniform_weights(config, seed=0)
        x, *targets = batch(config, spatial, B)
        torch.cuda.reset_peak_memory_stats()
        tr = UNetTrainer(config, weights)
        ms = time_it(lambda: tr.step(x, *targets), steps, warmup)
        peak = torch.cuda.max_memory_allocated()
        del tr
        torch.cuda.empty_cache()
        flops = step_flops(config, spatial, B)
        res.update({tag + 'step_ms': ms, tag + 'tflop_per_step': flops / 1e12, tag + 'achieved_tflops': flops / (ms * 1e-3) / 1e12,
                    tag + 'peak_mem_gb': peak / 1e9})
        if not default:
            res.update(batch=B, spatial=list(spatial), n_rays=config.n_rays)
            ms_t = time_it(torch_step_fn(config, weights, x, targets), steps, warmup)
            res.update(torch_cudnn_fp32_step_ms=ms_t, torch_achieved_tflops=flops / (ms_t * 1e-3) / 1e12)
            torch.cuda.empty_cache()
    res['gpu'] = gpu_info()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--case", default="all", choices=CASES + ["all"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_any_config_bench needs a CUDA device")
    res = []
    for c in (CASES if a.case == "all" else [a.case]):
        res.append(run_case(c, a.steps, a.warmup))
        print(json.dumps(res[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
