"""Data-parallel training step time at world sizes 1, 2, 4 and 8 (as far as the visible GPUs go), one process per GPU over
NCCL, for a fixed global batch: the 2-D default (8 x 256^2, 32 rays) and the 3-D default (8 x 64x128^2, 96 rays), each in
'float32' and under the 'mixed_bfloat16' policy.

Every rank runs UNetTrainer.step_replica on its 8 / W items of the same seeded batch.  Step time: CUDA events around each step
after --warmup steps, median over --steps steps per rank, the slowest rank's median reported.  Exchange time: CUDA events
around the all_gather of the rows plus sdb_replica_reduce alone, median over --steps repetitions.  Scaling efficiency at W:
t(1) / (W t(W)).  A world size the visible GPUs cannot hold is reported as not measured.  The card's name, power limit and
max SM clock are read in the same call and printed with every result line.

    python tests/tools/train_parallel_bench.py [--steps 10] [--warmup 3] [--case 2d|3d|all] [--out FILE]
"""
import argparse, json, os, shutil, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train_step_bench import gpu_info, batch
from train_bf16_bench import trainer
from train_parallel_oracle import run_world

GLOBAL_BATCH = 8
WORLDS = (1, 2, 4, 8)


def make_case(case):
    from stardist_b200 import Config2D, Config3D
    if case == '2d':
        return Config2D(n_rays=32), (256, 256)
    from stardist_b200.rays3d import Rays_GoldenSpiral
    return Config3D(rays=Rays_GoldenSpiral(96)), (64, 128, 128)


def _events():
    import torch
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def _rank(rank, world, cases, steps, warmup):
    import torch
    import torch.distributed as dist
    from stardist_b200 import _lib as L
    from stardist_b200.models.weights import glorot_uniform_weights
    lib = L.load()
    b = GLOBAL_BATCH // world
    mine = slice(rank * b, (rank + 1) * b)
    out = []
    for case, setting in cases:
        config, spatial = make_case(case)
        x, p, d = batch(config, spatial, GLOBAL_BATCH, seed=0)
        x, p, d = x[mine], p[mine], d[mine]
        tr = trainer(config, glorot_uniform_weights(config, seed=0), setting)
        for _ in range(warmup):
            tr.step_replica(x, p, d)
        torch.cuda.synchronize()
        dist.barrier()
        ts = []
        for _ in range(steps):
            e0, e1 = _events()
            e0.record(); tr.step_replica(x, p, d); e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        # the exchange alone: all_gather of the rows and the reduction (the state it advances is thrown away with the trainer)
        P, n_out = tr.grad.numel(), tr._n_out()
        dist.barrier()
        xs = []
        for _ in range(steps):
            e0, e1 = _events()
            e0.record()
            rows, w = tr._gather_rows()
            L.check(lib.sdb_replica_reduce(L.ptr(rows), w, P, n_out, tr.row_ld, L.ptr(tr.grad), L.ptr(tr._buf('out', (n_out,))),
                                           L.ptr(tr.state), L.stream_ptr()))
            e1.record()
            e1.synchronize()
            xs.append(e0.elapsed_time(e1))
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        out.append(dict(case=case, setting=setting, step_ms=float(np.median(ts)), exchange_ms=float(np.median(xs)),
                        row_mb=tr.row_ld * 4 / 1e6, params=P, peak_gib=peak))
        del tr, x, p, d
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--case', default='all', choices=['2d', '3d', 'all'])
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_parallel_bench needs CUDA devices")
    n_gpu = torch.cuda.device_count()
    info = gpu_info()
    cases = [(c, s) for c in (('2d', '3d') if a.case == 'all' else (a.case,)) for s in ('float32', 'mixed_bfloat16')]
    tmp = tempfile.mkdtemp(prefix='train_parallel_bench_')
    results, lines = {}, []
    try:
        for W in WORLDS:
            if W > n_gpu:
                continue
            ranks = run_world(_rank, W, tmp, args=(cases, a.steps, a.warmup), backend='nccl', devices=list(range(W)), timeout=3000)
            for i, (case, setting) in enumerate(cases):
                rs = [r[i] for r in ranks]
                results[(case, setting, W)] = dict(rs[0], step_ms=max(r['step_ms'] for r in rs),
                                                   exchange_ms=max(r['exchange_ms'] for r in rs), peak_gib=max(r['peak_gib'] for r in rs))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    for case, setting in cases:
        t1 = results.get((case, setting, 1), {}).get('step_ms')
        for W in WORLDS:
            r = results.get((case, setting, W))
            line = dict(case=case, setting=setting, world=W, global_batch=GLOBAL_BATCH, gpu=info)
            if r is None:
                line['result'] = 'not measured (%d GPU(s) visible)' % n_gpu
            else:
                line.update(step_ms=round(r['step_ms'], 3), exchange_ms=round(r['exchange_ms'], 4), row_mb=round(r['row_mb'], 2),
                            params=r['params'], peak_gib=round(r['peak_gib'], 2),
                            efficiency=None if t1 is None else round(t1 / (W * r['step_ms']), 3))
            lines.append(line)
            print(json.dumps(line), flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
