"""Data-parallel training on the device (models/train.py UNetTrainer.step_replica and train() with a torch.distributed
group, csrc/unet_train.cu sdb_replica_reduce).  The multi-rank checks run two ranks on one GPU over gloo, in one spawned
world whose results the tests below read: the per-step reduced gradient against the one-process mean of the halves'
gradients and float64 autograd, rank identity and determinism in fp32 / TF32 / mixed_bfloat16, empty sub-batches and
train() end to end.  A world of 1 is checked against train() without a group, and NCCL over two GPUs against gloo on one
where two GPUs are visible."""
import os, sys, warnings
import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_oracle as O
import train_oracle_classes as OC
from train_parallel_oracle import replica_reduce_np, run_world, digest

pytestmark = pytest.mark.gpu

GRAD_CASES = ['2d_default', '3d_default', '3d_pool122', '2d_classes3']
# float64 autograd within 1e-4: the 3-D U-Net of tests/test_gpu_train.py, whose bound it is.  The default 3-D U-Net on 16x32^2
# patches is left out: there the fp32 backward pass itself is 1.5e-4 from float64 in one tensor (down_level_1_no_0), while the
# reduced gradient is bit-equal to the one-process mean of the halves'.
F64_CASES = ['2d_default', '3d_pool122', '2d_classes3']


def _config(case, batch_size=2):
    from stardist_b200 import Config2D, Config3D
    if case == '2d_default':
        return Config2D(train_patch_size=(64, 64), train_batch_size=batch_size)
    if case == '2d_classes3':
        return Config2D(n_classes=3, train_patch_size=(64, 64), train_batch_size=batch_size)
    if case == '2d_small':
        return Config2D(n_rays=16, unet_n_depth=2, grid=(1, 1), train_patch_size=(64, 64), train_batch_size=batch_size,
                        train_learning_rate=1e-3)
    if case == '3d_pool122':
        from stardist_b200.rays3d import Rays_GoldenSpiral
        return Config3D(rays=Rays_GoldenSpiral(24), unet_n_depth=2, unet_n_filter_base=32, unet_pool=(1, 2, 2), grid=(1, 2, 2),
                        train_patch_size=(6, 16, 16), train_batch_size=batch_size, train_background_reg=1e-4)
    return Config3D(n_rays=48, train_patch_size=(16, 32, 32), train_batch_size=batch_size)


def _batches(config, seed=0, length=1):
    from test_gpu_train_any import _batches as batches
    return batches(config, seed=seed, length=length)


def _halves(batch, world=2):
    (x,), targets = batch
    b = x.shape[0] // world
    return [(x[r * b:(r + 1) * b], tuple(t[r * b:(r + 1) * b] for t in targets)) for r in range(world)]


def _flat_grad(tr, x, targets):
    tr.gradients(x, *targets)
    return tr.grad.cpu().numpy().copy()


def _state(tr):
    return tr.params, tr.m, tr.v, tr.state


# ------------------------------------------------------------------------------------------------ the two-rank world
def _world_checks(rank, world):
    from stardist_b200 import enable_tensor_float_32_execution
    from stardist_b200.mixed_precision import set_global_policy
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    res = {}
    # per-step gradient: the reduced gradient and loss row, and rank 0's one-process gradients of the two halves
    for case in GRAD_CASES:
        config = _config(case)
        weights = glorot_uniform_weights(config, seed=1)
        batch = _batches(config)[0]
        halves = _halves(batch)
        tr = UNetTrainer(config, weights)
        x, t = halves[rank]
        out = tr.step_replica(x, *t).cpu().numpy()
        r = dict(grad=tr.grad.cpu().numpy(), out=out, state=tr.state.cpu().numpy())
        if rank == 0:
            ref = UNetTrainer(config, weights)
            gs = [_flat_grad(ref, hx, ht) for hx, ht in halves]
            r.update(g_halves=gs, weights=weights, names=tr.names, offsets=tr.offsets, shapes=tr.shapes,
                     halves=[(hx.cpu().numpy(), [ti.cpu().numpy() for ti in ht]) for hx, ht in halves])
        res[('grad', case)] = r
    # rank identity and determinism in every precision mode: two runs of four steps each
    config = _config('2d_default', batch_size=4)
    batches = _batches(config, seed=5, length=4)
    for mode in ('fp32', 'tf32', 'bf16'):
        runs = []
        for _ in range(2):
            enable_tensor_float_32_execution(mode == 'tf32')
            set_global_policy('mixed_bfloat16' if mode == 'bf16' else 'float32')
            try:
                tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
            finally:
                enable_tensor_float_32_execution(False)
                set_global_policy('float32')
            losses = []
            for b in batches:
                x, t = _halves(b)[rank]
                losses.append(tr.step_replica(x, *t).cpu().numpy().copy())
            runs.append(dict(digest=digest(*_state(tr)), losses=np.stack(losses), state=tr.state.cpu().numpy()))
        res[('identity', mode)] = runs
    # empty sub-batches: rank 1's half, then both halves, without a labelled pixel
    config = _config('2d_small')
    weights = glorot_uniform_weights(config, seed=2)
    batch = _batches(config, seed=6)[0]
    for which in ('one', 'both'):
        (x, t) = _halves(batch)[rank]
        if rank == 1 or which == 'both':
            t = (torch.full_like(t[0], -1.0),) + tuple(t[1:])
        tr = UNetTrainer(config, weights)
        p0 = tr.params.cpu().numpy().copy()
        out = tr.step_replica(x, *t).cpu().numpy()
        r = dict(grad=tr.grad.cpu().numpy(), out=out, state=tr.state.cpu().numpy(), moved=not np.array_equal(p0, tr.params.cpu().numpy()),
                 digest=digest(*_state(tr)))
        if rank == 0 and which == 'one':
            r['g_half0'] = _flat_grad(UNetTrainer(config, weights), *_halves(batch)[0])
        res[('empty', which)] = r
    return res


def _train_e2e(rank, world, basedir):
    from test_gpu_train_any import _small_data
    from stardist_b200 import StarDist2D
    X, Y = _small_data(2, n=6, seed=10)
    config = _config('2d_small', batch_size=4)
    model = StarDist2D(config, name='m', basedir=os.path.join(basedir, 'rank%d' % rank))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        hist = model.train(X[:4], Y[:4], validation_data=(X[4:], Y[4:]), seed=0, epochs=4, steps_per_epoch=30)
    folder = model.logdir
    files = sorted(os.listdir(folder)) if os.path.exists(folder) else None
    return dict(history=hist.history, epoch=hist.epoch, weights=digest(*[a for n in sorted(model.weights) for a in model.weights[n]]),
                files=files)


def _identity_fp32(rank, world):
    """the fp32 rank-identity run of _world_checks alone (for the placement check)"""
    from stardist_b200.models.train import UNetTrainer
    from stardist_b200.models.weights import glorot_uniform_weights
    config = _config('2d_default', batch_size=4)
    tr = UNetTrainer(config, glorot_uniform_weights(config, seed=4))
    for b in _batches(config, seed=5, length=4):
        x, t = _halves(b)[rank]
        tr.step_replica(x, *t)
    return digest(*_state(tr))


@pytest.fixture(scope="module")
def world2(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("dp2")
    return run_world(_world_checks, 2, tmp, devices=[0, 0], timeout=1200)


# ------------------------------------------------------------------------------------------------ 1. the kernel
def test_reduction_kernel_bit_equal_to_numpy():
    from stardist_b200 import _lib as L
    lib = L.require_cuda()
    rng = np.random.default_rng(0)
    for W in range(1, 9):
        for P, n_out in ((1, 4), (4097, 5), (100003, 4)):
            # float4 rows, and rows off the 16-byte grid
            for ld in (-(-(P + n_out) // 4) * 4, P + n_out + (1 if (P + n_out + 1) % 4 else 2)):
                masks = [np.zeros(W, bool), np.ones(W, bool), rng.random(W) < 0.5]
                for ok in masks:
                    rows = (rng.standard_normal((W, ld)) * 1e3 ** rng.integers(-2, 3, (W, 1))).astype(np.float32)
                    rows[:, P + 3] = np.where(ok, 0, 1)
                    state0 = np.array([7, 3, 1], np.int32)
                    want_g, want_out, want_state = replica_reduce_np(rows, P, n_out, state0)
                    d_rows = torch.from_numpy(rows.reshape(-1)).cuda()
                    g = torch.full((P,), np.nan, dtype=torch.float32, device='cuda')
                    out = torch.empty(n_out, dtype=torch.float32, device='cuda')
                    st = torch.from_numpy(state0).cuda()
                    L.check(lib.sdb_replica_reduce(L.ptr(d_rows), W, P, n_out, ld, L.ptr(g), L.ptr(out), L.ptr(st), L.stream_ptr()))
                    case = (W, P, n_out, ld, ok.tolist())
                    assert np.array_equal(g.cpu().numpy().view(np.int32), want_g.view(np.int32)), case
                    assert np.array_equal(out.cpu().numpy().view(np.int32), want_out.view(np.int32)), case
                    assert np.array_equal(st.cpu().numpy(), want_state), case
    # a world of 1 reduces its row in place: g aliases the row's head
    P = 1001
    row = torch.from_numpy(rng.standard_normal(1008).astype(np.float32)).cuda()
    row[P + 3] = 0
    want = row[:P].cpu().numpy().copy()
    out = torch.empty(4, dtype=torch.float32, device='cuda')
    st = torch.zeros(3, dtype=torch.int32, device='cuda')
    L.check(lib.sdb_replica_reduce(L.ptr(row), 1, P, 4, 1008, L.ptr(row), L.ptr(out), L.ptr(st), L.stream_ptr()))
    assert np.array_equal(row[:P].cpu().numpy().view(np.int32), want.view(np.int32)) and tuple(st.cpu().numpy()) == (1, 0, 0)


# ------------------------------------------------------------------------------------------------ 2. per-step gradient
@pytest.mark.parametrize("case", GRAD_CASES)
def test_reduced_gradient_is_the_mean_of_the_halves(world2, case):
    r0, r1 = world2[0][('grad', case)], world2[1][('grad', case)]
    g0, g1 = r0['g_halves']
    want = ((g0 + g1) / np.float32(2)).astype(np.float32)
    assert np.array_equal(r0['grad'].view(np.int32), want.view(np.int32))
    assert np.array_equal(r1['grad'].view(np.int32), want.view(np.int32))
    assert np.array_equal(r0['out'].view(np.int32), r1['out'].view(np.int32))
    assert tuple(r0['state']) == tuple(r1['state']) == (1, 0, 0)


@pytest.mark.parametrize("case", F64_CASES)
def test_reduced_gradient_against_float64_autograd_of_the_mean_loss(world2, case):
    """within the relative L2 bound 1e-4 of tests/test_gpu_train_any.py, against float64 autograd of (L(half 0) + L(half 1)) / 2"""
    from test_gpu_train_any import _forward64
    r = world2[0][('grad', case)]
    config = _config(case)
    weights = r['weights']
    W = {n: tuple(torch.from_numpy(np.asarray(a, np.float64)).requires_grad_(True) for a in weights[n]) for n in r['names']}
    w = tuple(float(v) for v in config.train_loss_weights)
    losses = []
    for x, t in r['halves']:
        prob, dist, pc = _forward64(config, W, torch.from_numpy(x).double())
        tot, _, _ = O.loss64(prob, dist, torch.from_numpy(t[0]).double(), torch.from_numpy(t[1]).double(), dist_loss=config.train_dist_loss,
                             lam=float(config.train_background_reg), weights=w[:2])
        if pc is not None:
            tot = tot + w[2] * OC.class_loss64(pc, torch.from_numpy(t[2]).double(), config.train_class_weights)
        losses.append(tot)
    mean = (losses[0] + losses[1]) / 2
    mean.backward()
    assert abs(float(r['out'][0]) - mean.item()) <= 1e-4 * abs(mean.item())
    worst = 0.0
    for n in r['names']:
        (ks, bs), off = r['shapes'][n], r['offsets'][n]
        nk, nb = int(np.prod(ks)), int(np.prod(bs))
        for a, b in ((r['grad'][off:off + nk], W[n][0]), (r['grad'][off + nk:off + nk + nb], W[n][1])):
            b = b.grad.numpy().reshape(-1)
            rel = np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30)
            worst = max(worst, rel)
            assert rel <= 1e-4, (n, rel)
    print("%s: worst relative L2 gradient error %.3g" % (case, worst))


# ------------------------------------------------------------------------------------------------ 3. identity, determinism
@pytest.mark.parametrize("mode", ['fp32', 'tf32', 'bf16'])
def test_ranks_bit_identical_and_runs_deterministic(world2, mode):
    a, b = world2[0][('identity', mode)], world2[1][('identity', mode)]
    for run in range(2):
        assert a[run]['digest'] == b[run]['digest'], "params / m / v / state differ between ranks"
        assert np.array_equal(a[run]['losses'], b[run]['losses'])
        assert tuple(a[run]['state']) == (4, 0, 0)
    assert a[0]['digest'] == a[1]['digest'] and np.array_equal(a[0]['losses'], a[1]['losses'])


# ------------------------------------------------------------------------------------------------ 4. empty sub-batches
def test_one_empty_half_gives_the_other_halfs_gradient(world2):
    r0, r1 = world2[0][('empty', 'one')], world2[1][('empty', 'one')]
    want = r0['g_half0']
    for r in (r0, r1):
        assert np.array_equal(r['grad'].view(np.int32), want.view(np.int32))
        assert tuple(r['state']) == (1, 0, 0) and r['out'][3] == 0 and r['moved']
    assert r0['digest'] == r1['digest']


def test_both_halves_empty_skip_the_step_on_both_ranks(world2):
    r0, r1 = world2[0][('empty', 'both')], world2[1][('empty', 'both')]
    for r in (r0, r1):
        assert tuple(r['state']) == (0, 1, 1) and r['out'][3] == 1 and not r['moved']
    assert r0['digest'] == r1['digest']


# ------------------------------------------------------------------------------------------------ 5. a world of 1
def test_world_of_one_equals_training_without_a_group(tmp_path):
    import torch.distributed as dist
    from test_gpu_train_any import _small_data
    from stardist_b200 import StarDist2D
    X, Y = _small_data(2, n=5, seed=12)
    runs = []
    for grouped in (False, True):
        if grouped:
            dist.init_process_group('gloo', store=dist.FileStore(str(tmp_path / 'store1'), 1), rank=0, world_size=1)
        try:
            model = StarDist2D(_config('2d_small', batch_size=2), name=None, basedir=None)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                hist = model.train(X[:3], Y[:3], validation_data=(X[3:], Y[3:]), seed=3, epochs=2, steps_per_epoch=10)
        finally:
            if grouped:
                dist.destroy_process_group()
        runs.append((hist.history, digest(*[a for n in sorted(model.weights) for a in model.weights[n]])))
    (h0, w0), (h1, w1) = runs
    assert w0 == w1
    assert h0.keys() == h1.keys()
    for k in h0:
        assert np.array_equal(np.asarray(h0[k]), np.asarray(h1[k]), equal_nan=True), k


# ------------------------------------------------------------------------------------------------ 6. train() end to end
def test_train_two_ranks_end_to_end(tmp_path):
    r0, r1 = run_world(_train_e2e, 2, tmp_path, args=(str(tmp_path),), devices=[0, 0], timeout=1200)
    h = r0['history']
    print("val_loss per epoch:", ["%.4f" % v for v in h['val_loss']])
    assert h == r1['history'] and r0['epoch'] == r1['epoch'] == list(range(4))
    assert set(h) == {'loss', 'prob_loss', 'dist_loss', 'val_loss', 'val_prob_loss', 'val_dist_loss', 'lr'}
    assert h['val_loss'][-1] < h['val_loss'][0]
    assert r0['weights'] == r1['weights']
    assert r0['files'] == ['config.json', 'weights.npz', 'weights_last.npz'] and r1['files'] is None


# ------------------------------------------------------------------------------------------------ 7. placement
def test_nccl_on_two_gpus_equals_gloo_on_one(request, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("%d GPU visible: NCCL over two devices needs two" % torch.cuda.device_count())
    world2 = request.getfixturevalue('world2')
    got = run_world(_identity_fp32, 2, tmp_path, backend='nccl', devices=[0, 1], timeout=600)
    want = world2[0][('identity', 'fp32')][0]['digest']
    assert got[0] == got[1] == want
