"""Data-parallel training (models/train.py UNetTrainer.step_replica, csrc/unet_train.cu sdb_replica_reduce): the reduction rule
restated in numpy, and a runner that starts a torch.distributed world of spawned processes on a FileStore (no TCP port),
joins them with a timeout and terminates them on failure."""
import hashlib
import os
import traceback
import numpy as np


def replica_reduce_np(rows, n_params, n_out, state):
    """rows float32 [W][>= n_params + n_out] (gradient, then loss row (loss, prob_loss, dist_loss, skipped, ...)), state int
    (t, n_skipped, skip) -> (g [n_params], out [n_out], state): the mean over S, the replicas with skipped == 0 in ascending
    rank order or all of them when none is, as float32 additions from S's first member and one float32 division; the state
    advances once, as a skipped step when no replica is ok"""
    rows = np.asarray(rows, np.float32)
    W = rows.shape[0]
    ok = [r for r in range(W) if rows[r, n_params + 3] == 0]
    members = ok if ok else list(range(W))
    acc = rows[members[0], :n_params + n_out].copy()
    for r in members[1:]:
        acc = (acc + rows[r, :n_params + n_out]).astype(np.float32)
    red = (acc / np.float32(len(members))).astype(np.float32)
    state = np.array(state, np.int64).copy()
    skip = not ok
    state[2] = int(skip)
    state[1 if skip else 0] += 1
    return red[:n_params], red[n_params:], state


def digest(*arrays):
    """sha256 over the raw bytes of numpy arrays / tensors (bit-identity across processes)"""
    h = hashlib.sha256()
    for a in arrays:
        a = a.detach().cpu().numpy() if hasattr(a, 'detach') else np.asarray(a)
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _entry(rank, world, store_path, backend, devices, fn, args, q):
    try:
        os.environ.setdefault('GLOO_SOCKET_IFNAME', 'lo')          # the ranks talk over the loopback device only
        import torch
        import torch.distributed as dist
        if devices is not None:
            torch.cuda.set_device(devices[rank])
        store = dist.FileStore(store_path, world)
        dist.init_process_group(backend, store=store, rank=rank, world_size=world)
        try:
            q.put((rank, 'ok', fn(rank, world, *args)))
        finally:
            dist.destroy_process_group()
    except BaseException:
        q.put((rank, 'error', traceback.format_exc()))


def run_world(fn, world, tmp_path, args=(), backend='gloo', devices=None, timeout=900):
    """run fn(rank, world, *args) in `world` spawned processes of one torch.distributed group (FileStore under tmp_path;
    `devices`: each rank's CUDA device, None for none) and return their results by rank.  Processes still alive after
    `timeout` seconds, or after another rank failed, are terminated."""
    import queue
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    store = os.path.join(str(tmp_path), 'store_%s_%d' % (fn.__name__, os.getpid()))
    if os.path.exists(store):
        os.remove(store)
    procs = [ctx.Process(target=_entry, args=(r, world, store, backend, devices, fn, args, q)) for r in range(world)]
    for p in procs:
        p.start()
    out, errors = {}, []
    try:
        for _ in range(world):
            try:
                rank, status, res = q.get(timeout=timeout)
            except queue.Empty:
                errors.append('no result within %d s' % timeout)
                break
            if status != 'ok':
                errors.append('rank %d:\n%s' % (rank, res))
                break
            out[rank] = res
        for p in procs:
            p.join(timeout=60 if not errors else 5)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    assert not errors, '\n'.join(errors)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [out[r] for r in range(world)]
