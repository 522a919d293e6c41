"""numpy float32 restatement of the per-ray arithmetic of csrc/stardist.cu (k_star_dist_2d / k_star_dist_3d): every operation
is one float32 op in the kernel's order, np.rint is lrint's round-half-even.  Driven by a direction table, it pins the
table and the operation order against the reference's C++ without a GPU."""
import numpy as np

f32 = np.float32


def _walk(lbl16, starts, dirs, step_exit):
    """starts int [P, ndim] pixel positions, dirs float32 [ndim, R] -> float32 [P, R]"""
    ndim, R = dirs.shape
    P = len(starts)
    value = lbl16[tuple(starts.T)]
    out = np.zeros((P, R), f32)
    fg = np.flatnonzero(value != 0)
    if len(fg) == 0:
        return out
    pos = [np.broadcast_to(starts[fg, a].astype(f32)[:, None], (len(fg), R)) for a in range(ndim)]
    d = [np.broadcast_to(dirs[a][None, :], (len(fg), R)) for a in range(ndim)]
    acc = [np.zeros((len(fg), R), f32) for _ in range(ndim)]
    val = np.broadcast_to(value[fg][:, None], (len(fg), R))
    done = np.zeros((len(fg), R), bool)
    res = np.zeros((len(fg), R), f32)
    while not done.all():
        acc = [(a + b).astype(f32) for a, b in zip(acc, d)]
        idx = [np.rint((p + a).astype(f32)).astype(np.int64) for p, a in zip(pos, acc)]
        oob = np.zeros_like(done)
        for a in range(ndim):
            oob |= (idx[a] < 0) | (idx[a] >= lbl16.shape[a])
        clipped = tuple(np.clip(i, 0, s - 1) for i, s in zip(idx, lbl16.shape))
        stop = ~done & (oob | (lbl16[clipped] != val))
        if stop.any():
            res[stop] = step_exit([a[stop] for a in acc], [b[stop] for b in d])
            done |= stop
    out[fg] = res
    return out


def _exit_2d(acc, d):
    x, y = acc                      # axis 0 offset is the kernel's x (paired with dx = row 1), axis 1 its y (dy = row 0)
    dx, dy = d
    t1 = (f32(0.5) / np.maximum(np.abs(dx), np.abs(dy)).astype(f32)).astype(f32) - f32(1)
    x = (x + (t1 * dx).astype(f32)).astype(f32)
    y = (y + (t1 * dy).astype(f32)).astype(f32)
    return np.sqrt(((x * x).astype(f32) + (y * y).astype(f32)).astype(f32)).astype(f32)


def _exit_3d(acc, d):
    r = [np.rint(a).astype(np.int64) for a in acc]
    return np.sqrt((r[0] * r[0] + r[1] * r[1] + r[2] * r[2]).astype(np.float64)).astype(f32)


def _starts(shape, grid):
    out_shape = tuple((s - 1) // g + 1 for s, g in zip(shape, grid))
    idx = np.indices(out_shape).reshape(len(shape), -1).T
    return out_shape, idx * np.asarray(grid)


def star_dist_2d(lbl, table, grid=(1, 1)):
    """table float32 [2, R] = (dy, dx) as direction_table_2d returns it"""
    lbl16 = np.asarray(lbl).astype(np.uint16)
    out_shape, starts = _starts(lbl16.shape, grid)
    dirs = np.stack([table[1], table[0]]).astype(f32)       # per array axis: (row step dx, column step dy)
    return _walk(lbl16, starts, dirs, _exit_2d).reshape(out_shape + (table.shape[1],))


def star_dist_3d(lbl, table, grid=(1, 1, 1)):
    """table float32 [3, R] = (dz, dy, dx)"""
    lbl16 = np.asarray(lbl).astype(np.uint16)
    out_shape, starts = _starts(lbl16.shape, grid)
    return _walk(lbl16, starts, np.asarray(table, f32), _exit_3d).reshape(out_shape + (table.shape[1],))
