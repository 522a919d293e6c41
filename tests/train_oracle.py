"""float64 restatements for the training tests (test infrastructure only): the U-Net walk of
stardist_b200.models.weights.unet_layers with autograd through every parameter, the StarDist loss (stardist/models/base.py
:34-50 and :315-325 with Keras' SUM_OVER_BATCH_SIZE reduction; TF cannot be installed here, so this is unpinned against
TF), and Adam as float32 numpy with the operation order of the device kernel."""
import numpy as np
import torch
import torch.nn.functional as F

EPS = float(np.float32(1e-7))                      # Keras' backend epsilon, a float32 value
ONE_M_EPS = float(np.float32(1) - np.float32(1e-7))


def params64(weights, names):
    """name -> (kernel (Cout, Cin, k...), bias) float64 leaf tensors that require grad"""
    out = {}
    for n in names:
        k, b = weights[n]
        nd = k.ndim - 2
        kt = torch.from_numpy(np.asarray(k, np.float64)).permute(nd + 1, nd, *range(nd)).contiguous().requires_grad_(True)
        out[n] = (kt, torch.from_numpy(np.asarray(b, np.float64)).clone().requires_grad_(True))
    return out


def grads_keras(params):
    """the .grad of params64 back in Keras layout (k..., Cin, Cout)"""
    out = {}
    for n, (k, b) in params.items():
        nd = k.dim() - 2
        out[n] = (k.grad.permute(*range(2, nd + 2), 1, 0).numpy(), b.grad.numpy())
    return out


def forward64(config, P, x):
    """x float64 tensor [N, *sp, C] -> (prob [N, *sp'], dist [N, *sp', R]) channels-last, differentiable in P"""
    from stardist_b200.models.weights import unet_layers
    nd = config.n_dim
    conv = F.conv2d if nd == 2 else F.conv3d
    maxpool = F.max_pool2d if nd == 2 else F.max_pool3d
    t = x.permute(0, nd + 1, *range(1, nd + 1))
    skips = {}
    for l in unet_layers(config):
        if l['kind'] == 'conv':
            t = conv(t, P[l['name']][0], P[l['name']][1], padding='same')
            if l['act'] == 'relu':
                t = F.relu(t)
        elif l['kind'] == 'pool':
            if 'save_skip' in l:
                skips[l['save_skip']] = t
            t = maxpool(t, tuple(l['pool']))
        elif l['kind'] == 'up':
            t = F.interpolate(t, scale_factor=tuple(float(p) for p in l['pool']), mode='nearest')
            t = torch.cat([t, skips.pop(l['skip'])], dim=1)
        elif l['kind'] == 'head':
            break
    prob = torch.sigmoid(conv(t, *P['prob']))[:, 0]
    dist = conv(t, *P['dist']).permute(0, *range(2, nd + 2), 1)
    return prob, dist


def loss64(prob, dist, prob_t, dam, dist_loss='mae', lam=0.0, weights=(1.0, 0.2)):
    """(loss, prob_loss, dist_loss) float64 tensors; prob: sigmoid output [...], dist [..., R], prob_t [...], dam [..., R+1]"""
    prob_t = prob_t.reshape(prob.shape)
    R = dist.shape[-1]
    dam = dam.reshape(dist.shape[:-1] + (R + 1,))
    sel = prob_t >= 0
    t, y = prob_t[sel], prob[sel]
    c = torch.clamp(y, EPS, ONE_M_EPS)
    lp = -(t * torch.log(c + EPS) + (1 - t) * torch.log(1 - c + EPS)).mean()
    pen = torch.abs if dist_loss == 'mae' else torch.square
    d_t, m = dam[..., :R], dam[..., R:]
    per_pix = (m * pen(d_t - dist)).mean(dim=-1) / (m.mean() + EPS)
    if lam > 0:
        per_pix = per_pix + lam * ((1 - m) * pen(dist)).mean(dim=-1)
    ld = per_pix.mean()
    return weights[0] * lp + weights[1] * ld, lp, ld


def adam_np(w, g, m, v, lr, coef_t, b1=0.9, b2=0.999, eps=1e-7):
    """one float32 Adam update in the device kernel's operation order; returns (w, m, v)"""
    f = np.float32
    one = f(1)
    alpha = f(lr) * f(coef_t)
    m = m + (g - m) * (one - f(b1))
    v = v + (g * g - v) * (one - f(b2))
    w = w - (m * alpha) / (np.sqrt(v) + f(eps))
    return w.astype(np.float32), m.astype(np.float32), v.astype(np.float32)
