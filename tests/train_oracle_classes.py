"""float64 restatements of the multi-class branch for the training tests (test infrastructure only): the U-Net walk of
train_oracle.forward64 with the class branch (features_class, prob_class softmax) added, the weighted categorical
cross-entropy of stardist/models/base.py:108-126 with Keras' SUM_OVER_BATCH_SIZE reduction (unpinned against TF, like
train_oracle.loss64), and the softmax backward."""
import numpy as np
import torch
import torch.nn.functional as F

from train_oracle import EPS, ONE_M_EPS


def forward64_classes(config, P, x):
    """forward64 plus the class branch (model2d.py:338-347, model3d.py:388-396): (prob, dist, prob_class [N, *sp', C]) with
    prob_class the softmax output, channels last, differentiable in P"""
    from stardist_b200.models.weights import unet_layers
    nd = config.n_dim
    conv = F.conv2d if nd == 2 else F.conv3d
    maxpool = F.max_pool2d if nd == 2 else F.max_pool3d
    t = x.permute(0, nd + 1, *range(1, nd + 1))
    skips, base = {}, None
    for l in unet_layers(config):
        if l['kind'] == 'conv':
            if l['name'] == 'features':
                base = t
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
    base = t if base is None else base
    prob = torch.sigmoid(conv(t, *P['prob']))[:, 0]
    dist = conv(t, *P['dist']).permute(0, *range(2, nd + 2), 1)
    c = base
    if 'features_class' in P:
        c = conv(base, *P['features_class'], padding='same')
        if config.unet_activation == 'relu':
            c = F.relu(c)
    prob_class = torch.softmax(conv(c, *P['prob_class']), dim=1).permute(0, *range(2, nd + 2), 1)
    return prob, dist, prob_class


def class_loss64(s, t, class_weights):
    """weighted categorical cross-entropy (stardist/models/base.py:108-126) averaged over every pixel, ignored ones included
    (Keras' SUM_OVER_BATCH_SIZE): s the softmax output [..., C], t the prob_class target [..., C] (< 0: ignored)"""
    t = t.reshape(s.shape)
    w = torch.as_tensor(np.asarray(class_weights, np.float64)).to(s)
    q = s / (s + EPS).sum(dim=-1, keepdim=True)
    c = torch.clamp(q, EPS, ONE_M_EPS)
    mask = (t >= 0).to(s.dtype)
    return (-(w * mask * t * torch.log(c)).sum(dim=-1)).mean()


def softmax_backward64(s, ds):
    """dL/dz of z -> s = softmax(z) from dL/ds, both [..., C]"""
    return s * (ds - (s * ds).sum(dim=-1, keepdim=True))
