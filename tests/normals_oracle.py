"""fp64 checkers of the normal maps (sparf_b200/normals.py).  TEST INFRASTRUCTURE ONLY.

point_gradient: d raw / d x of the trunk (density_oracle.raw_density's op sequence) by a hand-written NumPy backward.
normal_map: the whole chain of one pass in fp64: x = o + d t, sigma = softplus(raw), the oracle's composite weights,
normals -g / |g| (0 where g = 0) and their weight-sum per ray.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import sparf_oracle as O


def _c2f(L, progress, barf_c2f):
    m = O.c2f_weights(L, float(progress), barf_c2f, dtype=torch.float64)
    return np.ones(L) if m is None else m.numpy()


def point_gradient(params, x, *, L=10, skip=(4,), progress=1.0, barf_c2f=None):
    """params: {mlp_feat.i.weight / .bias}, x [M, 3] -> d raw / d x [M, 3], all in NumPy fp64"""
    x = np.asarray(x, np.float64)
    n = len([k for k in params if k.startswith("mlp_feat.") and k.endswith(".weight")])
    Ws = [np.asarray(params["mlp_feat.%d.weight" % i], np.float64) for i in range(n)]
    bs = [np.asarray(params["mlp_feat.%d.bias" % i], np.float64) for i in range(n)]
    m = _c2f(L, progress, barf_c2f)
    f = 2.0 ** np.arange(L) * float(np.float32(math.pi))
    arg = x[:, :, None] * f                                              # [M, 3, L]
    enc = np.concatenate([x, np.stack([np.sin(arg) * m, np.cos(arg) * m], -2).reshape(len(x), -1)], 1)
    h, ins, pre = enc, [], []
    for li in range(n):
        if li in skip:
            h = np.concatenate([h, enc], 1)
        ins.append(h.shape[1])
        z = h @ Ws[li].T + bs[li]
        pre.append(z)
        h = np.maximum(z[:, 1:] if li == n - 1 else z, 0)
    g_z = np.zeros_like(pre[-1])
    g_z[:, 0] = 1.0                                                      # d raw / d z_last
    g_enc = np.zeros_like(enc)
    for li in range(n - 1, -1, -1):
        g_in = g_z @ Ws[li]
        if li in skip or li == 0:
            E = enc.shape[1]
            g_enc += g_in[:, -E:]
            g_in = g_in[:, :-E]
        if li > 0:
            g_z = g_in * (pre[li - 1] > 0)
    g_s = g_enc[:, 3:].reshape(len(x), 3, 2, L)
    return g_enc[:, :3] + ((g_s[:, :, 0] * np.cos(arg) - g_s[:, :, 1] * np.sin(arg)) * m * f).sum(-1)


def unit(g):
    norm = np.linalg.norm(g, axis=-1, keepdims=True)
    return np.where(norm > 0, -g / np.where(norm > 0, norm, 1), 0.0)


def normal_map(params, center, ray, t, *, progress=1.0, barf_c2f=None):
    """center, ray [R, 3], t [R, S] -> (normal [R, 3], weights [R, S]) in fp64"""
    from density_oracle import raw_density
    o, d, t = (torch.as_tensor(np.asarray(a), dtype=torch.float64) for a in (center, ray, t))
    x = o[:, None, :] + d[:, None, :] * t[..., None]
    p = {k: torch.as_tensor(np.asarray(v), dtype=torch.float64) for k, v in params.items() if k.startswith("mlp_feat.")}
    p["progress"] = torch.tensor(float(progress))
    raw, _ = raw_density(p, x, barf_c2f=barf_c2f)
    sigma = F.softplus(raw)
    w = O.composite(d[None], sigma[None], torch.zeros(*sigma.shape, 3, dtype=torch.float64)[None], t[None])["weights"]
    w = w[0, ..., 0].numpy()
    n = unit(point_gradient(p, x.reshape(-1, 3).numpy(), progress=progress, barf_c2f=barf_c2f)).reshape(*t.shape, 3)
    return (w[..., None] * n).sum(1), w
