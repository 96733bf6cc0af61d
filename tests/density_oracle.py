"""The trunk alone at arbitrary points, restated on the oracle's encoding (oracle/sparf_oracle.py): the checker of the
density queries (NeRF.compute_raw_density).  TEST INFRASTRUCTURE ONLY.

The op sequence is that of oracle.sparf_oracle.mlp_forward up to the raw density, so that mlp_forward's density is the
softplus of raw_density's raw bit for bit (tests/test_density_cpu.py checks it); tests/golden/density_raw.npz pins it
against the reference's own compute_raw_density.
"""
from typing import Dict, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import sparf_oracle as O


def raw_density(params: Dict[str, torch.Tensor], pts: torch.Tensor, *, L_3D: int = 10, skip: Sequence[int] = (4,),
                barf_c2f=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """pts [...,3] -> (raw density [...] before the softplus, relu(features) [...,256]).

    frequency_nerf.py:149-170 (compute_raw_density): trunk with the encoded input re-concatenated
    AFTER the features at the skip layer; the last trunk layer emits (raw_sigma | 256 features)."""
    dt = pts.dtype
    m3 = O.c2f_weights(L_3D, float(params["progress"]), barf_c2f, pts.device, dt)
    enc = torch.cat([pts, O.posenc(pts, L_3D, m3)], dim=-1)
    n_feat = len([k for k in params if k.startswith("mlp_feat.") and k.endswith(".weight")])
    h = enc
    for li in range(n_feat):
        if li in skip:
            h = torch.cat([h, enc], dim=-1)
        h = F.linear(h, params["mlp_feat.%d.weight" % li].to(dt), params["mlp_feat.%d.bias" % li].to(dt))
        if li == n_feat - 1:
            raw, h = h[..., 0], h[..., 1:]
        h = F.relu(h)
    return raw, h
