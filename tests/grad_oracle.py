"""Gradients of the oracle's eval branch on explicit rays by torch autograd, and the gradient goldens of
tests/golden/make_golden_grad.py.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np
import torch

from oracle import kpnerf_oracle as O
from tests import rays_oracle as RO
from tests.util import checksum, load_golden, scene_from_meta

MAPS = ("feat64", "feat8", "feat_tex")
OUT_KEYS = ["tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf"]
GRAD_CASES = ["grad_v3_k18", "grad_v4_k17"]


def oracle_grads(scene, weights, sp, rays, S_c, S_f, z_fine, G, dtype=torch.float64):
    """dL/d every weight (by state_dict name) and feature map (by scene key) of L = sum_k <out_k, G_k>, G_k in kpn_out's plane
    layout ((3, n) / (n,)), with the fine pass at the constant depths z_fine.  Also returns the outputs."""
    with O.precision(dtype):
        w = {k: torch.tensor(np.asarray(v), dtype=dtype, requires_grad=True) for k, v in weights.items()}
        sc = dict(scene)
        for k in MAPS:
            sc[k] = torch.tensor(scene[k], dtype=dtype, requires_grad=True)
        out = RO.render_rays(sc, O.fold_weights(w), *rays, S_c, S_f, True, sp, z_fine_override=torch.as_tensor(z_fine).to(dtype))
        G = {k: torch.as_tensor(v) for k, v in G.items()}
        loss = sum((out[k] * (G[k].t() if k.startswith("tex_fg") else G[k]).to(dtype)).sum() for k in G)
        loss.backward()
    return {k: v.grad for k, v in w.items()}, {k: sc[k].grad for k in MAPS}, out


def load_grad_case(name):
    """(golden arrays, meta, scene, weights, rays (o, d, near_far) as torch fp32, loss weights G)."""
    g, meta, sha = load_golden(name)
    g = {k: np.array(v, copy=True, order="C") for k, v in g.items()}
    scene, weights, _ = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    rays = tuple(torch.from_numpy(g[k]) for k in ("rays_o", "rays_d", "near_far"))
    G = {k: torch.from_numpy(g["G/" + k]) for k in OUT_KEYS}
    return g, meta, scene, weights, rays, G


def rel_errors(got, ref):
    """(relative L2 error, largest absolute error / largest absolute reference value)."""
    got = torch.as_tensor(got).double().reshape(-1)
    ref = torch.as_tensor(ref).double().reshape(-1)
    nrm, mx = float(ref.norm()), float(ref.abs().max())
    return float((got - ref).norm()) / nrm, float((got - ref).abs().max()) / mx
