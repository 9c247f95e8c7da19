"""CPU oracle of the eval branch of ``batch_render_pifu_nerf`` on explicit rays (reference ``src/model.py:1038-1096``).  TEST
INFRASTRUCTURE ONLY.

Built from ``oracle/kpnerf_oracle.py``'s own stages (``ray_bbox``, ``clip_near_far``, ``coarse_z``, ``eval_func``, ``composite``,
``importance_sample``) in the order its ``render_pixels`` runs them after ``ray_setup``, with each ray's own origin in place of the
lattice's shared camera centre; ``tests/test_rays_cpu.py`` checks that both give the same bits on lattice rays.
"""
from __future__ import annotations

import torch

from oracle import kpnerf_oracle as O

T = torch.Tensor


def render_rays(scene: dict, fw: dict, o: T, d: T, near_far: T, S_c: int, S_f: int = 0, fine: bool = False, sp=None,
                z_fine_override: T | None = None, disable_fg_mask: bool = False) -> dict:
    """Origins ``o`` (R,3), unit directions ``d`` (R,3), ``near_far`` (R,2) before the bounding-box clip.  Returns the flat
    per-ray outputs of ``O.render_pixels``."""
    o, d, near_far = O._t(o), O._t(d), O._t(near_far)
    near, far, hit = O.ray_bbox(scene["bounds"], o, d)
    n_r, f_r = O.clip_near_far(near_far[:, :1], near_far[:, 1:2], near, far, hit)
    z = O.coarse_z(n_r, f_r, S_c)
    R = d.shape[0]

    def shade(zz):
        S = zz.shape[1]
        pts = (o[:, None] + d[:, None] * zz[..., None]).reshape(-1, 3)
        view = d[:, None].expand(-1, S, -1).reshape(-1, 3)
        return O.eval_func(scene, fw, pts, view, sp, disable_fg_mask=disable_fg_mask).reshape(R, S, 5)

    rgba = shade(z)
    color, depth, acc, contrib, _ = O.composite(rgba, z)
    out = {"tex_fg": color, "depth": depth, "alpha": acc, "contrib": contrib, "z": z,
           "near": n_r, "far": f_r, "hit": hit, "rgba": rgba}
    if fine:
        z_mid = 0.5 * (z[:, 1:] + z[:, :-1])
        z_f = O.importance_sample(contrib[:, 1:-1], z_mid, S_f)
        z_all = torch.sort(torch.cat([z, z_f], -1), -1).values
        if z_fine_override is not None:
            z_all = O._t(z_fine_override)
        rgba_f = shade(z_all)
        color_f, depth_f, acc_f, contrib_f, sdf_f = O.composite(rgba_f, z_all)
        out.update({"tex_fg_fine": color_f, "depth_fine": depth_f, "alpha_fine": acc_f,
                    "sdf": sdf_f, "z_fine": z_all, "rgba_fine": rgba_f})
    return out
