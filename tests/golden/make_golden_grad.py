"""Golden gradients of the eval branch of batch_render_pifu_nerf, from the UNMODIFIED reference on CPU with autograd.

The reference's batch_render_pifu_nerf (src/model.py:942-1108, uniform=True, net.eval()) renders a 12 x 12 lattice (level 1) with
autograd on; the loss is a seeded linear combination of every output of both passes.  The fixture holds the gradient of every
hot-path parameter (``g/<state_dict name>``) and of the three feature maps (``g/feat64``, ``g/feat8``, ``g/feat_tex``), the loss
weights (``G/<output>``, laid out like kpn_out's planes: (3, n) / (n,)), the lattice's rays as the reference builds them
(src/model.py:1026-1036; origins, unit directions, near/far before the bounding-box clip), the fine depths it resampled (under
torch.no_grad, src/model.py:1118) and its outputs.  Same harness and file format as make_golden.py.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_grad.py              # every case below
    python tests/golden/make_golden_grad.py grad_v3_k18  # only the named cases
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402

syn = G.syn

OUT_KEYS = ["tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf"]
MAPS = ("feat64", "feat8", "feat_tex")

# grad_v3_k18: 3 views, 18 keypoints, 64^2 hull-mask sources, 12 x 12 rays, 16 + 16 samples.
# grad_v4_k17: 4 views, 17 keypoints, 64 x 48 hull-mask sources with holes, 12 x 12 rays, 16 + 16 samples.
GRAD_CASES = {
    "grad_v3_k18": dict(n_views=3, n_kpt=18, src_size=64, scene_seed=2, w_seed=26, fg_mode="hull", fg_hole=False, tgt_size=12,
                        azimuth=1.0, zoom=2.0, S_c=16, S_f=16, loss_seed=11),
    "grad_v4_k17": dict(n_views=4, n_kpt=17, src_size=64, src_height=48, scene_seed=2, w_seed=26, fg_mode="hull", fg_hole=True,
                        tgt_size=12, azimuth=2.5, zoom=2.0, S_c=16, S_f=16, loss_seed=12),
}


def lattice_rays(target):
    """The rays batch_render_pifu_nerf builds for a level-1 lattice (src/model.py:1019-1036), in the same torch fp32 ops."""
    n = target["width"]
    y, x = torch.meshgrid(torch.arange(0, target["height"]), torch.arange(0, n), indexing="ij")
    g = torch.stack([x, y], -1).view(-1, 2).float()[None]
    gh = torch.cat([g, torch.ones_like(g[..., :1])], -1)
    K, RT = torch.from_numpy(target["K"]), torch.from_numpy(target["RT"])
    inv_K = torch.inverse(K[:, :3, :3]).transpose(1, 2)
    zn = torch.norm(torch.bmm(target["znear"] * gh, inv_K), p=2, dim=-1, keepdim=True)
    zf = torch.norm(torch.bmm(target["zfar"] * gh, inv_K), p=2, dim=-1, keepdim=True)
    d = torch.nn.functional.normalize(torch.bmm(torch.bmm(gh, inv_K), RT[:, :3, :3]), p=2, dim=-1)[0]
    o = (-torch.bmm(RT[:, :3, 3][:, None], RT[:, :3, :3]))[0].expand(d.shape[0], -1)
    return tuple(np.ascontiguousarray(t.numpy()) for t in (o, d, torch.cat([zn[0], zf[0]], -1)))


def run_grad(M, net, scene, target, c):
    cam, cam_tar, sp_data, feat_geo, feat_tex, img, fg, bounds = G.ref_inputs(scene, target)
    leaves = {"feat64": feat_geo[0].clone().requires_grad_(), "feat8": feat_geo[1].clone().requires_grad_(),
              "feat_tex": feat_tex.clone().requires_grad_()}
    zs = []
    orig_r2o = M.KeypointNeRF.rgba2out

    def r2o(rgba, z):
        zs.append(z.detach().clone())
        return orig_r2o(rgba, z)

    M.KeypointNeRF.rgba2out = staticmethod(r2o)
    try:
        out = M.KeypointNeRF.batch_render_pifu_nerf(
            net, img, cam, scene["n_views"], cam_tar, level=1, stride=0, feat_geo=[leaves["feat64"], leaves["feat8"]],
            feat_tex=leaves["feat_tex"], sp_data=dict(sp_data), objcenter=torch.from_numpy(scene["kpt3d"][:, 0, :]),
            sample_per_ray_c=c["S_c"], sample_per_ray_f=c["S_f"], fine=True, uniform=True, bounds=bounds, src_foreground_mask=fg)
    finally:
        M.KeypointNeRF.rgba2out = orig_r2o
    n = target["width"] * target["height"]
    flat = {k: (out[k][0].reshape(3, n) if k.startswith("tex_fg") else out[k][0].reshape(n)) for k in OUT_KEYS}
    rng = np.random.default_rng(c["loss_seed"])
    Gw = {k: rng.standard_normal(tuple(flat[k].shape)).astype(np.float32) for k in OUT_KEYS}
    loss = sum((flat[k] * torch.from_numpy(Gw[k])).sum() for k in OUT_KEYS)
    loss.backward()
    res = {f"G/{k}": v for k, v in Gw.items()}
    res.update({k: np.ascontiguousarray(v.detach().numpy()) for k, v in flat.items()})
    for name, p in net.named_parameters():
        if name.startswith(("mlp_geo.", "mlp_tex.", "ibr_compress_gfeat.")):
            res["g/" + name] = np.ascontiguousarray(p.grad.numpy())
    for k, t in leaves.items():
        res["g/" + k] = np.ascontiguousarray(t.grad.numpy())
    res["z_fine"] = np.ascontiguousarray(zs[1][0].numpy())
    return res


def main():
    M = G.import_reference()
    torch.set_num_threads(8)
    for name in sys.argv[1:] or list(GRAD_CASES):
        c = GRAD_CASES[name]
        scene = syn.make_scene(src_size=c["src_size"], n_views=c["n_views"], n_kpt=c["n_kpt"], seed=c["scene_seed"], fg_mode=c["fg_mode"],
                               fg_hole=c["fg_hole"], src_height=c.get("src_height"))
        weights = syn.make_weights(c["n_kpt"], seed=c["w_seed"])
        target = syn.make_target(size=c["tgt_size"], azimuth=c["azimuth"], zoom=c["zoom"])
        net = G.build_net(M, c["n_kpt"], weights)
        res = run_grad(M, net, scene, target, c)
        o, d, nf = lattice_rays(target)
        res.update(rays_o=o, rays_d=d, near_far=nf)
        res["input_sha256"] = np.frombuffer(G.checksum(scene, weights).encode(), dtype=np.uint8)
        res["meta"] = np.frombuffer(json.dumps(c).encode(), dtype=np.uint8)
        G.save_golden(name, res, G.HERE)
        print(name, "alpha max", float(res["alpha"].max()), "alpha_fine max", float(res["alpha_fine"].max()),
              "|g feat64| max", float(np.abs(res["g/feat64"]).max()), flush=True)


if __name__ == "__main__":
    main()
