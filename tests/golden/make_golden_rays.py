"""Golden vectors for explicit ray batches (kpn_render_rays / KeypointNeRF.render_rays), from the UNMODIFIED reference on CPU.

The reference renders only pixel lattices; its eval branch (src/model.py:1038-1096) is written out below for given rays, calling
the reference's own ray_bbox_intersection, query, rgba2out and importance_sample.  Same harness and file format as
make_golden.py, whose functions this reuses.  The fixtures hold the rays (origins, dirs, near_far before the bounding-box clip)
next to the reference's outputs and intermediates.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_rays.py              # every case below
    python tests/golden/make_golden_rays.py rays_ortho   # only the named cases
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402

syn = G.syn

# rays_ortho: an orthographic bundle (one direction, origins on a plane 3 units in front of the box centre; rows past the box
#   miss it; every 7th ray starts inside the box), 3 views / 18 keypoints, coarse + fine.
# rays_mixed: the lattices of two pinhole cameras, shuffled into one batch, each ray's near/far moved off the cameras' planes,
#   4 views / 17 keypoints, holed silhouette masks, coarse + fine.
RAY_CASES = {
    "rays_ortho": dict(kind="ortho", n_views=3, n_kpt=18, src_size=64, scene_seed=2, w_seed=26, fg_mode="hull", fg_hole=False,
                       grid=24, azimuth=1.0, S_c=16, S_f=16, fine=True, ray_seed=0),
    "rays_mixed": dict(kind="mixed", n_views=4, n_kpt=17, src_size=64, scene_seed=2, w_seed=26, fg_mode="hull", fg_hole=True,
                       tgt_size=24, zoom=2.0, azimuths=[0.7, 2.9], S_c=16, S_f=16, fine=True, ray_seed=1),
}


def make_rays(c, scene):
    """(origins, dirs, near_far) float32 of a case, from its seed."""
    rng = np.random.default_rng(c["ray_seed"])
    if c["kind"] == "ortho":
        b = scene["bounds"].reshape(2, 3).astype(np.float64)
        ctr, half = b.mean(0), 0.5 * (b[1] - b[0])
        a = c["azimuth"]
        d = np.array([np.cos(a), 0.1, np.sin(a)])
        d /= np.linalg.norm(d)
        u = np.cross(d, [0.0, 1.0, 0.0])
        u /= np.linalg.norm(u)
        v = np.cross(u, d)
        s = np.linspace(-1.3, 1.3, c["grid"]) * float(half.max())
        ss, tt = np.meshgrid(s, s, indexing="ij")
        ss, tt = ss.reshape(-1), tt.reshape(-1)
        back = np.where(np.arange(ss.size) % 7 == 3, 0.05, 3.0)   # 0.05: the origin lies inside the box (when the ray meets it)
        o = ctr[None] - back[:, None] * d[None] + ss[:, None] * u[None] + tt[:, None] * v[None]
        dirs = np.broadcast_to(d, o.shape)
        nf = np.stack([np.zeros(ss.size), np.full(ss.size, 5.0)], -1)
        return o.astype(np.float32), np.ascontiguousarray(dirs, dtype=np.float32), nf.astype(np.float32)
    os_, ds, nfs = [], [], []
    for az in c["azimuths"]:
        t = syn.make_target(size=c["tgt_size"], azimuth=az, zoom=c["zoom"])
        # the reference's pinhole rays (src/model.py:1019-1036) in torch fp32
        n = c["tgt_size"]
        y, x = torch.meshgrid(torch.arange(0, n), torch.arange(0, n), indexing="ij")
        g = torch.stack([x, y], -1).view(-1, 2).float()
        gh = torch.cat([g, torch.ones_like(g[:, :1])], -1)[None]
        K, RT = torch.from_numpy(t["K"]), torch.from_numpy(t["RT"])
        inv_K = torch.inverse(K[:, :3, :3]).transpose(1, 2)
        zn = torch.norm(torch.bmm(t["znear"] * gh, inv_K), p=2, dim=-1, keepdim=True)
        zf = torch.norm(torch.bmm(t["zfar"] * gh, inv_K), p=2, dim=-1, keepdim=True)
        d = torch.nn.functional.normalize(torch.bmm(torch.bmm(gh, inv_K), RT[:, :3, :3]), p=2, dim=-1)[0]
        o = (-torch.bmm(RT[:, :3, 3][:, None], RT[:, :3, :3]))[0].expand(d.shape[0], -1)
        # near/far off the cameras' planes: near 0.8-1.1 x, far 1.0-1.3 x (the far end stays behind the box)
        f = torch.from_numpy(np.stack([rng.uniform(0.8, 1.1, d.shape[0]), rng.uniform(1.0, 1.3, d.shape[0])], -1).astype(np.float32))
        os_.append(o); ds.append(d); nfs.append(torch.cat([zn[0], zf[0]], -1) * f)
    perm = rng.permutation(sum(x.shape[0] for x in ds))
    return tuple(np.ascontiguousarray(torch.cat(x, 0).numpy()[perm]) for x in (os_, ds, nfs))


def run_rays(M, net, scene, o, d, nf, S_c, S_f, fine):
    """The eval branch of batch_render_pifu_nerf (src/model.py:978-997, 1038-1096) on the given rays, batch size 1."""
    dummy = syn.make_target(size=8)
    cam, _, sp_data, feat_geo, feat_tex, img, fg, bounds = G.ref_inputs(scene, dummy)
    objcenter = torch.from_numpy(scene["kpt3d"][:, 0, :])
    n_views = scene["n_views"]

    def eval_func(v, view, n_pts_samples):
        rgba, mask = net.query(v, cam, feat_geo, feat_tex, n_views=n_views, view=view, nerf=True, sp_data=dict(sp_data),
                               tx_data={"img": img}, bbox_center=objcenter, n_pts_samples=n_pts_samples, src_foreground_mask=fg)
        mask = mask.float()
        sdf = mask * rgba[..., :1] + (1.0 - mask) * (0.1 / cam["nml_scale"])
        alpha = mask * torch.relu(rgba[..., 1:2])
        return torch.cat([alpha, sdf, rgba[..., 2:]], -1)

    out = {}
    with torch.no_grad():
        cam_pos = torch.from_numpy(o)[None]     # (1, n, 3): one origin per ray
        cam_rays = torch.from_numpy(d)[None]
        znear_rays = torch.from_numpy(nf[:, :1])[None]
        zfar_rays = torch.from_numpy(nf[:, 1:2])[None]
        z1, z2, hit = M.KeypointNeRF.ray_bbox_intersection(bounds, cam_pos, cam_rays)
        mask_z1 = (hit & (z1 > znear_rays)).float()
        znear_rays = mask_z1 * z1 + (1.0 - mask_z1) * znear_rays
        mask_z2 = (hit & (z2 < zfar_rays)).float()
        zfar_rays = mask_z2 * z2 + (1.0 - mask_z2) * zfar_rays
        z = torch.linspace(0.0, 1.0, steps=S_c)[None, None, :].expand(*znear_rays.shape[:2], -1)
        z = znear_rays + (zfar_rays - znear_rays) * z
        pts = (cam_pos[:, :, None] + cam_rays[:, :, None] * z[..., None]).view(1, -1, 3)
        view = cam_rays[:, :, None, :].expand(-1, -1, S_c, -1).reshape(1, -1, 3)
        rgba = eval_func(pts, view, S_c).view(1, -1, S_c, 5)
        color, depth, alpha, contrib, _ = M.KeypointNeRF.rgba2out(rgba, z)
        out.update(tex_fg=color[0].t(), depth=depth[0], alpha=alpha[0], contrib_coarse=contrib[0], z_coarse=z[0])
        if fine:
            z_mid = 0.5 * (z[..., 1:] + z[..., :-1])
            z_fine = M.KeypointNeRF.importance_sample(contrib[..., 1:-1], z_mid, S_f, uniform=True)
            z_fine = torch.sort(torch.cat([z, z_fine], -1), -1)[0]
            pts = (cam_pos[:, :, None] + cam_rays[:, :, None] * z_fine[..., None]).view(1, -1, 3)
            view = cam_rays[:, :, None, :].expand(-1, -1, z_fine.shape[-1], -1).reshape(1, -1, 3)
            rgba_f = eval_func(pts, view, S_f).view(*z_fine.shape, 5)
            color_f, depth_f, alpha_f, _, sdf = M.KeypointNeRF.rgba2out(rgba_f, z_fine)
            out.update(tex_fg_fine=color_f[0].t(), depth_fine=depth_f[0], alpha_fine=alpha_f[0], sdf=sdf[0], z_fine=z_fine[0])
        out["hit"] = hit[0, :, 0]
    return {k: np.ascontiguousarray(v.numpy()) for k, v in out.items()}


def scene_of(c):
    scene = syn.make_scene(src_size=c["src_size"], n_views=c["n_views"], n_kpt=c["n_kpt"], seed=c["scene_seed"], fg_mode=c["fg_mode"],
                           fg_hole=c["fg_hole"])
    return scene, syn.make_weights(c["n_kpt"], seed=c["w_seed"])


def main():
    M = G.import_reference()
    torch.set_num_threads(8)
    for name in sys.argv[1:] or list(RAY_CASES):
        c = RAY_CASES[name]
        scene, weights = scene_of(c)
        o, d, nf = make_rays(c, scene)
        res = run_rays(M, G.build_net(M, c["n_kpt"], weights), scene, o, d, nf, c["S_c"], c["S_f"], c["fine"])
        res.update(rays_o=o, rays_d=d, near_far=nf)
        res["input_sha256"] = np.frombuffer(G.checksum(scene, weights).encode(), dtype=np.uint8)
        res["meta"] = np.frombuffer(json.dumps(c).encode(), dtype=np.uint8)
        G.save_golden(name, res, G.HERE)
        print(name, o.shape[0], "rays, hit", int(res["hit"].sum()), "alpha mean", float(res["alpha"].mean()), "alpha max",
              float(res["alpha"].max()), flush=True)


if __name__ == "__main__":
    main()
