"""CPU oracle for the KeypointNeRF ray-march hot path.  TEST INFRASTRUCTURE ONLY.

This file is a from-scratch restatement (plain torch-CPU tensor arithmetic, no
``grid_sample``/``nn.Module``) of the algorithm the reference implements in
``/root/reference/src/model.py:690-1302``, ``src/spatial.py:63-118`` and
``src/utils.py:74-95,476-748``.  Each function cites the lines it follows.

Precision: fp32 by default, like the reference.  ``with precision(torch.float64): ...`` runs the
same arithmetic in fp64 (inputs, constants and intermediates), which gives a reference whose own
round-off is far below any kernel's, so that a kernel's error can be told apart from the fp32
oracle's.  The fp32 results do not depend on this switch existing.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may
import it; the product path (``keypointnerf_b200``) never does and has no CPU fallback.

Parity pin: the reference publishes no golden vectors or tests (SURVEY.md section 4), so
this oracle is pinned against outputs of the *reference itself*, run in the build
container by ``tests/golden/make_golden.py`` and frozen under ``tests/golden/*.npz``
(``tests/test_oracle_golden.py``).
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch

T = torch.Tensor

_DTYPE = torch.float32   # arithmetic type of every function below (see ``precision``)


@contextlib.contextmanager
def precision(dtype: torch.dtype):
    """Run the oracle in ``dtype`` (torch.float32 or torch.float64) inside the ``with`` block."""
    global _DTYPE
    assert dtype in (torch.float32, torch.float64)
    prev, _DTYPE = _DTYPE, dtype
    try:
        yield
    finally:
        _DTYPE = prev


def _t(x, dtype=None):
    dtype = _DTYPE if dtype is None else dtype
    if isinstance(x, torch.Tensor):
        return x.to(dtype)
    return torch.as_tensor(np.asarray(x)).to(dtype)


# --------------------------------------------------------------------------------------
# parameters
# --------------------------------------------------------------------------------------
def fold_weights(w: dict) -> dict:
    """Effective (W, b) per layer.  Weight-normed layers: W = g * v / ||v||_row
    (``torch.nn.utils.weight_norm`` dim=0, reference ``src/utils.py:542-543``)."""
    out = {}
    names = sorted({k.rsplit(".", 1)[0] for k in w if k != "mlp_tex.ani_al"})
    for n in names:
        if n + ".weight_v" in w:
            v = _t(w[n + ".weight_v"])
            g = _t(w[n + ".weight_g"])
            W = v * (g / v.norm(dim=1, keepdim=True))
        else:
            W = _t(w[n + ".weight"])
        out[n] = (W.contiguous(), _t(w[n + ".bias"]))
    out["ani_al"] = _t(w["mlp_tex.ani_al"]).reshape(())
    return out


def softplus100(x: T) -> T:
    """``Softplus(beta=100, threshold=20)`` (reference ``src/utils.py:523-524``)."""
    bx = 100.0 * x
    return torch.where(bx > 20.0, x, torch.log1p(torch.exp(torch.clamp(bx, max=20.0))) / 100.0)


def elu(x: T) -> T:
    return torch.where(x > 0, x, torch.expm1(torch.clamp(x, max=0.0)))


def lin(fw: dict, name: str, x: T) -> T:
    W, b = fw[name]
    return x @ W.t() + b


# --------------------------------------------------------------------------------------
# rays and depth samples
# --------------------------------------------------------------------------------------
def pixel_lattice(width: int, height: int, step: int, x_off: int, y_off: int) -> T:
    """Strided pixel lattice of one pass, row-major over (y, x) (reference ``src/model.py:1019-1024``)."""
    ys = torch.arange(0, height, step)
    xs = torch.arange(0, width, step)
    yy, xx = torch.meshgrid(ys, xs, indexing="ij")
    g = torch.stack([xx + x_off, yy + y_off], -1).reshape(-1, 2)
    return g.to(_DTYPE)


def ray_setup(pix: T, K_t: T, RT_t: T, znear: float, zfar: float):
    """Rays through pixels (reference ``src/model.py:1026-1036``).  ``pix`` (R,2) float."""
    pix = _t(pix)
    K3 = _t(K_t).reshape(-1, 4, 4)[0, :3, :3]
    RT = _t(RT_t).reshape(-1, 4, 4)[0]
    R, t = RT[:3, :3], RT[:3, 3]
    inv_K_T = torch.inverse(K3).t()
    gh = torch.cat([pix, torch.ones_like(pix[:, :1])], -1)
    d_c = gh @ inv_K_T
    n_r = ((znear * gh) @ inv_K_T).norm(dim=-1, keepdim=True)
    f_r = ((zfar * gh) @ inv_K_T).norm(dim=-1, keepdim=True)
    d = d_c @ R
    d = d / d.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    o = -(t[None] @ R)  # (1,3)
    return o, d, n_r, f_r


def ray_bbox(bounds: T, o: T, d: T):
    """Slab test with the reference's "exactly two face hits" rule (``src/model.py:1178-1237``)."""
    b = _t(bounds).reshape(2, 3) + torch.tensor([-0.01, 0.01], dtype=_DTYPE)[:, None]
    dd = d.clone()
    dd[dd.abs() < 1e-5] = 1e-5
    t6 = ((b[None] - o[:, None]) / dd[:, None]).reshape(-1, 6)  # order: min xyz, max xyz
    p = t6[..., None] * dd[:, None] + o[:, None]  # (R,6,3)
    lo, hi = b[0] - 1e-6, b[1] + 1e-6
    inside = ((p >= lo) & (p <= hi)).all(-1)  # (R,6)
    hit = inside.sum(-1) == 2
    dist = (p - o[:, None]).norm(dim=-1) / dd.norm(dim=-1, keepdim=True)  # (R,6)
    near = torch.where(inside, dist, torch.full_like(dist, float("inf"))).min(-1).values
    far = torch.where(inside, dist, torch.full_like(dist, -float("inf"))).max(-1).values
    near = torch.where(hit, near, torch.ones_like(near))
    far = torch.where(hit, far, torch.ones_like(far))
    return near[:, None], far[:, None], hit[:, None]


def clip_near_far(n_r: T, f_r: T, near: T, far: T, hit: T):
    """Reference ``src/model.py:1040-1043``."""
    n = torch.where(hit & (near > n_r), near, n_r)
    f = torch.where(hit & (far < f_r), far, f_r)
    return n, f


def coarse_z(n_r: T, f_r: T, S: int) -> T:
    """Uniform (eval, ``uniform=True``) depths (reference ``src/model.py:1045-1055``)."""
    lin01 = torch.linspace(0.0, 1.0, steps=S, dtype=_DTYPE)
    return n_r + (f_r - n_r) * lin01[None]


# --------------------------------------------------------------------------------------
# per-sample query
# --------------------------------------------------------------------------------------
def project(scene: dict, pts: T):
    """World points -> normalised source-view coordinates (reference ``src/model.py:713-723``).
    Returns xy (V,N,2) in [-1,1] (align_corners convention) and z (V,N,1)."""
    KRT = _t(scene["KRT"])
    pts = _t(pts)
    vh = torch.einsum("vij,nj->vni", KRT[:, :3, :3], pts) + KRT[:, None, :3, 3]
    zc = vh[..., 2:3]
    xy = vh[..., :2] / zc
    W, H = float(scene["width"]), float(scene["height"])
    x = 2.0 * (xy[..., 0] / (W - 1.0)) - 1.0
    y = 2.0 * (xy[..., 1] / (H - 1.0)) - 1.0
    zn, zf = float(scene["znear"]), float(scene["zfar"])
    z = 2.0 * (zc - zn) / (zf - zn) - 1.0
    return torch.stack([x, y], -1), z


def bilinear_border(fmap: T, xy: T) -> T:
    """``grid_sample(bilinear, padding_mode='border', align_corners=True)`` restated
    (reference ``src/utils.py:74-89``).  fmap (V,C,H,W), xy (V,N,2) -> (V,N,C)."""
    V, C, H, W = fmap.shape
    ix = ((xy[..., 0] + 1.0) * 0.5 * (W - 1)).clamp(0.0, float(W - 1))
    iy = ((xy[..., 1] + 1.0) * 0.5 * (H - 1)).clamp(0.0, float(H - 1))
    x0 = ix.floor()
    y0 = iy.floor()
    fx = ix - x0
    fy = iy - y0
    x0i = x0.long()
    y0i = y0.long()
    x1i = (x0i + 1).clamp(max=W - 1)  # weight is 0 whenever the clamp is active
    y1i = (y0i + 1).clamp(max=H - 1)
    flat = fmap.reshape(V, C, H * W)

    def tap(yi, xi):
        idx = (yi * W + xi)[:, None, :].expand(-1, C, -1)
        return torch.gather(flat, 2, idx)  # (V,C,N)

    out = (tap(y0i, x0i) * ((1 - fx) * (1 - fy))[:, None]
           + tap(y0i, x1i) * (fx * (1 - fy))[:, None]
           + tap(y1i, x0i) * ((1 - fx) * fy)[:, None]
           + tap(y1i, x1i) * (fx * fy)[:, None])
    return out.permute(0, 2, 1)


def validity(scene: dict, xy: T, z: T, disable_fg_mask: bool = False) -> T:
    """Sample valid iff inside every view's frustum and foreground in every view
    (reference ``src/model.py:725-739``).  Returns (N,) bool."""
    eps = 1e-2
    m = ((xy >= -1.0 - eps) & (xy <= 1.0 + eps)).all(-1) & (z[..., 0] >= -1.0)  # (V,N)
    ok = m.all(0)
    if not disable_fg_mask:
        fg = bilinear_border(_t(scene["fg"]), xy)[..., 0]  # (V,N)
        ok = ok & (fg > 0.1).all(0)
    return ok


def pixel_weight(xy: T, z: T, valid: T) -> T:
    """Boundary-smooth view weights (reference ``src/model.py:750-759``).  -> (V,N,1)."""
    xyz = 0.5 * torch.cat([xy, z], -1) + 0.5
    db = torch.minimum(xyz, 1.0 - xyz)
    s = torch.sigmoid(5.0 * (db / 0.1 - 1.0))
    pw = (s[..., 0] * s[..., 1] * s[..., 2])[..., None] * valid[None, :, None].to(s.dtype)
    return pw / (pw.sum(0, keepdim=True) + 1e-6)


def encode_rel_z_decay(scene: dict, pts: T, sp_level: int = 3, scale: float = 1.0, sigma: float = 0.1) -> T:
    """Relative spatial keypoint encoding, ``sp_type='rel_z_decay'``
    (reference ``src/spatial.py:76,81-85,110-118`` and ``position_embedding`` 23-47).
    Output (V,N,(1+2L)K) with layout [r*K+k], r = 0: dz, 1+2l: sin(pi 2^l dz), 2+2l: cos(pi 2^l dz)."""
    E = _t(scene["extrin"])
    kpt = _t(scene["kpt3d"]).reshape(-1, 3)
    pts = _t(pts)
    c = torch.einsum("vij,nj->vni", E[:, :3, :3], pts) + E[:, None, :3, 3]  # (V,N,3)
    ck = torch.einsum("vij,kj->vki", E[:, :3, :3], kpt) + E[:, None, :3, 3]  # (V,K,3)
    dz = scale * (c[:, :, None, 2] - ck[:, None, :, 2])  # (V,N,K)
    d2 = ((c[:, :, None, :] - ck[:, None, :, :]) ** 2).sum(-1)
    wk = torch.exp(-d2 / (2.0 * sigma ** 2))
    freqs = [np.float32(np.pi * (2 ** l)) if _DTYPE == torch.float32 else np.pi * (2 ** l) for l in range(sp_level)]
    # reference layout: cat(sin(y), cos(y)) along the keypoint axis then flattened:
    # [dz(K) | l0: sin(K) cos(K) | l1: sin cos | ...]  (src/spatial.py:35-39); sp_level 0 is the dz row alone (31-32)
    rows = [dz]
    for f in freqs:
        y = dz * float(f)  # (V,N,K)
        rows.append(torch.sin(y))
        rows.append(torch.cos(y))
    enc = torch.stack(rows, 2) * wk[:, :, None, :]  # (V,N,1+2L,K)
    return enc.reshape(enc.shape[0], enc.shape[1], -1)


def geo_mlp(fw: dict, enc: T, f64: T, f8: T):
    """Per-(sample,view) MLP-UNet with feature skips at layers 0 and 2
    (reference ``src/utils.py:691-720``; dims ``configs/zju.json:52-73``)."""
    p = "mlp_geo.layers1.layers."
    h = softplus100(lin(fw, p + "0.linear", torch.cat([enc, f64], -1)))
    h = softplus100(lin(fw, p + "1.linear", h))
    h = softplus100(lin(fw, p + "2.linear", torch.cat([h, f8], -1)))
    return lin(fw, p + "3.linear", h)  # (V,N,64)


def pool_mean_var(xv: T, pw: T) -> T:
    """Weighted mean || variance over views (reference ``src/utils.py:612-647,722-748``)."""
    mean = (pw * xv).sum(0)
    var = (pw * (xv - mean[None]) ** 2).sum(0)
    return torch.cat([mean, var], -1)  # (N,128)


def density_head(fw: dict, x_pool: T) -> T:
    """``layers2`` 128->64->64->2 (reference ``src/utils.py:577-587``)."""
    p = "mlp_geo.layers2.layers."
    h = softplus100(lin(fw, p + "0.linear", x_pool))
    h = softplus100(lin(fw, p + "1.linear", h))
    return lin(fw, p + "2.linear", h)  # (N,2) = [sdf_raw, rad]


def source_centres(scene: dict) -> T:
    """C_v = (KRT^-1)[:3,3] (reference ``src/model.py:822-824``)."""
    return torch.inverse(_t(scene["KRT"]))[:, :3, 3]


def ray_diff(scene: dict, pts: T, view: T) -> T:
    """[unit(dir - dir_src), dir . dir_src] per view (reference ``src/model.py:825-832``).  (V,N,4)"""
    C = source_centres(scene)
    pts, view = _t(pts), _t(view)
    r = pts[None] - C[:, None]
    r = r / r.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    diff = view[None] - r
    nrm = diff.norm(dim=-1, keepdim=True)
    dot = (r * view[None]).sum(-1, keepdim=True)
    return torch.cat([diff / nrm.clamp_min(1e-6), dot], -1)


def ibr_head(fw: dict, f: T, rd: T, mask: T, src_rgb: T) -> T:
    """IBRNet-style blending head (reference ``src/model.py:1267-1302``).
    f (V,N,35), rd (V,N,4), mask (V,N,1) float, src_rgb (V,N,3) -> (N,3)."""
    t = "mlp_tex."
    e = elu(lin(fw, t + "ray_encoder.2", elu(lin(fw, t + "ray_encoder.0", rd))))
    f = f + e
    dot = rd[..., 3:4]
    ex = torch.exp(fw["ani_al"].abs() * (dot - 1.0))
    w = (ex - ex.min(0, keepdim=True).values) * mask
    w = w / (w.sum(0, keepdim=True) + 1e-8)
    mean = (f * w).sum(0, keepdim=True)
    var = (w * (f - mean) ** 2).sum(0, keepdim=True)
    V = f.shape[0]
    x = torch.cat([mean.expand(V, -1, -1), var.expand(V, -1, -1), f], -1)
    x = elu(lin(fw, t + "base_layer.2", elu(lin(fw, t + "base_layer.0", x))))
    pv = elu(lin(fw, t + "vis_layer1.2", elu(lin(fw, t + "vis_layer1.0", x * w))))
    res, vis = pv[..., :32], pv[..., 32:33]
    x = x + res
    v2 = lin(fw, t + "vis_layer2.2", elu(lin(fw, t + "vis_layer2.0", x * torch.sigmoid(vis) * mask)))
    vis2 = torch.sigmoid(v2) * mask
    h = elu(lin(fw, t + "out_layer.0", torch.cat([x, vis2, rd], -1)))
    h = elu(lin(fw, t + "out_layer.2", h))
    logit = lin(fw, t + "out_layer.4", h)
    logit = torch.where(mask == 0, torch.full_like(logit, -1e9), logit)
    sm = torch.softmax(logit, dim=0)
    return (src_rgb * sm).sum(0)


def query(scene: dict, fw: dict, pts: T, view: T, sp: dict | None = None,
          disable_fg_mask: bool = False, return_parts: bool = False):
    """``KeypointNeRF.query`` + ``query_color`` (reference ``src/model.py:690-843``).
    pts, view (N,3).  Returns out (N,5) = [sdf_raw, rad, r, g, b] and valid (N,) bool."""
    sp = sp or {}
    pts, view = _t(pts), _t(view)
    xy, z = project(scene, pts)
    valid = validity(scene, xy, z, disable_fg_mask)
    pw = pixel_weight(xy, z, valid)
    f64 = bilinear_border(_t(scene["feat64"]), xy)
    f8 = bilinear_border(_t(scene["feat8"]), xy)
    enc = encode_rel_z_decay(scene, pts, sp.get("sp_level", 3), sp.get("scale", 1.0), sp.get("sigma", 0.1))
    xv = geo_mlp(fw, enc, f64, f8)
    x_pool = pool_mean_var(xv, pw)
    geo = density_head(fw, x_pool)
    # colour branch (src/model.py:806-841)
    rgb_src = bilinear_border(_t(scene["img"]), xy)
    tex = bilinear_border(_t(scene["feat_tex"]), xy)
    lat = lin(fw, "ibr_compress_gfeat", x_pool)
    V = xy.shape[0]
    f = torch.cat([rgb_src, tex, lat[None].expand(V, -1, -1)], -1)
    rd = ray_diff(scene, pts, view)
    mask = valid[None, :, None].to(xy.dtype).expand(V, -1, -1)
    rgb = ibr_head(fw, f, rd, mask, rgb_src)
    out = torch.cat([geo, rgb], -1)
    if return_parts:
        return out, valid, {"xy": xy, "z": z, "pw": pw, "f64": f64, "f8": f8, "enc": enc,
                            "x_view": xv, "x_pool": x_pool, "rgb_src": rgb_src, "tex": tex,
                            "lat": lat, "ray_diff": rd}
    return out, valid


def eval_func(scene: dict, fw: dict, pts: T, view: T, sp=None, chunk: int = 1 << 18,
              disable_fg_mask: bool = False) -> T:
    """Closure ``eval_func`` of the tile renderer (reference ``src/model.py:978-997``):
    returns (N,5) = [alpha, sdf, r, g, b]."""
    outs = []
    for s in range(0, pts.shape[0], chunk):
        o, valid = query(scene, fw, pts[s:s + chunk], view[s:s + chunk], sp, disable_fg_mask)
        m = valid.to(o.dtype)[:, None]
        sdf = m * o[:, :1] + (1.0 - m) * (0.1 / float(scene["nml_scale"]))
        alpha = m * torch.relu(o[:, 1:2])
        outs.append(torch.cat([alpha, sdf, o[:, 2:]], -1))
    return torch.cat(outs, 0)


# --------------------------------------------------------------------------------------
# compositing and hierarchical sampling
# --------------------------------------------------------------------------------------
def composite(rgba: T, z: T):
    """``rgba2out`` (reference ``src/model.py:1150-1176``).  rgba (R,S,5)=[alpha,sdf,rgb], z (R,S)."""
    alpha, sdf, rgb = rgba[..., 0], rgba[..., 1], rgba[..., 2:]
    dist = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1)
    a = 1.0 - torch.exp(-alpha * dist)
    Tr = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), 1.0 - a[:, :-1]], -1), -1)
    c = a * Tr
    color = (rgb * c[..., None]).sum(-2)
    acc = c.sum(-1)
    sdf_o = (sdf * c).sum(-1) / (acc + 1e-8)
    depth = (z * c).sum(-1) / (acc + 1e-8)
    return color, depth, acc, c, sdf_o


def importance_sample(contrib_mid: T, z_mid: T, S_f: int) -> T:
    """Deterministic (``uniform=True``) inverse-CDF resampling (reference ``src/model.py:1110-1148``).
    contrib_mid (R,S_c-2), z_mid (R,S_c-1) -> (R,S_f)."""
    c = contrib_mid + 1e-5
    pdf = c / c.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)
    u = torch.linspace(0.0, 1.0, steps=S_f, dtype=contrib_mid.dtype)[None].expand(cdf.shape[0], -1).contiguous()
    idx = torch.searchsorted(cdf.contiguous(), u, right=True)
    lo = (idx - 1).clamp(min=0)
    hi = idx.clamp(max=cdf.shape[-1] - 1)
    c_lo, c_hi = torch.gather(cdf, -1, lo), torch.gather(cdf, -1, hi)
    z_lo, z_hi = torch.gather(z_mid, -1, lo), torch.gather(z_mid, -1, hi)
    den = c_hi - c_lo
    den = torch.where(den < 1e-5, torch.ones_like(den), den)
    return z_lo + ((u - c_lo) / den) * (z_hi - z_lo)


def render_pixels(scene: dict, fw: dict, target: dict, pix: T, S_c: int, S_f: int = 0, fine: bool = False,
                  sp=None, z_fine_override: T | None = None, disable_fg_mask: bool = False) -> dict:
    """Eval branch of ``batch_render_pifu_nerf`` for an arbitrary pixel list
    (reference ``src/model.py:1026-1096``).  Returns flat per-ray outputs."""
    o, d, n_r, f_r = ray_setup(pix, target["K"], target["RT"], float(target["znear"]), float(target["zfar"]))
    near, far, hit = ray_bbox(scene["bounds"], o, d)
    n_r, f_r = clip_near_far(n_r, f_r, near, far, hit)
    z = coarse_z(n_r, f_r, S_c)
    R = pix.shape[0]

    def shade(zz):
        S = zz.shape[1]
        pts = (o[:, None] + d[:, None] * zz[..., None]).reshape(-1, 3)
        view = d[:, None].expand(-1, S, -1).reshape(-1, 3)
        return eval_func(scene, fw, pts, view, sp, disable_fg_mask=disable_fg_mask).reshape(R, S, 5)

    rgba = shade(z)
    color, depth, acc, contrib, _ = composite(rgba, z)
    out = {"tex_fg": color, "depth": depth, "alpha": acc, "contrib": contrib, "z": z,
           "near": n_r, "far": f_r, "hit": hit, "rgba": rgba}
    if fine:
        z_mid = 0.5 * (z[:, 1:] + z[:, :-1])
        z_f = importance_sample(contrib[:, 1:-1], z_mid, S_f)
        z_all = torch.sort(torch.cat([z, z_f], -1), -1).values
        if z_fine_override is not None:
            z_all = _t(z_fine_override)
        rgba_f = shade(z_all)
        color_f, depth_f, acc_f, contrib_f, sdf_f = composite(rgba_f, z_all)
        out.update({"tex_fg_fine": color_f, "depth_fine": depth_f, "alpha_fine": acc_f,
                    "sdf": sdf_f, "z_fine": z_all, "rgba_fine": rgba_f})
    return out


def render_tile(scene, fw, target, level: int, x_off: int, y_off: int, S_c: int, S_f: int = 0,
                fine: bool = False, sp=None, **kw) -> dict:
    """One strided pass of ``batch_render_pifu_nerf`` (reference ``src/model.py:1018-1024``):
    returns images shaped like the reference's (3,h,w)/(h,w)."""
    step = 2 ** (level - 1)
    W, H = int(target["width"]), int(target["height"])
    pix = pixel_lattice(W, H, step, x_off, y_off)
    h, w = H // step, W // step
    flat = render_pixels(scene, fw, target, pix, S_c, S_f, fine, sp, **kw)
    out = {}
    for k, v in flat.items():
        if k in ("tex_fg", "tex_fg_fine"):
            out[k] = v.reshape(h, w, 3).permute(2, 0, 1)
        elif k in ("depth", "alpha", "depth_fine", "alpha_fine", "sdf"):
            out[k] = v.reshape(h, w)
        else:
            out[k] = v
    return out


def render_frame(scene, fw, target, S_c: int, S_f: int = 0, fine: bool = False, sp=None,
                 chunk_rays: int = 4096, **kw) -> dict:
    """Full frame.  The reference assembles it from stride^2 strided passes + pixel_shuffle
    (``src/model.py:916-938``); rays are independent so the result equals rendering every
    pixel in row-major order, which is what this does (in ray chunks to bound memory)."""
    W, H = int(target["width"]), int(target["height"])
    pix = pixel_lattice(W, H, 1, 0, 0)
    keys = ["tex_fg", "depth", "alpha"] + (["tex_fg_fine", "depth_fine", "alpha_fine", "sdf"] if fine else [])
    acc = {k: [] for k in keys}
    for s in range(0, pix.shape[0], chunk_rays):
        flat = render_pixels(scene, fw, target, pix[s:s + chunk_rays], S_c, S_f, fine, sp, **kw)
        for k in keys:
            acc[k].append(flat[k])
    out = {}
    for k in keys:
        v = torch.cat(acc[k], 0)
        out[k] = v.reshape(H, W, 3).permute(2, 0, 1) if v.dim() == 2 else v.reshape(H, W)
    return out
