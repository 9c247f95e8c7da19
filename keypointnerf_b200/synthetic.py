"""Synthetic scenes, cameras and weights for the ray-march hot path.

Everything here is numpy-only and seeded with ``numpy.random.default_rng`` so that the
golden-vector generator (which runs the reference in the build container), the CPU
oracle and the GPU tests/bench all see bit-identical inputs without shipping them.

The recipe follows SURVEY.md section 8(d): pinhole source cameras on a radius-3 circle
looking at the origin (znear=2, zfar=5 as hard-coded at reference ``src/model.py:43,345``),
K keypoints in a 0.6 x 1.6 x 0.4 m box, random feature maps with the shapes the
reference encoders emit for a given source resolution, and He-style re-initialised
MLP weights with a x30 gain on the density row (the reference's default init gives
density ~0, SURVEY.md section 8(c)).

Parameter names are the reference's ``KeypointNeRF.state_dict()`` keys
(``src/model.py:584-587``, ``src/utils.py:476-553``, ``src/model.py:1242-1258``).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def look_at_extrinsic(azimuth: float, radius: float = 3.0, height: float = 0.0) -> np.ndarray:
    """World->camera 4x4 for a camera on a circle in the XZ plane looking at the origin.

    Camera axes: +z forward (positive depth, as the projection at reference
    ``src/model.py:713-715`` needs), +y down the image, +x right.
    """
    c = np.array([radius * np.sin(azimuth), height, radius * np.cos(azimuth)], dtype=np.float64)
    zc = -c / np.linalg.norm(c)
    up = np.array([0.0, 1.0, 0.0])
    xc = np.cross(up, zc)
    xc /= np.linalg.norm(xc)
    yc = np.cross(zc, xc)
    # image y grows downwards: flip so that world +y maps to image -y
    R = np.stack([xc, -yc, zc], 0)
    if np.linalg.det(R) < 0:
        R[0] = -R[0]
    Rt = np.eye(4)
    Rt[:3, :3] = R
    Rt[:3, 3] = -R @ c
    return Rt.astype(F32)


def intrinsic(size: int, focal_at_512: float = 550.0, height: int | None = None) -> np.ndarray:
    """Pinhole K for a ``size`` (width) x ``height`` image (square when ``height`` is None): the focal length scales with the
    width, the principal point is the image centre (W/2, H/2)."""
    height = size if height is None else height
    s = size / 512.0
    K = np.eye(4, dtype=np.float64)
    K[0, 0] = K[1, 1] = focal_at_512 * s
    K[0, 2] = 256.0 * s
    K[1, 2] = 256.0 * (height / 512.0)
    return K.astype(F32)


def feature_shapes(src_size: int, n_views: int = 3, src_height: int | None = None):
    """Shapes the reference encoders produce for ``src_size`` (width) x ``src_height`` inputs (square when ``src_height`` is
    None; SURVEY.md section 8 header)."""
    W, H = src_size, (src_size if src_height is None else src_height)
    return {
        "feat64": (n_views, 64, H // 8, W // 8),
        "feat8": (n_views, 8, H // 2, W // 2),
        "feat_tex": (n_views, 8, H // 4, W // 4),
        "img": (n_views, 3, H, W),
        "fg": (n_views, 1, H, W),
    }


def silhouette_masks(K: np.ndarray, extrin: np.ndarray, src_size: int, semi_axes=(0.22, 0.64, 0.15),
                     src_height: int | None = None) -> np.ndarray:
    """Foreground masks (V,1,H,W) bool = silhouettes of an origin-centred ellipsoid seen by each source camera.

    The intersection of the silhouette cones (the visual hull the validity test carves, reference ``src/model.py:729-739``)
    lies strictly inside the keypoint bounding box, so the LAST sample of every target ray (at the bbox exit, or at zfar for
    rays that miss the box) is invalid: the reference's final-sample step (``dist[-1] = 1e10``, ``src/model.py:1166``) then
    multiplies a density of exactly 0 and no ray sits on that discontinuity (SURVEY.md section 7.4)."""
    V = K.shape[0]
    W, H = src_size, (src_size if src_height is None else src_height)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    pix = np.stack([xs, ys, np.ones_like(xs)], -1).reshape(-1, 3)
    inv_ax = 1.0 / np.asarray(semi_axes, dtype=np.float64)
    out = np.zeros((V, 1, H, W), dtype=bool)
    for v in range(V):
        R = extrin[v, :3, :3].astype(np.float64)
        t = extrin[v, :3, 3].astype(np.float64)
        c = -R.T @ t                                             # camera centre
        d = (pix @ np.linalg.inv(K[v, :3, :3].astype(np.float64)).T) @ R   # world-space pixel rays
        ds, cs = d * inv_ax, c * inv_ax                          # unit-sphere coordinates
        a = (ds * ds).sum(-1)
        b = ds @ cs
        disc = b * b - a * ((cs * cs).sum() - 1.0)
        out[v, 0] = (disc >= 0.0).reshape(H, W)
    return out


def make_scene(src_size: int = 512, n_views: int = 3, n_kpt: int = 18, seed: int = 2,
               src_azimuths=(0.0, 2.1, 4.2, 5.25), fg_hole: bool = False, fg_mode: str | None = None,
               src_height: int | None = None) -> dict:
    """Source-side inputs of the hot path (everything ``query`` reads, reference ``src/model.py:690-782``).

    The source images are ``src_size`` wide and ``src_height`` high (square when ``src_height`` is None).
    ``fg_mode``: "ones" (SURVEY.md section 8d recipe, the bench scene) or "hull" (ellipsoid silhouettes, see
    ``silhouette_masks``); ``fg_hole`` additionally punches rectangular holes into either."""
    if fg_mode is None:
        fg_mode = "ones"
    assert fg_mode in ("ones", "hull")
    assert len(src_azimuths) >= n_views
    rng_k = np.random.default_rng(1)
    box = np.array([0.6, 1.6, 0.4])
    kpt3d = ((rng_k.random((n_kpt, 3)) - 0.5) * box).astype(F32)[None]  # (1,K,3)
    bounds = np.stack([kpt3d[0].min(0) - 0.1, kpt3d[0].max(0) + 0.1], 0).astype(F32)[None]  # (1,2,3)

    rng = np.random.default_rng(seed)
    W, H = src_size, (src_size if src_height is None else src_height)
    sh = feature_shapes(W, n_views, H)
    feat64 = rng.standard_normal(sh["feat64"], dtype=F32)
    feat8 = rng.standard_normal(sh["feat8"], dtype=F32)
    feat_tex = rng.standard_normal(sh["feat_tex"], dtype=F32)
    img = rng.random(sh["img"], dtype=F32)
    K = intrinsic(W, height=H)
    extrin = np.stack([look_at_extrinsic(a) for a in src_azimuths[:n_views]], 0)
    Ks = np.broadcast_to(K, (n_views, 4, 4)).copy()
    fg = silhouette_masks(Ks, extrin, W, src_height=H) if fg_mode == "hull" else np.ones(sh["fg"], dtype=bool)
    if fg_hole:
        # punch rectangular holes so that the foreground-mask term of the validity test
        # (reference src/model.py:737-739) is exercised, including its bilinear edge.
        for v in range(n_views):
            ay, ax = H // 4 + v * (H // 16), W // 4 + v * (W // 16)
            fg[v, 0, ay:ay + H // 8, ax:ax + W // 6] = False
        fg[:, :, : H // 10, :] = False

    KRT = np.einsum("vij,vjk->vik", Ks.astype(np.float64), extrin.astype(np.float64)).astype(F32)
    return {
        "n_views": n_views, "n_kpt": n_kpt, "src_size": src_size, "fg_mode": fg_mode,
        "kpt3d": kpt3d, "bounds": bounds,
        "feat64": feat64, "feat8": feat8, "feat_tex": feat_tex, "img": img, "fg": fg,
        "K": Ks, "extrin": extrin, "KRT": KRT,
        "width": float(W), "height": float(H),
        "znear": 2.0, "zfar": 5.0, "nml_scale": 100.0,
    }


def make_target(size: int = 512, azimuth: float = 1.0, znear: float = 2.0, zfar: float = 5.0, zoom: float = 1.0,
                width: int | None = None, height: int | None = None) -> dict:
    """Target camera dict as ``decode_batch`` builds it (reference ``src/model.py:309-414``); ``zoom`` scales the focal length
    (small test targets zoom in so that most of their rays cross the visual hull).  The image is ``width`` x ``height``
    (each defaults to ``size``)."""
    W, H = (size if width is None else width), (size if height is None else height)
    K = intrinsic(W, 550.0 * zoom, height=H)[None]
    RT = look_at_extrinsic(azimuth)[None]
    KRT = (K[0].astype(np.float64) @ RT[0].astype(np.float64)).astype(F32)[None]
    return {"K": K, "RT": RT, "KRT": KRT, "width": W, "height": H,
            "znear": znear, "zfar": zfar, "nml_scale": 100.0}


def layer_table(n_kpt: int = 18, sp_level: int = 3):
    """(key prefix, out, in, weight-normed?) for every dense layer on the path (SURVEY.md Appendix D).  Layer 0 reads the
    (1 + 2 sp_level) n_kpt keypoint encoding and the 64 feat64 channels."""
    enc = (1 + 2 * sp_level) * n_kpt
    return [
        ("mlp_geo.layers1.layers.0.linear", 128, enc + 64, True),
        ("mlp_geo.layers1.layers.1.linear", 128, 128, True),
        ("mlp_geo.layers1.layers.2.linear", 120, 136, True),
        ("mlp_geo.layers1.layers.3.linear", 64, 120, False),
        ("mlp_geo.layers2.layers.0.linear", 64, 128, True),
        ("mlp_geo.layers2.layers.1.linear", 64, 64, True),
        ("mlp_geo.layers2.layers.2.linear", 2, 64, False),
        ("ibr_compress_gfeat", 24, 128, False),
        ("mlp_tex.ray_encoder.0", 16, 4, False),
        ("mlp_tex.ray_encoder.2", 35, 16, False),
        ("mlp_tex.base_layer.0", 64, 105, False),
        ("mlp_tex.base_layer.2", 32, 64, False),
        ("mlp_tex.vis_layer1.0", 32, 32, False),
        ("mlp_tex.vis_layer1.2", 33, 32, False),
        ("mlp_tex.vis_layer2.0", 32, 32, False),
        ("mlp_tex.vis_layer2.2", 1, 32, False),
        ("mlp_tex.out_layer.0", 16, 37, False),
        ("mlp_tex.out_layer.2", 8, 16, False),
        ("mlp_tex.out_layer.4", 1, 8, False),
    ]


def make_weights(n_kpt: int = 18, seed: int = 26, density_gain: float = 30.0, sp_level: int = 3, dz_scale: float = 1.0) -> dict:
    """Seeded hot-path parameters keyed like the reference state_dict, for a ``sp_level`` keypoint encoding.

    ``dz_scale``: the layer-0 columns that read the encoding's dz row (the first n_kpt inputs) are divided by it, so that with
    ``sp_args.scale = dz_scale`` layer 0 sees inputs of the size a model trained in those units would (the sin / cos rows are
    bounded by 1 at any scale)."""
    rng = np.random.default_rng(seed)
    w = {}
    for name, n_out, n_in, wn in layer_table(n_kpt, sp_level):
        if wn:
            v = (rng.standard_normal((n_out, n_in)) * np.sqrt(2.0 / n_in)).astype(F32)
            if dz_scale != 1.0 and name == "mlp_geo.layers1.layers.0.linear":
                v[:, :n_kpt] = (v[:, :n_kpt] / np.float32(dz_scale)).astype(F32)
            w[name + ".weight_v"] = v
            w[name + ".weight_g"] = np.linalg.norm(v.astype(np.float64), axis=1, keepdims=True).astype(F32)
        else:
            w[name + ".weight"] = (rng.standard_normal((n_out, n_in)) * np.sqrt(1.0 / n_in)).astype(F32)
        w[name + ".bias"] = (rng.standard_normal((n_out,)) * 0.1).astype(F32)
    w["mlp_geo.layers2.layers.2.linear.weight"][1] *= density_gain
    w["mlp_geo.layers2.layers.2.linear.bias"][1] *= density_gain
    w["mlp_tex.ani_al"] = np.array(0.2, dtype=F32)
    return w


def sp_args(n_kpt: int = 18, **overrides) -> dict:
    """``configs/zju.json:38-44`` with n_kpt and any of ``sp_level`` / ``scale`` / ``sigma`` overridden; ``sigma=None`` leaves the
    key out, so that the reference's default (150, ``src/spatial.py:112``) applies."""
    sp = {"sp_level": 3, "sp_type": "rel_z_decay", "scale": 1.0, "sigma": 0.1, "n_kpt": n_kpt}
    unknown = set(overrides) - {"sp_level", "scale", "sigma"}
    if unknown:
        raise ValueError(f"unknown sp_args overrides {sorted(unknown)}")
    sp.update(overrides)
    if sp["sigma"] is None:
        del sp["sigma"]
    return sp
