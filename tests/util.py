"""Shared helpers for the tests: golden loading and scene reconstruction from fixture metadata."""
import hashlib
import json
import os

import numpy as np

from keypointnerf_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# Golden files stay below 1 MB each: float32 arrays are stored losslessly as their four byte planes ("<key>__bp"; "<key>__bpd"
# when the array is sorted along its last axis and its bit patterns are delta-coded along it first), which compresses far
# better than the raw floats, and a fixture that is still too large is split into parts <name>.npz, <name>.1.npz, ...
PART_BYTES = 900_000


def _encode(k, a):
    if a.dtype != np.float32 or a.ndim == 0:
        return {k: a}
    u = np.ascontiguousarray(a).view(np.uint32)
    suffix = "__bp"
    if a.shape[-1] > 1 and bool(np.all(np.diff(a, axis=-1) >= 0)):
        u = np.diff(u.astype(np.int64), axis=-1, prepend=0).astype(np.uint32)
        suffix = "__bpd"
    return {k + suffix: np.ascontiguousarray(np.moveaxis(u.view(np.uint8).reshape(u.shape + (4,)), -1, 0))}


def _decode(k, a):
    if k.endswith("__bpd") or k.endswith("__bp"):
        u = np.ascontiguousarray(np.moveaxis(a, 0, -1)).view(np.uint32)[..., 0]
        if k.endswith("__bpd"):
            u = np.cumsum(u.astype(np.uint64), axis=-1).astype(np.uint32)
        return k.rsplit("__", 1)[0], u.view(np.float32)
    return k, a


def save_golden(name, arrays, directory=GOLDEN):
    import io
    enc = {}
    for k, a in arrays.items():
        enc.update(_encode(k, np.asarray(a)))
    parts, cur = [], {}
    for k in sorted(enc, key=lambda k: enc[k].nbytes):
        trial = dict(cur, **{k: enc[k]})
        buf = io.BytesIO()
        np.savez_compressed(buf, **trial)
        if cur and len(buf.getvalue()) > PART_BYTES:
            parts.append(cur)
            cur = {k: enc[k]}
        else:
            cur = trial
    parts.append(cur)
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(directory, name + (f".{i}" if i else "") + ".npz"), **part)


def load_golden(name):
    g, i = {}, 0
    while True:
        path = os.path.join(GOLDEN, name + (f".{i}" if i else "") + ".npz")
        if not os.path.exists(path):
            break
        z = np.load(path)
        g.update(_decode(k, z[k]) for k in z.files)
        i += 1
    meta = json.loads(bytes(g.pop("meta")).decode())
    sha = bytes(g.pop("input_sha256")).decode()
    return g, meta, sha


def target_wh(meta):
    """(width, height) of a fixture's target image; fixtures without the keys are square."""
    return int(meta.get("tgt_width") or meta["tgt_size"]), int(meta.get("tgt_height") or meta["tgt_size"])


def scene_from_meta(meta):
    """Seeded scene, weights and target of a fixture.  ``src_height`` / ``tgt_width`` / ``tgt_height`` describe non-square
    sources and targets; older fixtures do not have them and are square (``src_size`` / ``tgt_size``).  ``n_views``,
    ``sp_level`` and ``dz_scale`` default to 3, 3 and 1 (fixtures that predate them)."""
    scene = syn.make_scene(src_size=meta["src_size"], n_views=meta.get("n_views", 3), n_kpt=meta["n_kpt"], seed=meta["scene_seed"],
                           fg_hole=meta["fg_hole"], fg_mode=meta.get("fg_mode", "ones"), src_height=meta.get("src_height"))
    weights = syn.make_weights(meta["n_kpt"], seed=meta["w_seed"], sp_level=meta.get("sp_level", 3),
                               dz_scale=meta.get("dz_scale", 1.0))
    w, h = target_wh(meta)
    target = syn.make_target(size=meta["tgt_size"], azimuth=meta["azimuth"], zoom=meta.get("zoom", 1.0), width=w, height=h)
    return scene, weights, target


def sp_from_meta(meta):
    """The fixture's ``sp_args`` overrides for ``testing.build_model`` (sigma None: left out of the config, so 150) and the same
    parameters as the oracle's ``sp`` dict (which needs the value itself)."""
    sp = {"sp_level": meta.get("sp_level", 3), "scale": meta.get("scale", 1.0), "sigma": meta.get("sigma", 0.1)}
    return sp, dict(sp, sigma=150.0 if sp["sigma"] is None else sp["sigma"])


def checksum(scene, weights):
    h = hashlib.sha256()
    for k in ("feat64", "feat8", "feat_tex", "img", "fg", "kpt3d", "KRT", "extrin"):
        h.update(np.ascontiguousarray(scene[k]).tobytes())
    for k in sorted(weights):
        h.update(np.ascontiguousarray(weights[k]).tobytes())
    return h.hexdigest()


# Warpgroups per CTA of the tensor-core engine's kernels, which launch at most one CTA per SM (kpn_shade_tc.cuh): the geometry
# front kernel's depend on the keypoint count (front_wgs there, the same for 3 and 4 views), the density tail runs GWG, the colour
# kernel CWG.  One persistent wave of a kernel is SMs x warpgroups x samples per tile.
def front_wgs(n_kpt):
    return 2 if n_kpt <= 14 else 3 if n_kpt <= 20 else 2 if n_kpt <= 28 else 1


TAIL_WGS = 2
COLOUR_WGS = 3


def tile_samples(n_views):
    """Samples per tile of the geometry front kernel (two warps of 32 // n_views samples), the density tail and the colour
    kernel (four warps)."""
    return 2 * (32 // n_views), 64, 4 * (32 // n_views)


def psnr(a, b):
    mse = float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))
    return 99.0 if mse == 0 else 10.0 * np.log10(1.0 / mse)
