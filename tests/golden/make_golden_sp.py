"""Golden vectors for the spatial-encoding parameters (sp_args.sp_level / scale / sigma) and for one and two source views, from
the UNMODIFIED reference on CPU (same harness and file format as make_golden.py, whose functions this reuses).

The case meta carries ``n_views``, ``sp_level``, ``scale`` and ``sigma``; ``sigma`` null means the key is left out of the
reference's config, so that its own default (150, src/spatial.py:112) applies.  ``dz_scale`` divides the layer-0 columns of the
dz row (``synthetic.make_weights``), so that with a large ``scale`` layer 0 still sees inputs of the usual size.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_sp.py            # every case below
    python tests/golden/make_golden_sp.py tiny_v1    # only the named cases
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402

syn = G.syn


def _c(**kw):
    d = dict(n_views=3, sp_level=3, scale=1.0, sigma=0.1, dz_scale=1.0)
    d.update(kw)
    return G._c(**d)


_TINY = dict(src_size=64, tgt_size=32, zoom=2.0, level=1, S_c=12, S_f=8, fine=True, capture="all")

# one and two views with every intermediate; two views with non-square sources and target, level 2 with offsets and 17
# keypoints; two views at config size (hull scene, one strided pass of BASELINE config 2); every sp_level other than 3, including
# 0 (the dz row alone) and 4 with 24 keypoints (a 280-float layer-0 input, the widest the fp32 engine's 288-float rows hold);
# sp_level 1 with two views; scale / sigma other than 1 / 0.1; a large |scale * dz| (|dz| up to ~60: the level-2 sin / cos
# arguments span ~120 periods); sigma left out of the config (150).  tiny_dz stops at scale 100: at 1000 the reference's own fp32
# encoding is 2.5e-3 from the exact one (camera-depth round-off times scale * 4 pi) and its image 2.4e-4 from the fp64 oracle's,
# beyond the fp32 engine's 1e-4 gate, and one of its fine samples changes the image by 0.06 when its depth moves by one ulp.
SP_CASES = {
    "tiny_v1": _c(n_views=1, **dict(_TINY, S_c=16, S_f=16)),
    "tiny_v2": _c(n_views=2, **dict(_TINY, S_c=16, S_f=16)),
    "rect_v2_k17": _c(n_views=2, src_size=128, src_height=80, tgt_size=48, tgt_width=48, tgt_height=32, zoom=3.5, level=2,
                      x_off=1, y_off=1, S_c=12, S_f=8, fine=True, n_kpt=17, fg_hole=True, capture="all"),
    "cfg2_pass_v2": _c(n_views=2, x_off=3, y_off=5, S_c=128, capture="some"),
    "tiny_L0_k32": _c(sp_level=0, n_kpt=32, azimuth=1.5, w_seed=29, **_TINY),
    "tiny_L2": _c(sp_level=2, **_TINY),
    "tiny_L4_k24": _c(sp_level=4, n_kpt=24, azimuth=2.5, scene_seed=3, w_seed=5, **_TINY),
    "tiny_v2_L1": _c(n_views=2, sp_level=1, **_TINY),
    "tiny_sig": _c(scale=2.5, sigma=0.25, **_TINY),
    "tiny_dz": _c(scale=100.0, sigma=0.15, dz_scale=100.0, w_seed=27, **_TINY),
    "tiny_nosigma": _c(sigma=None, **_TINY),
}

SOME_KEYS = ["tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf", "z_fine", "contrib_coarse", "z_coarse"]


def main():
    M = G.import_reference()
    torch.set_num_threads(8)
    names = sys.argv[1:] or list(SP_CASES)
    for name in names:
        c = SP_CASES[name]
        scene = syn.make_scene(src_size=c["src_size"], n_views=c["n_views"], n_kpt=c["n_kpt"], seed=c["scene_seed"],
                               fg_mode=c["fg_mode"], fg_hole=c["fg_hole"], src_height=c.get("src_height"))
        weights = syn.make_weights(c["n_kpt"], seed=c["w_seed"], sp_level=c["sp_level"], dz_scale=c["dz_scale"])
        target = syn.make_target(size=c["tgt_size"], azimuth=c["azimuth"], zoom=c["zoom"], width=c.get("tgt_width"),
                                 height=c.get("tgt_height"))
        sp = syn.sp_args(c["n_kpt"], sp_level=c["sp_level"], scale=c["scale"], sigma=c["sigma"])
        net = G.build_net(M, c["n_kpt"], weights, sp)
        assert net.sp_encoder.kwargs.get("sigma", 150.0) == (150.0 if c["sigma"] is None else c["sigma"])
        res = G.run_tile(M, net, scene, target, level=c["level"], x_off=c["x_off"], y_off=c["y_off"], S_c=c["S_c"],
                         S_f=c["S_f"], fine=c["fine"], capture=c["capture"] != "none")
        valid_frac = float(res["query_valid"].mean()) if "query_valid" in res else float("nan")
        if c["capture"] == "some":
            res = {k: res[k] for k in SOME_KEYS if k in res}
        meta = {k: v for k, v in c.items() if k != "capture"}
        res["input_sha256"] = np.frombuffer(G.checksum(scene, weights).encode(), dtype=np.uint8)
        res["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        res.pop("rgba_fine", None)
        if not c["fine"]:
            res.pop("z_coarse", None)
        G.save_golden(name, res, G.HERE)
        print(name, res["tex_fg"].shape, "valid frac", valid_frac, "alpha mean", float(res["alpha"].mean()),
              "alpha max", float(res["alpha"].max()), flush=True)


if __name__ == "__main__":
    main()
