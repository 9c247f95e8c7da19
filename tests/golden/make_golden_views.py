"""Golden vectors for four source views, from the UNMODIFIED reference on CPU (same harness and file format as make_golden.py,
whose functions this reuses).  The case meta carries ``n_views``; make_golden.main builds three-view scenes, so the scenes are
built by the loop below.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_views.py            # every case below
    python tests/golden/make_golden_views.py tiny_v4    # only the named cases
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
    return G._c(n_views=4, **kw)


# every intermediate with 18 keypoints; the Human3.6M shape (four cameras, 17 keypoints, non-square sources and target, level 2
# with offsets); 32 keypoints (one front warpgroup per CTA, the widest layer 0); one strided pass of BASELINE config 2 at config
# size (hull scene)
VIEW_CASES = {
    "tiny_v4": _c(src_size=64, tgt_size=32, zoom=2.0, level=1, S_c=16, S_f=16, fine=True, capture="all"),
    "rect_v4_k17": _c(src_size=128, src_height=80, tgt_size=48, tgt_width=48, tgt_height=32, zoom=3.5, level=2, x_off=1, y_off=1,
                      S_c=12, S_f=8, fine=True, n_kpt=17, fg_hole=True, capture="all"),
    "tiny_v4_k32": _c(src_size=64, tgt_size=32, zoom=2.0, azimuth=1.5, level=1, S_c=12, S_f=8, fine=True, n_kpt=32,
                      scene_seed=5, w_seed=9, capture="all"),
    "cfg2_pass_v4": _c(x_off=3, y_off=5, S_c=128, capture="some"),
}

SOME_KEYS = ["tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf", "z_fine", "contrib_coarse", "z_coarse"]


def main():
    M = G.import_reference()
    torch.set_num_threads(8)
    names = sys.argv[1:] or list(VIEW_CASES)
    for name in names:
        c = VIEW_CASES[name]
        scene = syn.make_scene(src_size=c["src_size"], n_views=c["n_views"], n_kpt=c["n_kpt"], seed=c["scene_seed"],
                               fg_mode=c["fg_mode"], fg_hole=c["fg_hole"], src_height=c.get("src_height"))
        weights = syn.make_weights(c["n_kpt"], seed=c["w_seed"])
        target = syn.make_target(size=c["tgt_size"], azimuth=c["azimuth"], zoom=c["zoom"], width=c.get("tgt_width"),
                                 height=c.get("tgt_height"))
        net = G.build_net(M, c["n_kpt"], weights)
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
