"""Golden vectors for the geometry-only grid query (kpn_query_grid): the UNMODIFIED reference's ``KeypointNeRF.query`` at the points
of a regular grid over the scene's bounds, run on CPU (same harness and file format as make_golden.py, whose functions this
reuses).  Each file holds ``grid_out`` = [sdf_raw, rad] (N,2), ``grid_valid`` (N,) and the input checksum; the meta carries the
scene parameters and ``grid`` = {origin, spacing, dims}.  Point (i,j,k) has id (k ny + j) nx + i and sits at
origin + spacing * idx in fp32 (one multiply, one add; tests/mesh_ref.grid_points).  The view direction does not enter
[sdf_raw, rad]; (0, 0, 1) is passed, and the colour branch, which groups the points into rays of n_pts_samples, is given
the grid's rows (nx points each).

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_grid.py              # every case below
    python tests/golden/make_golden_grid.py grid_tiny    # only the named cases
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402
from tests.mesh_ref import grid_points  # noqa: E402

syn = G.syn


def _c(dims, **kw):
    d = G._c(**dict({"n_views": 3}, **kw))
    d["grid_dims"] = list(dims)
    return d


# three views with 18 keypoints; the Human3.6M shape (four views, 17 keypoints, hull masks with holes, non-square sources); two
# views (the fp32 engine's shape)
GRID_CASES = {
    "grid_tiny": _c((30, 28, 26), src_size=64, tgt_size=32, zoom=2.0),
    "grid_rect_v4_k17": _c((32, 26, 30), n_views=4, n_kpt=17, src_size=128, src_height=80, tgt_size=48, fg_hole=True),
    "grid_v2": _c((28, 30, 24), n_views=2, src_size=64, tgt_size=32, zoom=2.0, fg_hole=True),
}


def grid_for(bounds, dims):
    """fp32 origin and spacing of a grid of ``dims`` points spanning ``bounds`` (returned as the float values of the fp32s)."""
    b = np.asarray(bounds, np.float64).reshape(2, 3)
    origin = b[0].astype(np.float32)
    spacing = ((b[1] - b[0]) / (np.asarray(dims) - 1)).astype(np.float32)
    return [float(x) for x in origin], [float(x) for x in spacing]


def main():
    M = G.import_reference()
    torch.set_num_threads(8)
    names = sys.argv[1:] or list(GRID_CASES)
    for name in names:
        c = dict(GRID_CASES[name])
        dims = c.pop("grid_dims")
        scene = syn.make_scene(src_size=c["src_size"], n_views=c["n_views"], n_kpt=c["n_kpt"], seed=c["scene_seed"],
                               fg_mode=c["fg_mode"], fg_hole=c["fg_hole"], src_height=c.get("src_height"))
        weights = syn.make_weights(c["n_kpt"], seed=c["w_seed"])
        target = syn.make_target(size=c["tgt_size"], azimuth=c["azimuth"], zoom=c["zoom"])
        net = G.build_net(M, c["n_kpt"], weights)
        cam, _, sp_data, feat_geo, feat_tex, img, fg, _ = G.ref_inputs(scene, target)
        origin, spacing = grid_for(scene["bounds"], dims)
        pts = torch.from_numpy(grid_points(origin, spacing, dims).reshape(1, -1, 3))
        view = torch.zeros_like(pts)
        view[..., 2] = 1.0
        with torch.no_grad():
            out, valid = net.query(pts, cam, feat_geo, feat_tex, n_views=c["n_views"], view=view, nerf=True, sp_data=dict(sp_data),
                                   tx_data={"img": img}, n_pts_samples=dims[0], src_foreground_mask=fg)
        valid = valid[0, :, 0].numpy().astype(bool)
        res = {"grid_out": np.ascontiguousarray(out[0, :, :2].numpy()), "grid_valid": valid}
        meta = {k: v for k, v in c.items() if k != "capture"}
        meta["grid"] = {"origin": origin, "spacing": spacing, "dims": dims}
        res["input_sha256"] = np.frombuffer(G.checksum(scene, weights).encode(), dtype=np.uint8)
        res["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        G.save_golden(name, res, G.HERE)
        print(name, dims, "valid frac", float(valid.mean()), "rad max", float(res["grid_out"][valid, 1].max()), flush=True)


if __name__ == "__main__":
    main()
