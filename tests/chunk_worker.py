"""Renders of the chunk-boundary tests of tests/test_gpu_coverage.py, shared by the test process and a child process.

``KPN_CHUNK_SAMPLES`` (samples per render chunk) is read once per process, so the multi-chunk side of those comparisons runs here,
in a child started with the variable set; the test process runs ``render_config`` itself with the default chunk size and
compares.  Usage: ``python tests/chunk_worker.py CONFIG OUT_DIR`` writes ``OUT_DIR/CONFIG.npz``.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from keypointnerf_b200 import synthetic as syn  # noqa: E402
from keypointnerf_b200.testing import build_model, scene_tensors  # noqa: E402

# config -> (rays, samples per ray of the longest pass) for the callers' chunk arithmetic
SHAPES = {"partial": (97 * 83, 48 + 40), "bench": (512 * 512, 128)}


def _bind(scene, weights, target, n_kpt=18):
    net = build_model(weights, n_kpt, "cuda:0")
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    return m, a


def _render(m, out, key, **kw):
    """One render; stores its outputs under "<key>.<name>" and its valid-sample count and kernel launches."""
    before = m.stats()["kernel_launches"]
    r = m.render(**kw)
    st = m.stats()
    out[key + ".launches"] = np.array(st["kernel_launches"] - before)
    out[key + ".samples_valid"] = np.array(st["samples_valid"])
    for k, v in r.items():
        out[key + "." + k] = v.cpu().numpy()
    return r


def render_config(name):
    out = {}
    if name == "partial":
        # 97 x 83 rays of 48 coarse + 40 fine samples, early-ray termination, dense weights (density gain x600) so that rays do
        # terminate; with 65536 samples per chunk this is 13 chunks of 640 rays, the last one partial
        scene = syn.make_scene(src_size=128, n_kpt=18, fg_mode="hull", fg_hole=True)
        weights = syn.make_weights(18, density_gain=600.0)
        target = syn.make_target(size=97, azimuth=0.7, zoom=1.6, width=97, height=83)
        m, a = _bind(scene, weights, target)
        kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=97, ny=83, S_c=48, S_f=40,
                  fine=True, ert_eps=1e-3)
        for engine in (0, 1):
            r = _render(m, out, f"e{engine}", engine=engine, debug=True, **kw)
            # the fine pass on given depths (a copy, so that the override is read from its own buffer)
            _render(m, out, f"e{engine}_override", engine=engine, z_fine_override=r["z_fine"].clone(), **kw)
    elif name == "bench":
        # the 512 x 512 x 128 bench frame: one chunk of 4 non-empty geometry slices by default, 32 one-slice chunks with 2^20
        # samples per chunk
        scene = syn.make_scene(src_size=512, n_kpt=18)
        weights = syn.make_weights(18)
        target = syn.make_target(size=512)
        m, a = _bind(scene, weights, target)
        _render(m, out, "e0", K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=512, ny=512,
                S_c=128, engine=0)
    else:
        raise ValueError(name)
    torch.cuda.synchronize()
    m.check_health()
    return out


if __name__ == "__main__":
    cfg, out_dir = sys.argv[1], sys.argv[2]
    res = render_config(cfg)
    np.savez(os.path.join(out_dir, cfg + ".npz"), **res)
    print("CHUNK_WORKER_OK", cfg, os.environ.get("KPN_CHUNK_SAMPLES"))
