"""The backward of tests/test_gpu_grad_edges.py's multi-chunk case, shared by the test process and a child process.

``KPN_CHUNK_SAMPLES`` (samples per chunk) is read once per process, so the multi-chunk side runs here, in a child started with
the variable set; the test process runs ``grad_config`` itself with the default chunk size and compares.  1300 rays of 64 + 64
samples: with 65536 samples per chunk that is chunks of 512 rays, three of them, the last one partial.
Usage: ``python tests/grad_chunk_worker.py OUT_DIR`` writes ``OUT_DIR/grad_chunks.npz``.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from keypointnerf_b200 import synthetic as syn  # noqa: E402
from keypointnerf_b200.model import param_grads  # noqa: E402
from tests import grad_oracle as GO  # noqa: E402

N_RAYS, S_C, S_F, N_KPT = 1300, 64, 64, 18
SP = {"sp_level": 3, "scale": 1.0, "sigma": 0.1}


def inputs():
    """Scene, weights, the 1300 rays (the first rows of a 26 x 50 lattice, which covers the box) and the loss weights G."""
    scene = syn.make_scene(src_size=64, n_views=3, n_kpt=N_KPT, fg_mode="hull")
    weights = syn.make_weights(N_KPT)
    target = syn.make_target(size=50, width=50, height=26, zoom=2.0)
    o, d, nf = GO.lattice_rays(target, 50)   # 50 x 50 lattice of a 50-wide target; its first 26 rows
    rays = (o[:N_RAYS].contiguous(), d[:N_RAYS].contiguous(), nf[:N_RAYS].contiguous())
    return scene, weights, target, rays, GO.loss_weights(N_RAYS, seed=5)


def grad_config(subsets=()):
    """The engine-1 forward's fine depths, then the backward at them (launch count, raw and parameter gradients); the same for
    each ray range of `subsets` (prefixed "s<i>/")."""
    scene, weights, target, rays, G = inputs()
    net, a = GO.bind(scene, weights, SP, target, N_KPT)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    r = [t.to(GO.DEV) for t in rays]
    kw = dict(S_c=S_C, S_f=S_F, fine=True)
    z = m.render_rays(*r, engine=1, debug=True, **kw)["z_fine"]
    out = {"z_fine": z.cpu().numpy()}

    def backward(prefix, sl):
        before = m.stats()["kernel_launches"]
        g = m.render_rays_backward(*(t[sl] for t in r), {k: v[..., sl].to(GO.DEV) for k, v in G.items()}, z_fine_override=z[sl], **kw)
        torch.cuda.synchronize()
        out[prefix + "launches"] = np.array(m.stats()["kernel_launches"] - before)
        names = [n + s for n, _, _, wn in syn.layer_table(N_KPT) for s in ((".weight_v", ".weight_g", ".bias") if wn else (".weight", ".bias"))]
        for k, v in zip(names + ["mlp_tex.ani_al"], param_grads(net, g, net.hot_parameters())):
            out[prefix + "p/" + k] = v.detach().cpu().numpy()
        for k in GO.MAPS:
            out[prefix + "m/" + k] = g["d_" + k].cpu().numpy()

    backward("", slice(None))
    for i, (lo, hi) in enumerate(subsets):
        backward(f"s{i}/", slice(lo, hi))
    m.check_health()
    return out


if __name__ == "__main__":
    out_dir = sys.argv[1]
    np.savez(os.path.join(out_dir, "grad_chunks.npz"), **grad_config())
    print("GRAD_CHUNK_WORKER_OK", os.environ.get("KPN_CHUNK_SAMPLES"))
