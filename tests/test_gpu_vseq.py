"""Engine 3 (an alias of the default tensor-core engine; it selected a view-sequential geometry kernel on an earlier
architecture): same gates as tests/test_gpu_parity.py, against the reference's goldens, the fp32 engine and engine 4."""
import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model, scene_tensors
from tests.test_gpu_parity import ALL, TOL, _golden_case, _render_tile, check
from tests.util import psnr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["tiny", "tiny_fg", "rect", "rect_k24", "cfg1_tile", "cfg2_pass", "cfg4_pass"])
def test_vseq_matches_reference(name):
    g, meta, scene, weights, target, net = _golden_case(name)
    r = _render_tile(net, dict(meta, fine=False), scene, target, engine=3)
    t = TOL[0]
    rep = []
    good = check(rep, "tex_fg", r["tex_fg"], g["tex_fg"][0], ALL, t["rgb"])
    good &= check(rep, "alpha", r["alpha"], g["alpha"][0], ALL, t["alpha"])
    p = psnr(r["tex_fg"], g["tex_fg"][0])
    print(f"vseq {name}: " + "; ".join(rep) + f"; psnr {p:.1f} dB")
    net.marcher().check_health()
    assert good and p > t["psnr"], rep


def test_vseq_query_and_frame_agree_with_fp32_engine():
    scene = syn.make_scene(src_size=512, n_kpt=18)
    weights = syn.make_weights(18)
    target = syn.make_target(size=256)
    net = build_model(weights, 18, "cuda:0")
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    gen = torch.Generator().manual_seed(0)
    n = 100000
    pts = ((torch.rand(n, 3, generator=gen) - 0.5) * torch.tensor([0.8, 1.8, 0.6])).cuda()
    view = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1).cuda()
    o1, v1 = m.query(pts, view, engine=1)
    o3, v3 = m.query(pts, view, engine=3)
    o3b, _ = m.query(pts, view, engine=3)
    torch.cuda.synchronize()
    m.check_health()
    assert torch.equal(v3, v1) and torch.equal(o3, o3b)
    d = (o3 - o1).abs()[v1]
    print(f"vseq per-sample vs fp32: rgb {float(d[:, 2:].max()):.2e} rad {float(d[:, 1].max()):.2e} sdf {float(d[:, 0].max()):.2e}")
    assert float(d[:, 2:].max()) < 5e-4 and float(d[:, 1].max()) < 5e-2 and float(d[:, 0].max()) < 5e-3
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, S_c=96, x0=0, y0=0, step=1, nx=256, ny=256)
    f3 = m.render(engine=3, **kw)
    f0 = m.render(engine=4, **kw)
    f1 = m.render(engine=1, **kw)
    torch.cuda.synchronize()
    m.check_health()
    flipped = (f3["alpha"] - f1["alpha"]).abs() > 0.05
    e = float((f3["tex_fg"] - f1["tex_fg"]).abs().amax(0)[~flipped].max())
    flipped0 = (f0["alpha"] - f1["alpha"]).abs() > 0.05   # (rays on the final-sample step flip independently per engine)
    e0 = float((f0["tex_fg"] - f1["tex_fg"]).abs().amax(0)[~flipped0].max())
    print(f"vseq 256^2x96 frame vs fp32 engine: max rgb err {e:.2e} (engine 4: {e0:.2e}), flipped {float(flipped.float().mean()):.4%}")
    assert e < 1e-3 and float(flipped.float().mean()) < 0.01
