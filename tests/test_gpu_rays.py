"""Explicit ray batches on the GPU (kpn_render_rays / kpn_camera_rays, RayMarcher.render_rays / camera_rays,
KeypointNeRF.render_rays).

The lattice render marches the rays camera_rays returns, so render_rays of any subset, order or concatenation of them equals
render at those pixels bit for bit, in every plane, on every engine.  The fixtures of tests/golden/make_golden_rays.py (the
reference's eval branch on an orthographic bundle and on a shuffled two-camera batch) pin the values, with the gates of
tests/test_gpu_parity.py.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from keypointnerf_b200 import _lib as L
from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.renderer import RayMarcher
from keypointnerf_b200.testing import build_model, scene_tensors
from oracle import kpnerf_oracle as O  # checker only
from tests import test_gpu_parity as P
from tests.rays_util import RAY_CASES, load_rays_case
from tests.util import checksum, load_golden, scene_from_meta, target_wh

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
_NETS = {}


def _bound(scene, weights, n_kpt, target=None):
    """(model, marcher with the scene bound, scene tensors); one model per weight set."""
    key = (n_kpt, id(weights))
    if key not in _NETS:
        _NETS.clear()
        _NETS[key] = build_model(weights, n_kpt, DEV)
    net = _NETS[key]
    a = scene_tensors(scene, target if target is not None else syn.make_target(8), DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    return net, m, a


def _lattice(meta, target, a):
    step = 2 ** (meta["level"] - 1)
    w, h = target_wh(meta)
    return dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=target["znear"], zfar=target["zfar"], x0=meta["x_off"],
                y0=meta["y_off"], step=step, nx=w // step, ny=h // step)


def _flat(res, idx=None):
    """render's planes as (C, R) / (R,) / (R, S) per-ray arrays, at the rays idx."""
    out = {}
    for k, v in res.items():
        v = v.reshape(3, -1) if k.startswith("tex_fg") else (v if k in ("contrib", "z_fine") else v.reshape(-1))
        if idx is not None:
            v = v[..., idx] if k.startswith("tex_fg") else v[idx]
        out[k] = v
    return out


def _assert_bits(rays_res, ref):
    assert set(rays_res) == set(ref)
    for k, v in rays_res.items():
        assert torch.equal(v.view(torch.int32), ref[k].contiguous().view(torch.int32)), k


@pytest.fixture(scope="module", params=["tiny", "rect", "rect_v4_k17", "tiny_v4_k32"])
def lattice_case(request):
    g, meta, sha = load_golden(request.param)
    scene, weights, target = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    return g, meta, scene, weights, target


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_round_trip_equals_render(lattice_case, engine):
    """render_rays(camera_rays(T)) == render(T) bit for bit: debug outputs, early-ray termination, z_fine_override."""
    g, meta, scene, weights, target = lattice_case
    net, m, a = _bound(scene, weights, meta["n_kpt"], target)
    lat = _lattice(meta, target, a)
    o, d, nf = m.camera_rays(**lat)
    kw = dict(S_c=meta["S_c"], S_f=meta["S_f"], fine=True, engine=engine)
    for extra in (dict(debug=True), dict(ert_eps=1e-3), dict(z_fine_override=torch.from_numpy(g["z_fine"]).to(DEV))):
        ref = _flat(m.render(**lat, **kw, **extra))
        _assert_bits(m.render_rays(o, d, nf, **kw, **extra), ref)
    torch.cuda.synchronize()
    assert float(ref["alpha"].max()) > 0.05


def test_camera_rays_are_the_oracle_rays(lattice_case):
    g, meta, scene, weights, target = lattice_case
    net, m, a = _bound(scene, weights, meta["n_kpt"], target)
    lat = _lattice(meta, target, a)
    o, d, nf = (t.cpu() for t in m.camera_rays(**lat))
    pix = O.pixel_lattice(lat["nx"] * lat["step"], lat["ny"] * lat["step"], lat["step"], lat["x0"], lat["y0"])
    oo, dd, n_r, f_r = O.ray_setup(pix, target["K"], target["RT"], float(target["znear"]), float(target["zfar"]))
    assert float((o - oo).abs().max()) < 1e-5 and float((d - dd).abs().max()) < 1e-6
    assert float((nf - torch.cat([n_r, f_r], -1)).abs().max()) < 1e-5
    oh, dh, nfh = m.camera_rays(**dict(lat, K=a["cam_tar"]["K"].cpu(), RT=a["cam_tar"]["RT"].cpu()))   # host path
    assert not oh.is_cuda and torch.equal(oh, o) and torch.equal(dh, d) and torch.equal(nfh, nf)


def _subset_scene():
    g, meta, _ = load_golden("rect")
    scene, weights, target = scene_from_meta(meta)
    return g, meta, scene, weights, target


def test_subsets_and_orders_equal_render():
    g, meta, scene, weights, _ = _subset_scene()
    target = syn.make_target(size=48, width=48, height=32, azimuth=meta["azimuth"], zoom=2.0)   # the box covers part of the image
    net, m, a = _bound(scene, weights, meta["n_kpt"], target)
    lat = _lattice(meta, target, a)
    o, d, nf = m.camera_rays(**lat)
    R = o.shape[0]
    kw = dict(S_c=meta["S_c"], S_f=meta["S_f"], fine=True, debug=True)
    gen = torch.Generator().manual_seed(3)
    pix = O.pixel_lattice(lat["nx"] * lat["step"], lat["ny"] * lat["step"], lat["step"], lat["x0"], lat["y0"])
    oo, dd, _, _ = O.ray_setup(pix, target["K"], target["RT"], 2.0, 5.0)
    at_box = O.ray_bbox(scene["bounds"], oo, dd)[2][:, 0]            # mask_at_box: the pixels whose ray meets the bounds
    subsets = {"random mask": torch.nonzero(torch.rand(R, generator=gen) < 0.3)[:, 0], "mask_at_box": torch.nonzero(at_box)[:, 0],
               "permutation": torch.randperm(R, generator=gen), "one ray": torch.tensor([R // 2 + 3])}
    assert 0 < len(subsets["mask_at_box"]) < R
    for engine in (0, 1):
        ref = _flat(m.render(**lat, **kw, engine=engine))
        for name, idx in subsets.items():
            i = idx.to(DEV)
            _assert_bits(m.render_rays(o[i], d[i], nf[i], **kw, engine=engine), _flat(ref, i))


def test_batch_of_several_chunks_equals_render():
    """300 000 rays x 128 coarse samples is more than one 32 Mi-sample chunk: the second chunk reads the inputs at an offset."""
    scene = syn.make_scene(src_size=128, n_kpt=18, fg_mode="hull")
    weights = syn.make_weights(18)
    target = syn.make_target(size=640, width=640, height=480, azimuth=1.3, zoom=2.0)
    net, m, a = _bound(scene, weights, 18, target)
    lat = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=640, ny=480)
    o, d, nf = m.camera_rays(**lat)
    ref = _flat(m.render(**lat, S_c=128))
    perm = torch.randperm(o.shape[0], generator=torch.Generator().manual_seed(1))[:300000].to(DEV)
    _assert_bits(m.render_rays(o[perm], d[perm], nf[perm], S_c=128), _flat(ref, perm))
    assert m.stats()["samples_valid"] > 0 and float(ref["alpha"].max()) > 0.05


def test_two_cameras_in_one_batch_equal_two_renders():
    g, meta, scene, weights, target = _subset_scene()
    net, m, a = _bound(scene, weights, meta["n_kpt"], target)
    kw = dict(S_c=16, S_f=16, fine=True)
    parts, refs = [], []
    for az, (w, h) in ((1.0, (40, 24)), (2.6, (24, 32))):
        t = syn.make_target(size=w, width=w, height=h, azimuth=az, zoom=3.0)
        lat = dict(K=torch.from_numpy(t["K"]).to(DEV), RT=torch.from_numpy(t["RT"]).to(DEV), znear=2.0, zfar=5.0, x0=0, y0=0, step=1,
                   nx=w, ny=h)
        parts.append(m.camera_rays(**lat))
        refs.append(_flat(m.render(**lat, **kw)))
    res = m.render_rays(*(torch.cat(x, 0) for x in zip(*parts)), **kw)
    for k, v in res.items():
        cat = torch.cat([refs[0][k], refs[1][k]], -1)
        assert torch.equal(v, cat), k
    assert float(refs[1]["alpha"].max()) > 0.05


@pytest.fixture(scope="module", params=RAY_CASES)
def rays_case(request):
    return load_rays_case(request.param)


def _fixture_render(rays_case, engine, **kw):
    g, meta, scene, weights, o, d, nf = rays_case
    net, m, a = _bound(scene, weights, meta["n_kpt"])
    r = m.render_rays(o.to(DEV), d.to(DEV), nf.to(DEV), S_c=meta["S_c"], S_f=meta["S_f"], fine=True, engine=engine, **kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in r.items()}


@pytest.mark.parametrize("engine", [0, 1])
def test_coarse_matches_reference(rays_case, engine):
    g = rays_case[0]
    r = _fixture_render(rays_case, engine, debug=True)
    t, rep = P.TOL[engine], []
    good = P.check(rep, "tex_fg", r["tex_fg"], g["tex_fg"], P.ALL, t["rgb"])
    good &= P.check(rep, "alpha", r["alpha"], g["alpha"], P.ALL, t["alpha"])
    good &= P.check(rep, "contrib", r["contrib"], g["contrib_coarse"], P.ALL, t["contrib"])
    good &= P.check(rep, "depth", r["depth"], g["depth"], P.ALL, t["depth"])
    p = P.masked_psnr(r["tex_fg"], g["tex_fg"], P.ALL)
    print(f"rays coarse engine {engine}: " + "; ".join(rep) + f"; psnr {p:.1f} dB")
    assert good and p > t["psnr"], rep


@pytest.mark.parametrize("engine", [0, 1])
def test_fine_with_reference_depths(rays_case, engine):
    g = rays_case[0]
    r = _fixture_render(rays_case, engine, z_fine_override=torch.from_numpy(g["z_fine"]))
    t, rep = P.TOL[engine], []
    good = P.check(rep, "tex_fg_fine", r["tex_fg_fine"], g["tex_fg_fine"], P.ALL, t["rgb"])
    good &= P.check(rep, "alpha_fine", r["alpha_fine"], g["alpha_fine"], P.ALL, t["alpha"])
    good &= P.check(rep, "sdf", r["sdf"], g["sdf"], P.ALL, t["sdf"])
    good &= P.check(rep, "depth_fine", r["depth_fine"], g["depth_fine"], P.ALL, t["depth"])
    print(f"rays fine@ref-z engine {engine}: " + "; ".join(rep))
    assert good, rep


@pytest.mark.parametrize("engine", [0, 1])
def test_fine_free_running(rays_case, engine):
    g = rays_case[0]
    r = _fixture_render(rays_case, engine, debug=True)
    dz = np.abs(r["z_fine"] - g["z_fine"])
    e = np.abs(r["tex_fg_fine"] - g["tex_fg_fine"]).reshape(-1)
    p = P.masked_psnr(r["tex_fg_fine"], g["tex_fg_fine"], P.ALL)
    print(f"rays fine free engine {engine}: z q99 {np.quantile(dz, 0.99):.2e} rgb q99 {np.quantile(e, 0.99):.2e} psnr {p:.1f}")
    assert np.quantile(dz, 0.99) < 1e-3 and p > 50.0 and np.quantile(e, 0.99) < P.TOL[engine]["q99_fine"]


def test_validity_is_exact_on_random_rays():
    """samples_valid of a random ray batch (origins around the box, random directions, random near/far) equals the oracle's
    count of valid coarse and fine samples exactly."""
    scene = syn.make_scene(src_size=128, n_kpt=18, fg_mode="hull", fg_hole=True)
    weights = syn.make_weights(18)
    net, m, a = _bound(scene, weights, 18)
    gen = torch.Generator().manual_seed(7)
    n = 4000
    b = torch.from_numpy(scene["bounds"]).reshape(2, 3)
    o = b[0] - 0.5 + (b[1] - b[0] + 1.0) * torch.rand(n, 3, generator=gen)
    tgt = b.mean(0) + 0.3 * torch.randn(n, 3, generator=gen)
    d = torch.nn.functional.normalize(tgt - o, dim=-1)
    nf = torch.stack([0.5 * torch.rand(n, generator=gen), 2.0 + 3.0 * torch.rand(n, generator=gen)], -1)
    S_c, S_f = 24, 16
    r = m.render_rays(o.to(DEV), d.to(DEV), nf.to(DEV), S_c=S_c, S_f=S_f, fine=True, engine=1, debug=True)
    got = m.stats()["samples_valid"]
    near, far, hit = O.ray_bbox(scene["bounds"], o, d)
    n_r, f_r = O.clip_near_far(nf[:, :1], nf[:, 1:], near, far, hit)
    want = 0
    for zz in (O.coarse_z(n_r, f_r, S_c), r["z_fine"].cpu()):
        xy, zc = O.project(scene, (o[:, None] + d[:, None] * zz[..., None]).reshape(-1, 3))
        want += int(O.validity(scene, xy, zc).sum())
    print(f"random rays: valid samples {got} (oracle {want})")
    assert got == want and want > 0


def test_host_path_errors_and_refusals():
    g, meta, scene, weights, o, d, nf = load_rays_case("rays_mixed")
    net, m, a = _bound(scene, weights, meta["n_kpt"])
    kw = dict(S_c=meta["S_c"], S_f=meta["S_f"], fine=True, debug=True)
    dev = m.render_rays(o.to(DEV), d.to(DEV), nf.to(DEV), **kw)
    host = m.render_rays(o.pin_memory(), d.pin_memory(), nf.pin_memory(), **kw)   # host in, host out
    mixed = m.render_rays(o, d, nf, out_device="cuda", **kw)                       # host in, device out
    for k in dev:
        assert not host[k].is_cuda and torch.equal(host[k], dev[k].cpu()) and torch.equal(mixed[k], dev[k]), k
    empty = m.render_rays(o[:0].to(DEV), d[:0].to(DEV), nf[:0].to(DEV), **kw)
    assert empty["tex_fg"].shape == (3, 0) and empty["alpha"].shape == (0,) and empty["contrib"].shape == (0, meta["S_c"])
    # null arrays: KPN_ERR_ARG
    rays = L.KpnRays()
    rays.n, rays.mem = 4, L.KPN_MEM_DEVICE
    op, out = L.KpnOpts(), L.KpnOut()
    op.sample_per_ray_c = 8
    rc = m.lib.kpn_render_rays(m.ctx, C.byref(rays), C.byref(op), C.byref(out), m._stream())
    assert rc == -1
    with pytest.raises(L.KpnError, match="status -1"):
        L.check(m.lib, m.ctx, rc, "kpn_render_rays")
    # no scene: KPN_ERR_STATE
    fresh = RayMarcher(0)
    with pytest.raises(L.KpnError, match="status -3"):
        fresh.render_rays(o.to(DEV), d.to(DEV), nf.to(DEV), S_c=8)
    fresh.close()
    # a two-view scene on the default engine: render's refusal
    s2 = syn.make_scene(src_size=64, n_views=2, n_kpt=18, fg_mode="hull")
    w2 = syn.make_weights(18)
    _, m2, a2 = _bound(s2, w2, 18)
    with pytest.raises(L.KpnError, match="request engine = 1"):
        m2.render_rays(o[:64].to(DEV), d[:64].to(DEV), nf[:64].to(DEV), S_c=8, engine=0)
    with pytest.raises(L.KpnError, match="request engine = 1"):
        m2.render(K=a2["cam_tar"]["K"], RT=a2["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=8, ny=8, S_c=8, engine=0)


def test_model_api_on_the_mixed_batch():
    g, meta, scene, weights, o, d, nf = load_rays_case("rays_mixed")
    net = build_model(weights, meta["n_kpt"], DEV)
    a = scene_tensors(scene, syn.make_target(8), DEV)
    cfg = dict(sample_per_ray_c=meta["S_c"], sample_per_ray_f=meta["S_f"], fine=True, uniform=True, src_foreground_mask=a["fg"],
               bounds=a["bounds"], feat_geo=a["feat_geo"], feat_tex=a["feat_tex"])
    with torch.no_grad():
        out = net.render_rays(net, a["img"], a["cam"], o.to(DEV), d.to(DEV), nf.to(DEV), sp_data=a["sp_data"], **cfg)
    assert out["tex_fg"].shape == (3, o.shape[0]) and out["sdf"].shape == (o.shape[0],) and out["alpha"].is_cuda
    r = {k: v.cpu().numpy() for k, v in out.items()}
    t, rep = P.TOL[0], []
    good = P.check(rep, "tex_fg", r["tex_fg"], g["tex_fg"], P.ALL, t["rgb"])
    good &= P.check(rep, "alpha", r["alpha"], g["alpha"], P.ALL, t["alpha"])
    p = P.masked_psnr(r["tex_fg_fine"], g["tex_fg_fine"], P.ALL)
    print("model render_rays: " + "; ".join(rep) + f"; fine psnr {p:.1f}")
    assert good and p > 50.0, rep
    for bad in (dict(uniform=False), dict(rand_noise_std=0.1), dict(separate_cf=True)):
        with pytest.raises(NotImplementedError):
            net.render_rays(net, a["img"], a["cam"], o.to(DEV), d.to(DEV), nf.to(DEV), sp_data=a["sp_data"], **dict(cfg, **bad))
    net.marcher().check_health()


def test_zz_health_is_clean_at_the_end():
    for net in _NETS.values():
        net.marcher().check_health()
