"""Four source views on the tensor-core engine (engines 0 and 2-4) and the fp32 engine (engine 1).

Goldens from the unmodified reference: tiny_v4 (18 keypoints, every intermediate), rect_v4_k17 (four cameras and 17 keypoints,
the Human3.6M shape: non-square sources and target, level 2 with offsets), tiny_v4_k32 (one warpgroup per geometry-front CTA,
the widest layer 0) and cfg2_pass_v4 (config size).  They run through the same parity tests and gates as the three-view
fixtures (tests/test_gpu_parity.py).  A sweep over every keypoint count 1..32 against the CPU oracle reaches every 4-view
front-kernel instantiation.
"""
import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200._lib import KpnError
from keypointnerf_b200.config import default_cfg
from keypointnerf_b200.model import KeypointNeRF
from keypointnerf_b200.testing import build_model, scene_tensors
from oracle import kpnerf_oracle as O  # checker only
from tests import test_gpu_parity as P
from tests.test_gpu_coverage import GATE
from tests.test_gpu_kpt import _valid_count
from tests.util import COLOUR_WGS, TAIL_WGS, checksum, front_wgs, load_golden, psnr, target_wh, tile_samples

pytestmark = pytest.mark.gpu

ENGINES = [0, 1]
# samples per tile with 4 views and warpgroups per CTA (one CTA per SM) of the geometry front kernel at 18 keypoints, the density
# tail and the colour kernel
TILE_ROWS = tile_samples(4)
WGS = (front_wgs(18), TAIL_WGS, COLOUR_WGS)


def scene_from_meta_views(meta):
    """Seeded scene, weights and target of a fixture with ``meta["n_views"]`` source views."""
    scene = syn.make_scene(src_size=meta["src_size"], n_views=meta["n_views"], n_kpt=meta["n_kpt"], seed=meta["scene_seed"],
                           fg_hole=meta["fg_hole"], fg_mode=meta.get("fg_mode", "ones"), src_height=meta.get("src_height"))
    weights = syn.make_weights(meta["n_kpt"], seed=meta["w_seed"])
    w, h = target_wh(meta)
    target = syn.make_target(size=meta["tgt_size"], azimuth=meta["azimuth"], zoom=meta.get("zoom", 1.0), width=w, height=h)
    return scene, weights, target


def _golden_case(name):
    g, meta, sha = load_golden(name)
    assert meta["n_views"] == 4
    scene, weights, target = scene_from_meta_views(meta)
    assert scene["img"].shape[0] == 4
    assert checksum(scene, weights) == sha
    return g, meta, scene, weights, target, build_model(weights, meta["n_kpt"], "cuda:0")


@pytest.fixture(scope="module", params=["tiny_v4", "rect_v4_k17", "tiny_v4_k32"])
def case(request):
    return _golden_case(request.param)


@pytest.mark.parametrize("engine", ENGINES)
def test_query_matches_reference(case, engine):
    P.test_query_matches_reference(case, engine)


@pytest.mark.parametrize("engine", ENGINES)
def test_tile_coarse_matches_reference(case, engine):
    P.test_tile_coarse_matches_reference(case, engine)


@pytest.mark.parametrize("engine", ENGINES)
def test_tile_fine_with_reference_depths(case, engine):
    P.test_tile_fine_with_reference_depths(case, engine)


@pytest.mark.parametrize("engine", ENGINES)
def test_tile_fine_free_running(case, engine):
    P.test_tile_fine_free_running(case, engine)


@pytest.mark.parametrize("engine", ENGINES)
def test_config_size_pass_with_4_views(engine):
    """One strided pass of BASELINE config 2 (512^2 sources, 128 samples) with 4 views against the reference's own output of that
    pass, every ray under the config-size gates (RGB 1e-3 on the tensor-core engine)."""
    g, meta, scene, weights, target, net = _golden_case("cfg2_pass_v4")
    r = P._render_tile(net, meta, scene, target, engine=engine, debug=True)
    t = P.TOL[engine]
    rep = []
    good = P.check(rep, "tex_fg", r["tex_fg"], g["tex_fg"][0], P.ALL, t["rgb"])
    good &= P.check(rep, "alpha", r["alpha"], g["alpha"][0], P.ALL, t["alpha"])
    good &= P.check(rep, "depth", r["depth"], g["depth"][0], P.ALL, t["depth"])
    good &= P.check(rep, "contrib", r["contrib"], g["contrib_coarse"], P.ALL, t["contrib"])
    p = psnr(r["tex_fg"], g["tex_fg"][0])
    print(f"cfg2_pass_v4 engine {engine}: " + "; ".join(rep) + f"; psnr (all rays) {p:.1f} dB")
    assert good and p > t["psnr"], rep


@pytest.mark.parametrize("n_kpt", range(1, 33))
def test_every_keypoint_count_against_oracle(n_kpt):
    """A 16 x 16 pixel frame of a 4-view silhouette-mask scene, 12 coarse + 8 fine samples, for every keypoint count: both engines
    shade exactly the samples the oracle finds valid, and meet the parity gates on the coarse image and compositing weights and
    on the fine image rendered at the oracle's resampled depths.  The weights are the first seed from 26 on whose frame is not
    empty."""
    scene = syn.make_scene(src_size=64, n_views=4, n_kpt=n_kpt, fg_mode="hull")
    target = syn.make_target(size=16, zoom=2.0)
    S_c, S_f, n = 12, 8, 16
    pix = O.pixel_lattice(n, n, 1, 0, 0)
    for seed in range(26, 36):
        weights = syn.make_weights(n_kpt, seed=seed)
        ref = O.render_pixels(scene, O.fold_weights(weights), target, pix, S_c, S_f, True)
        if float(ref["alpha"].max()) > 0.05:
            break
    assert float(ref["alpha"].max()) > 0.05, "no seed gives a frame with content"
    want = _valid_count(scene, target, pix, ref["z"]) + _valid_count(scene, target, pix, ref["z_fine"])
    assert want > 0
    net = build_model(weights, n_kpt, "cuda:0")
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    img = lambda v: v.reshape(n, n, 3).permute(2, 0, 1).numpy()
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=float(target["znear"]), zfar=float(target["zfar"]), x0=0, y0=0,
              step=1, nx=n, ny=n, S_c=S_c, S_f=S_f, fine=True)
    for engine in ENGINES:
        r = m.render(debug=True, engine=engine, **kw)
        r2 = m.render(z_fine_override=ref["z_fine"], engine=engine, **kw)
        got = m.stats()["samples_valid"]
        torch.cuda.synchronize()
        t = P.TOL[engine]
        rep = []
        good = P.check(rep, "tex_fg", r["tex_fg"].cpu().numpy(), img(ref["tex_fg"]), P.ALL, t["rgb"])
        good &= P.check(rep, "contrib", r["contrib"].cpu().numpy(), ref["contrib"].numpy(), P.ALL, t["contrib"])
        good &= P.check(rep, "tex_fg_fine@oracle-z", r2["tex_fg_fine"].cpu().numpy(), img(ref["tex_fg_fine"]), P.ALL, t["rgb"])
        good &= P.check(rep, "alpha_fine@oracle-z", r2["alpha_fine"].cpu().numpy(), ref["alpha_fine"].reshape(n, n).numpy(), P.ALL,
                        t["alpha"])
        print(f"4 views, n_kpt {n_kpt} engine {engine}: valid {got} (oracle {want}); " + "; ".join(rep))
        assert got == want and good, rep


@pytest.fixture(scope="module")
def bench4():
    """The bench scene (512^2 sources, all-ones masks, 18 keypoints) with 4 views, and 40k points the oracle finds valid (enough
    for two persistent waves of every kernel): a box around the keypoints and gaussian clouds around them."""
    scene = syn.make_scene(src_size=512, n_views=4, n_kpt=18)
    weights = syn.make_weights(18)
    target = syn.make_target(size=512)
    net = build_model(weights, 18, "cuda:0")
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    rng = np.random.default_rng(5)
    kpt = scene["kpt3d"][0]
    cand = np.concatenate([rng.uniform([-0.5, -1.0, -0.5], [0.5, 1.0, 0.5], (60000, 3)),
                           kpt[rng.integers(0, len(kpt), 12000)] + rng.normal(0.0, 0.015, (12000, 3))]).astype(np.float32)
    view = rng.normal(size=cand.shape)
    view = (view / np.linalg.norm(view, axis=-1, keepdims=True)).astype(np.float32)
    xy, z = O.project(scene, torch.from_numpy(cand))
    idx = rng.permutation(np.flatnonzero(O.validity(scene, xy, z).numpy()))[:40000]
    pts, view = cand[idx], view[idx]
    with O.precision(torch.float64):
        ref, valid = O.query(scene, O.fold_weights(weights), torch.from_numpy(pts), torch.from_numpy(view))
    assert bool(valid.all()), "the pool holds only points the oracle finds valid"
    return m, a, torch.from_numpy(pts).cuda(), torch.from_numpy(view).cuda(), ref.numpy()


def _batch_sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns = {1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65}
    for rows, wgs in zip(TILE_ROWS, WGS):
        wave = sms * wgs * rows   # one full persistent wave of the kernel
        ns |= {wave - 1, wave, wave + 1, 2 * wave + 1}
    return sorted(ns)


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_query_result_does_not_depend_on_the_batch(bench4, engine):
    """At 4 views, query(pool[:n]) equals the first n rows of query(pool) bit for bit, for batch sizes around the front tile (16)
    and the colour tile (32) and around one and two full persistent waves of each kernel."""
    m, a, pts, view, ref = bench4
    assert max(_batch_sizes()) <= pts.shape[0], pts.shape
    full, _ = m.query(pts, view, engine=engine)
    bad = []
    for n in _batch_sizes():
        assert n <= pts.shape[0]
        out, valid = m.query(pts[:n], view[:n], engine=engine)
        if not (torch.equal(out, full[:n]) and bool(valid.all())):
            bad.append(n)
    m.check_health()
    assert not bad, f"engine {engine}: batches of {bad} samples differ from the same samples shaded in the whole pool"


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_query_against_fp64_oracle(bench4, engine):
    """Per-sample error of each engine at 4 views against the fp64 oracle, under the 3-view gates of test_gpu_coverage."""
    m, a, pts, view, ref = bench4
    out, valid = m.query(pts, view, engine=engine)
    assert bool(valid.all())
    out = out.cpu().numpy().astype(np.float64)
    err = {k: float(np.abs(out[:, c] - ref[:, c]).max()) for k, c in (("sdf", slice(0, 1)), ("rad", slice(1, 2)),
                                                                      ("rgb", slice(2, 5)))}
    print(f"4 views, engine {engine}: " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert all(err[k] <= GATE[engine][k] for k in err), (err, GATE[engine])


def test_engine_aliases_are_bit_identical(bench4):
    """At 4 views, engines 3 and 4 run the same kernels as engine 0."""
    m, a, pts, view, ref = bench4
    o0, v0 = m.query(pts, view, engine=0)
    for engine in (3, 4):
        o, v = m.query(pts, view, engine=engine)
        assert torch.equal(o, o0) and torch.equal(v, v0), engine
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=1, y0=2, step=4, nx=128, ny=128, S_c=32, S_f=32,
              fine=True, debug=True)
    f0 = m.render(engine=0, **kw)
    for engine in (3, 4):
        f = m.render(engine=engine, **kw)
        for k in f0:
            assert torch.equal(f[k], f0[k]), (engine, k)


def test_17_keypoints_and_4_views_through_the_model_api():
    """KeypointNeRF(cfg) with sp_args.n_kpt = 17 renders rect_v4_k17 (four source images) through render_pifu_nerf on the default
    (tensor-core) engine and matches the reference's own images of that frame."""
    g, meta, sha = load_golden("rect_v4_k17")
    scene, weights, target = scene_from_meta_views(meta)
    assert checksum(scene, weights) == sha
    net = KeypointNeRF(default_cfg(17))
    net.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in weights.items()}, strict=False)
    net = net.cuda().eval()
    assert net.engine == 0
    a = scene_tensors(scene, target, "cuda:0")
    assert a["img"].shape[0] == 4
    w, h = target_wh(meta)
    with torch.no_grad():
        o = net.render_pifu_nerf(net, a["img"], a["cam"], a["cam_tar"], level=meta["level"], sp_data=a["sp_data"],
                                 feat_geo=a["feat_geo"], feat_tex=a["feat_tex"], src_foreground_mask=a["fg"], bounds=a["bounds"],
                                 mask_at_box=None, sample_per_ray_c=meta["S_c"], sample_per_ray_f=meta["S_f"], fine=True,
                                 uniform=True)
    torch.cuda.synchronize()
    assert o["tex_fg"].shape == (3, h, w)
    # the golden holds one strided pass (level 2, offset (1, 1)): the frame's pixels of that lattice phase
    step = 2 ** (meta["level"] - 1)
    sub = (slice(None), slice(meta["y_off"], None, step), slice(meta["x_off"], None, step))
    rep = []
    good = P.check(rep, "tex_fg", o["tex_fg"].cpu().numpy()[sub], g["tex_fg"][0], P.ALL, P.TOL[0]["rgb"])
    good &= P.check(rep, "alpha", o["alpha"].cpu().numpy()[sub], g["alpha"][0], P.ALL, P.TOL[0]["alpha"])
    p = psnr(o["tex_fg_fine"].cpu().numpy()[sub], g["tex_fg_fine"][0])
    print("17 keypoints, 4 views through the model API: " + "; ".join(rep) + f"; fine psnr {p:.1f} dB")
    assert good and p > 50.0, rep


def test_view_count_refusals_and_health():
    """5 views are refused with KPN_ERR_UNSUPPORTED on every engine; 1 view on the tensor-core engine says to request
    engine = 1, which renders it; the device watchdog is clean after the 4-view runs of this module."""
    weights = syn.make_weights(18)
    net = build_model(weights, 18, "cuda:0")
    target = syn.make_target(size=16, azimuth=1.0)
    s5 = syn.make_scene(src_size=64, n_views=5, n_kpt=18, src_azimuths=(0.0, 2.1, 4.2, 5.25, 1.0))
    a5 = scene_tensors(s5, target, "cuda:0")
    with pytest.raises(KpnError, match=r"status -4: n_views=5 unsupported \(1\.\.4\)"):
        net._bind_scene(a5["cam"], a5["feat_geo"], a5["feat_tex"], a5["sp_data"], a5["img"], a5["fg"], a5["bounds"])
    s1 = syn.make_scene(src_size=64, n_views=1, n_kpt=18)
    a1 = scene_tensors(s1, target, "cuda:0")
    m1 = net._bind_scene(a1["cam"], a1["feat_geo"], a1["feat_tex"], a1["sp_data"], a1["img"], a1["fg"], a1["bounds"])
    kw = dict(K=a1["cam_tar"]["K"], RT=a1["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=16, ny=16, S_c=8)
    with pytest.raises(KpnError, match="engine = 1"):
        m1.render(**kw)
    r1 = m1.render(engine=1, **kw)
    torch.cuda.synchronize()
    ref1 = O.render_pixels(s1, O.fold_weights(weights), target, O.pixel_lattice(16, 16, 1, 0, 0), 8)
    assert np.abs(r1["tex_fg"].cpu().numpy().reshape(3, -1).T - ref1["tex_fg"].numpy()).max() < 1e-4
    m1.check_health()
