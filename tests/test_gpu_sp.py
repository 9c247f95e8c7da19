"""The spatial-encoding parameters (sp_args.sp_level / scale / sigma) and one / two source views on the GPU.

Goldens from the unmodified reference (tests/golden/make_golden_sp.py): one and two views (tiny_v1, tiny_v2, rect_v2_k17,
cfg2_pass_v2 at config size), every sp_level other than 3 (tiny_L0_k32, tiny_L2, tiny_L4_k24: the widest layer-0 input the fp32
engine holds, tiny_v2_L1), scale / sigma other than 1 / 0.1 (tiny_sig), a large |scale * dz| (tiny_dz: scale 100, the sin / cos
arguments span ~120 periods) and sigma left out of the config (tiny_nosigma: the reference's default of 150).  Only the
fp32 engine (engine 1) renders fewer than 3 views or sp_level != 3; the 3-view scale / sigma fixtures also run on the
tensor-core engine (engines 0 and 2).  They go through the parity tests and gates of tests/test_gpu_parity.py.

Besides: a sweep of every sp_level 0-4 with every view count 1-4 against the CPU oracle, per-sample errors against the fp64 oracle
at three (scale, sigma) settings, batch independence with 1 and 2 views, the model API, the refusals, and weights changed while
a scene is bound.
"""
import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200._lib import KpnError
from keypointnerf_b200.config import default_cfg
from keypointnerf_b200.model import KeypointNeRF
from keypointnerf_b200.renderer import RayMarcher
from keypointnerf_b200.testing import build_model, scene_tensors
from oracle import kpnerf_oracle as O  # checker only
from tests import test_gpu_parity as P
from tests.test_gpu_coverage import GATE
from tests.test_gpu_kpt import _valid_count
from tests.util import checksum, load_golden, psnr, scene_from_meta, sp_from_meta, target_wh

pytestmark = pytest.mark.gpu

TINY = ["tiny_v1", "tiny_v2", "rect_v2_k17", "tiny_L0_k32", "tiny_L2", "tiny_L4_k24", "tiny_v2_L1", "tiny_sig", "tiny_dz",
        "tiny_nosigma"]
TC_CASES = ["tiny_sig", "tiny_dz", "tiny_nosigma"]   # 3 views, sp_level 3: the tensor-core engine covers them
CASE_ENGINES = [(n, 1) for n in TINY] + [(n, e) for n in TC_CASES for e in (0, 2)]


def _golden_case(name):
    g, meta, sha = load_golden(name)
    scene, weights, target = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    assert scene["img"].shape[0] == meta["n_views"]
    net = build_model(weights, meta["n_kpt"], "cuda:0", sp_args=sp_from_meta(meta)[0])
    return g, meta, scene, weights, target, net


_CASES = {}


def _case(name):
    if name not in _CASES:
        _CASES.clear()   # one fixture's model at a time
        _CASES[name] = _golden_case(name)
    return _CASES[name]


@pytest.mark.parametrize("name,engine", CASE_ENGINES)
def test_query_matches_reference(name, engine):
    P.test_query_matches_reference(_case(name), engine)


@pytest.mark.parametrize("name,engine", CASE_ENGINES)
def test_tile_coarse_matches_reference(name, engine):
    P.test_tile_coarse_matches_reference(_case(name), engine)


@pytest.mark.parametrize("name,engine", CASE_ENGINES)
def test_tile_fine_with_reference_depths(name, engine):
    P.test_tile_fine_with_reference_depths(_case(name), engine)


@pytest.mark.parametrize("name,engine", CASE_ENGINES)
def test_tile_fine_free_running(name, engine):
    P.test_tile_fine_free_running(_case(name), engine)


def test_config_size_pass_with_2_views():
    """One strided pass of BASELINE config 2 (512^2 sources, 128 samples) with 2 views on the fp32 engine, every ray under the
    config-size gates."""
    P.test_config_size_pass_matches_reference("cfg2_pass_v2", 1)


def _first_seed_with_content(scene, target, pix, S_c, S_f, n_kpt, sp_level, sp):
    for seed in range(26, 46):
        weights = syn.make_weights(n_kpt, seed=seed, sp_level=sp_level)
        ref = O.render_pixels(scene, O.fold_weights(weights), target, pix, S_c, S_f, True, sp)
        if float(ref["alpha"].max()) > 0.05:
            return weights, ref
    raise AssertionError("no seed gives a frame with content")


@pytest.mark.parametrize("n_views", [1, 2, 3, 4])
@pytest.mark.parametrize("sp_level", [0, 1, 2, 3, 4])
def test_every_sp_level_and_view_count_against_oracle(sp_level, n_views):
    """A 16 x 16 pixel frame of a silhouette-mask scene with 18 keypoints, 12 coarse + 8 fine samples, for every sp_level and view
    count on the fp32 engine: it shades exactly the samples the oracle finds valid, and meets the parity gates on the coarse image
    and compositing weights and on the fine image rendered at the oracle's resampled depths.  The weights are the first seed from
    26 on whose frame is not empty."""
    n_kpt, S_c, S_f, n = 18, 12, 8, 16
    sp = {"sp_level": sp_level, "scale": 1.0, "sigma": 0.1}
    scene = syn.make_scene(src_size=64, n_views=n_views, n_kpt=n_kpt, fg_mode="hull")
    target = syn.make_target(size=n, zoom=2.0)
    pix = O.pixel_lattice(n, n, 1, 0, 0)
    weights, ref = _first_seed_with_content(scene, target, pix, S_c, S_f, n_kpt, sp_level, sp)
    want = _valid_count(scene, target, pix, ref["z"]) + _valid_count(scene, target, pix, ref["z_fine"])
    assert want > 0
    net = build_model(weights, n_kpt, "cuda:0", sp_args=sp)
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    img = lambda v: v.reshape(n, n, 3).permute(2, 0, 1).numpy()
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=float(target["znear"]), zfar=float(target["zfar"]), x0=0, y0=0,
              step=1, nx=n, ny=n, S_c=S_c, S_f=S_f, fine=True, engine=1)
    r = m.render(debug=True, **kw)
    r2 = m.render(z_fine_override=ref["z_fine"], **kw)
    got = m.stats()["samples_valid"]
    torch.cuda.synchronize()
    t = P.TOL[1]
    rep = []
    good = P.check(rep, "tex_fg", r["tex_fg"].cpu().numpy(), img(ref["tex_fg"]), P.ALL, t["rgb"])
    good &= P.check(rep, "contrib", r["contrib"].cpu().numpy(), ref["contrib"].numpy(), P.ALL, t["contrib"])
    good &= P.check(rep, "tex_fg_fine@oracle-z", r2["tex_fg_fine"].cpu().numpy(), img(ref["tex_fg_fine"]), P.ALL, t["rgb"])
    good &= P.check(rep, "alpha_fine@oracle-z", r2["alpha_fine"].cpu().numpy(), ref["alpha_fine"].reshape(n, n).numpy(), P.ALL,
                    t["alpha"])
    print(f"sp_level {sp_level}, {n_views} views: valid {got} (oracle {want}); " + "; ".join(rep))
    assert got == want and good, rep


def _pool(scene, n=40000, seed=5):
    """Points the oracle finds valid in ``scene`` (a box around the keypoints and gaussian clouds around them) and directions."""
    rng = np.random.default_rng(seed)
    kpt = scene["kpt3d"][0]
    cand = np.concatenate([rng.uniform([-0.5, -1.0, -0.5], [0.5, 1.0, 0.5], (60000, 3)),
                           kpt[rng.integers(0, len(kpt), 12000)] + rng.normal(0.0, 0.015, (12000, 3))]).astype(np.float32)
    view = rng.normal(size=cand.shape)
    view = (view / np.linalg.norm(view, axis=-1, keepdims=True)).astype(np.float32)
    xy, z = O.project(scene, torch.from_numpy(cand))
    idx = rng.permutation(np.flatnonzero(O.validity(scene, xy, z).numpy()))[:n]
    return cand[idx], view[idx]


# (scale, sigma, dz_scale) of the per-sample checks: the default, tiny_sig and tiny_dz
SP_PARAMS = {"default": (1.0, 0.1, 1.0), "sig": (2.5, 0.25, 1.0), "dz": (100.0, 0.15, 100.0)}


@pytest.fixture(scope="module", params=list(SP_PARAMS))
def sp_pool(request):
    """The bench scene (512^2 sources, 3 views, 18 keypoints) bound with weights for one (scale, sigma), 40k valid points, and the
    oracle's outputs on them in fp64 and fp32."""
    scale, sigma, dz_scale = SP_PARAMS[request.param]
    sp = {"sp_level": 3, "scale": scale, "sigma": sigma}
    scene = syn.make_scene(src_size=512, n_kpt=18)
    weights = syn.make_weights(18, dz_scale=dz_scale)
    target = syn.make_target(size=512)
    net = build_model(weights, 18, "cuda:0", sp_args=sp)
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    pts, view = _pool(scene)
    fw = O.fold_weights(weights)
    ref32, _ = O.query(scene, fw, torch.from_numpy(pts), torch.from_numpy(view), sp)
    with O.precision(torch.float64):
        ref, valid = O.query(scene, O.fold_weights(weights), torch.from_numpy(pts), torch.from_numpy(view), sp)
    assert bool(valid.all())
    return request.param, m, torch.from_numpy(pts).cuda(), torch.from_numpy(view).cuda(), ref.numpy(), ref32.numpy()


def _errors(out, ref):
    err = np.abs(np.asarray(out, np.float64) - ref)
    return {"sdf": float(err[:, 0].max()), "rad": float(err[:, 1].max()), "rgb": float(err[:, 2:].max())}


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_query_against_fp64_oracle(sp_pool, engine):
    """Per-sample error of each engine against the fp64 oracle under the gates of test_gpu_coverage, at the default (scale,
    sigma), at tiny_sig's and at tiny_dz's.  At scale 100 fp32 arithmetic itself is further from the exact encoding (the
    camera-space depth's round-off times scale * 4 pi), so there each gate is widened by twice the fp32 oracle's own distance from
    the fp64 oracle on the same points; at the other two settings the gates are unchanged."""
    name, m, pts, view, ref, ref32 = sp_pool
    out, valid = m.query(pts, view, engine=engine)
    assert bool(valid.all())
    err = _errors(out.cpu().numpy(), ref)
    d32 = _errors(ref32, ref)
    gate = {k: GATE[engine][k] + (2.0 * d32[k] if name == "dz" else 0.0) for k in err}
    print(f"{name} engine {engine}: " + ", ".join(f"{k} {v:.2e} (gate {gate[k]:.2e})" for k, v in err.items()) +
          "; fp32 oracle: " + ", ".join(f"{k} {v:.2e}" for k, v in d32.items()))
    assert all(err[k] <= gate[k] for k in err), (err, gate)


@pytest.mark.parametrize("n_views", [1, 2])
def test_query_result_does_not_depend_on_the_batch(n_views):
    """With 1 and 2 views, the fp32 engine's query(pool[:n]) equals the first n rows of query(pool) bit for bit, for batch sizes
    around its 64-sample tile and around one and two full waves of tiles."""
    scene = syn.make_scene(src_size=256, n_views=n_views, n_kpt=18)
    weights = syn.make_weights(18)
    net = build_model(weights, 18, "cuda:0")
    a = scene_tensors(scene, syn.make_target(size=64), "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    pts, view = _pool(scene, n=30000)
    pts, view = torch.from_numpy(pts).cuda(), torch.from_numpy(view).cuda()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns = {1, 2, 63, 64, 65, 127, 128, 129}
    for k in (1, 2):
        ns |= {k * sms * 64 - 1, k * sms * 64, k * sms * 64 + 1}
    assert max(ns) <= pts.shape[0], pts.shape
    full, vfull = m.query(pts, view, engine=1)
    assert bool(vfull.all())
    bad = []
    for n in sorted(ns):
        out, valid = m.query(pts[:n], view[:n], engine=1)
        if not (torch.equal(out, full[:n]) and bool(valid.all())):
            bad.append(n)
    m.check_health()
    assert not bad, f"{n_views} views: batches of {bad} samples differ from the same samples shaded in the whole pool"


def _model_api_render(net, name, engine):
    g, meta, sha = load_golden(name)
    scene, weights, target = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    net.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in weights.items()}, strict=False)
    net = net.cuda().eval()
    net.engine = engine
    a = scene_tensors(scene, target, "cuda:0")
    with torch.no_grad():
        o = net.render_pifu_nerf(net, a["img"], a["cam"], a["cam_tar"], level=meta["level"], sp_data=a["sp_data"],
                                 feat_geo=a["feat_geo"], feat_tex=a["feat_tex"], src_foreground_mask=a["fg"], bounds=a["bounds"],
                                 mask_at_box=None, sample_per_ray_c=meta["S_c"], sample_per_ray_f=meta["S_f"], fine=True,
                                 uniform=True)
    torch.cuda.synchronize()
    w, h = target_wh(meta)
    assert o["tex_fg"].shape == (3, h, w)
    rep = []
    good = P.check(rep, "tex_fg", o["tex_fg"].cpu().numpy(), g["tex_fg"][0], P.ALL, P.TOL[engine]["rgb"])
    good &= P.check(rep, "alpha", o["alpha"].cpu().numpy()[0], g["alpha"][0], P.ALL, P.TOL[engine]["alpha"])
    p = psnr(o["tex_fg_fine"].cpu().numpy(), g["tex_fg_fine"][0])
    print(f"{name} through the model API, engine {engine}: " + "; ".join(rep) + f"; fine psnr {p:.1f} dB")
    assert good and p > 50.0, rep


def test_sp_level_2_through_the_model_api():
    """KeypointNeRF(cfg) with sp_args.sp_level = 2 and net.engine = 1 renders tiny_L2 through render_pifu_nerf and matches the
    reference's own images of that frame."""
    cfg = default_cfg(18)
    cfg["models"]["KeypointNeRF"]["sp_args"]["sp_level"] = 2
    net = KeypointNeRF(cfg)
    assert net.mlp_geo.layers1.layers[0].linear.weight_v.shape == (128, 5 * 18 + 64)
    _model_api_render(net, "tiny_L2", 1)


def test_config_without_sigma_through_the_model_api():
    """A config whose sp_args has no sigma takes the reference's default of 150 and matches tiny_nosigma on the default
    (tensor-core) engine."""
    cfg = default_cfg(18)
    del cfg["models"]["KeypointNeRF"]["sp_args"]["sigma"]
    net = KeypointNeRF(cfg)
    assert net.engine == 0
    _model_api_render(net, "tiny_nosigma", 0)


def test_refusals():
    """sp_level != 3 on the tensor-core engine says to request engine = 1; sp_level 5 and a layer-0 input wider than the fp32
    engine's 288-float rows (sp_level 4 with 25 keypoints: 9 * 25 + 64 = 289) are refused when the weights are set."""
    scene = syn.make_scene(src_size=64, n_kpt=18)
    target = syn.make_target(size=16)
    a = scene_tensors(scene, target, "cuda:0")
    net = build_model(syn.make_weights(18, sp_level=2), 18, "cuda:0", sp_args={"sp_level": 2})
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=16, ny=16, S_c=8)
    with pytest.raises(KpnError, match="engine = 1"):
        m.render(**kw)
    m.render(engine=1, **kw)
    torch.cuda.synchronize()
    for n_kpt, level in ((18, 5), (25, 4)):
        net = build_model(syn.make_weights(n_kpt, sp_level=level), n_kpt, "cuda:0", sp_args={"sp_level": level})
        with pytest.raises(KpnError, match=f"status -4: sp_level={level} unsupported"):
            net.marcher()
    # the widest accepted input: sp_level 4 with 24 keypoints (280 floats)
    build_model(syn.make_weights(24, sp_level=4), 24, "cuda:0", sp_args={"sp_level": 4}).marcher()


# ---- weights changed while a scene is bound (RayMarcher / C ABI callers; KeypointNeRF re-binds after every weight change) ----
def _bind(m, a):
    c = a["cam"]
    m.set_scene(KRT=c["KRT"], extrin=a["sp_data"]["extrin"], kpt3d=a["sp_data"]["kpt3d"].reshape(-1, 3), bounds=a["bounds"],
                feat64=a["feat_geo"][0], feat8=a["feat_geo"][1], feat_tex=a["feat_tex"], img=a["img"], fg=a["fg"],
                width=c["width"], height=c["height"], znear=c["znear"], zfar=c["zfar"], nml_scale=c["nml_scale"])


def _stale_setup():
    scene = syn.make_scene(src_size=64, n_kpt=18, fg_mode="hull")
    target = syn.make_target(size=32, zoom=2.0)
    a = scene_tensors(scene, target, "cuda:0")
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=0, y0=0, step=1, nx=32, ny=32, S_c=12, S_f=8,
              fine=True, debug=True)
    return a, kw


STALE = [  # (first weights' sp args, second weights' sp args, engine)
    (dict(sp_level=3, sp_scale=1.0, sp_sigma=0.1), dict(sp_level=3, sp_scale=1.0, sp_sigma=0.25), 0),
    (dict(sp_level=3, sp_scale=1.0, sp_sigma=0.1), dict(sp_level=3, sp_scale=1.0, sp_sigma=0.25), 1),
    (dict(sp_level=3, sp_scale=1.0, sp_sigma=0.1), dict(sp_level=3, sp_scale=2.5, sp_sigma=0.1), 0),
    (dict(sp_level=3, sp_scale=1.0, sp_sigma=0.1), dict(sp_level=3, sp_scale=2.5, sp_sigma=0.1), 1),
    (dict(sp_level=3, sp_scale=1.0, sp_sigma=0.1), dict(sp_level=2, sp_scale=1.0, sp_sigma=0.1), 1),
    (dict(sp_level=2, sp_scale=1.0, sp_sigma=0.1), dict(sp_level=4, sp_scale=1.0, sp_sigma=0.1), 1),
]


@pytest.mark.parametrize("first,second,engine", STALE)
def test_new_sp_args_reach_a_bound_scene(first, second, engine):
    """set_weights -> set_scene -> set_weights with another sigma, scale or sp_level, then render: the frame is bit-identical to
    one rendered after binding the scene afresh with the new weights, and differs from the frame of the first weights."""
    a, kw = _stale_setup()
    w1 = syn.make_weights(18, sp_level=first["sp_level"])
    w2 = syn.make_weights(18, sp_level=second["sp_level"])
    fresh = RayMarcher(0)
    fresh.set_weights(w2, 18, **second)
    _bind(fresh, a)
    want = fresh.render(engine=engine, **kw)
    m = RayMarcher(0)
    m.set_weights(w1, 18, **first)
    _bind(m, a)
    old = m.render(engine=engine, **kw)
    m.set_weights(w2, 18, **second)
    got = m.render(engine=engine, **kw)
    torch.cuda.synchronize()
    assert float(want["alpha"].max()) > 0.05
    assert not torch.equal(old["tex_fg"], want["tex_fg"])
    for k in want:
        assert torch.equal(got[k], want[k]), k


def test_new_keypoint_count_unbinds_the_scene():
    """Weights for another keypoint count can not use the bound scene's keypoints: render and query fail with KPN_ERR_STATE
    until a scene is bound again, which then renders like a fresh context."""
    a, kw = _stale_setup()
    m = RayMarcher(0)
    m.set_weights(syn.make_weights(18), 18)
    _bind(m, a)
    m.render(**kw)
    m.set_weights(syn.make_weights(17), 17)
    with pytest.raises(KpnError, match="status -3"):
        m.render(**kw)
    with pytest.raises(KpnError, match="status -3"):
        m.query(torch.zeros(4, 3, device="cuda"), torch.ones(4, 3, device="cuda"))
    s17 = syn.make_scene(src_size=64, n_kpt=17, fg_mode="hull")
    a17 = scene_tensors(s17, syn.make_target(size=32, zoom=2.0), "cuda:0")
    _bind(m, a17)
    got = m.render(**kw)
    fresh = RayMarcher(0)
    fresh.set_weights(syn.make_weights(17), 17)
    _bind(fresh, a17)
    want = fresh.render(**kw)
    torch.cuda.synchronize()
    for k in want:
        assert torch.equal(got[k], want[k]), k
