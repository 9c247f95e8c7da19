"""Spatial-encoding parameters and one / two source views on the CPU: the oracle against the goldens of the unmodified reference
(tests/golden/make_golden_sp.py) at the tolerances of tests/test_oracle_golden.py, in fp32 and in fp64, and the seeded weights'
handling of sp_level."""
import hashlib

import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model
from oracle import kpnerf_oracle as O
from tests.test_oracle_golden import check_query_stages, check_tile_coarse, check_tile_fine
from tests.util import checksum, load_golden, scene_from_meta, sp_from_meta

TINY = ["tiny_v1", "tiny_v2", "rect_v2_k17", "tiny_L0_k32", "tiny_L2", "tiny_L4_k24", "tiny_v2_L1", "tiny_sig", "tiny_dz",
        "tiny_nosigma"]


def load_case(name):
    g, meta, sha = load_golden(name)
    scene, weights, target = scene_from_meta(meta)
    assert checksum(scene, weights) == sha, "seeded inputs drifted from the ones the golden run used"
    assert scene["img"].shape[0] == meta["n_views"]
    return g, meta, scene, weights, target


@pytest.fixture(scope="module", params=TINY)
def case(request):
    return load_case(request.param)


def test_query_stages_match_reference(case):
    sp = sp_from_meta(case[1])[1]
    assert case[0]["enc"].shape[-1] == (1 + 2 * sp["sp_level"]) * case[1]["n_kpt"]
    check_query_stages(case, sp=sp)


def test_tile_coarse_matches_reference(case):
    check_tile_coarse(case, sp=sp_from_meta(case[1])[1])


def test_tile_fine_matches_reference(case):
    check_tile_fine(case, sp=sp_from_meta(case[1])[1])


@pytest.mark.parametrize("name", [n for n in TINY if n != "tiny_dz"])
def test_fp64_oracle_meets_the_same_tolerances(name):
    """The fp64 oracle (the yardstick of the GPU per-sample tests) meets the same tolerances, with the f8 exception of
    tests/test_oracle_golden.py.  tiny_dz is held to the bounds of the next test instead."""
    case = load_case(name)
    sp = sp_from_meta(case[1])[1]
    with O.precision(torch.float64):
        check_query_stages(case, f8_atol=3e-5, sp=sp)
        check_tile_coarse(case, sp=sp)
        check_tile_fine(case, sp=sp)


def test_fp64_oracle_with_large_scale():
    """tiny_dz (scale 100): the reference's fp32 encoding is less well conditioned there.  The camera-space depths carry fp32
    round-off of ~2e-7 m, which scale * pi * 2^l turns into ~2.5e-4 of the level-2 sin / cos values, and the product
    dz * float(pi 2^l) (|y| up to ~750) adds its own rounding.  The fp32 oracle repeats that arithmetic and meets the usual
    tolerances (above); the fp64 oracle computes the exact encoding and differs from the reference by the reference's own
    round-off.  Measured on this fixture: encoding 2.5e-4, x_view 7.1e-5, geometry output 3.5e-4, per-sample rgb 1.8e-6, coarse
    rgb 1.3e-5, alpha 2.1e-5, compositing weights 3.4e-5, fine rgb / alpha at the reference's depths 5.7e-6 / 8.9e-6.  Bounds are
    2x those, or the usual tolerance where that is larger."""
    g, meta, scene, weights, target = load_case("tiny_dz")
    sp = sp_from_meta(meta)[1]
    e = lambda a, b: float(np.abs(np.asarray(a, np.float64) - b).max())
    with O.precision(torch.float64):
        fw = O.fold_weights(weights)
        out, valid, parts = O.query(scene, fw, torch.from_numpy(g["query_pts"]), torch.from_numpy(g["query_view"]), sp,
                                    return_parts=True)
        sel, v = g["sel"], g["query_valid"]
        assert np.array_equal(valid.numpy(), v)
        assert e(parts["enc"].numpy()[:, sel], g["enc"]) < 5e-4
        assert e(parts["x_view"].numpy()[:, sel], g["x_view"]) < 1.5e-4
        assert e(out[:, :2].numpy(), g["geo_out"]) < 2e-3
        assert e(out[:, 2:].numpy()[v], g["ibr_rgb"][v]) < 2e-4
        r = O.render_tile(scene, fw, target, meta["level"], meta["x_off"], meta["y_off"], meta["S_c"], meta["S_f"], True, sp)
        assert e(r["tex_fg"].numpy(), g["tex_fg"][0]) < 3e-5
        assert e(r["alpha"].numpy(), g["alpha"][0]) < 4.5e-5
        assert e(r["contrib"].numpy(), g["contrib_coarse"]) < 7e-5
        r2 = O.render_tile(scene, fw, target, meta["level"], meta["x_off"], meta["y_off"], meta["S_c"], meta["S_f"], True, sp,
                           z_fine_override=g["z_fine"])
        assert e(r2["tex_fg_fine"].numpy(), g["tex_fg_fine"][0]) < 3e-5
        assert e(r2["alpha_fine"].numpy(), g["alpha_fine"][0]) < 3e-5


def test_config_size_pass_with_2_views_matches_reference():
    """cfg2_pass_v2: one strided pass of BASELINE config 2 with 2 views, oracle against the reference."""
    g, meta, scene, weights, target = load_case("cfg2_pass_v2")
    r = O.render_tile(scene, O.fold_weights(weights), target, meta["level"], meta["x_off"], meta["y_off"], meta["S_c"],
                      meta["S_f"], meta["fine"], sp_from_meta(meta)[1])
    np.testing.assert_allclose(r["tex_fg"].numpy(), g["tex_fg"][0], atol=2e-5)
    np.testing.assert_allclose(r["alpha"].numpy(), g["alpha"][0], atol=2e-5)
    np.testing.assert_allclose(r["contrib"].numpy(), g["contrib_coarse"], atol=2e-5)


def test_fixtures_cover_what_they_claim():
    """Every fixture has content (alpha > 0.05); the large-|scale * dz| fixture really wraps its sin / cos arguments many periods;
    the sigma-less fixture leaves sigma out of the config."""
    for name in TINY + ["cfg2_pass_v2"]:
        g, meta, _ = load_golden(name)
        assert float(g["alpha"].max()) > 0.05, name
    g, meta, scene, weights, target = load_case("tiny_dz")
    v = g["query_valid"]
    pts = torch.from_numpy(g["query_pts"][v])
    E = torch.from_numpy(scene["extrin"]).double()
    kpt = torch.from_numpy(scene["kpt3d"][0]).double()
    zc = (pts.double() @ E[:, 2, :3].T + E[:, 2, 3])           # (N,V) camera depths of the samples
    zk = kpt @ E[:, 2, :3].T + E[:, 2, 3]                       # (K,V) camera depths of the keypoints
    arg = np.pi * 4 * meta["scale"] * (zc[:, None] - zk[None]).abs()   # the level-2 argument
    assert float(arg.median()) > 20 * 2 * np.pi and float(arg.max()) > 100 * 2 * np.pi
    _, meta, _ = load_golden("tiny_nosigma")
    assert meta["sigma"] is None and "sigma" not in syn.sp_args(18, sigma=None)


def test_default_weights_are_unchanged():
    """sp_level / dz_scale default to the values every earlier fixture used: the default weights keep their bytes (these digests
    are those of the generator before it took sp_level), and sp_level only changes layer 0's input width."""
    want = {5: "621ba290c18435b3", 18: "6445e64b5f79e5f7", 24: "c96ee17c915c5d2c", 32: "5bcd1f57f408e8e0"}
    for n_kpt, digest in want.items():
        for w in (syn.make_weights(n_kpt), syn.make_weights(n_kpt, sp_level=3, dz_scale=1.0)):
            h = hashlib.sha256()
            for k in sorted(w):
                h.update(np.ascontiguousarray(w[k]).tobytes())
            assert h.hexdigest()[:16] == digest, n_kpt
    assert syn.layer_table(18) == syn.layer_table(18, 3)
    for level in range(5):
        t = syn.layer_table(24, level)
        assert t[0][2] == (1 + 2 * level) * 24 + 64 and t[1:] == syn.layer_table(24)[1:]
        w = syn.make_weights(24, sp_level=level)
        assert w["mlp_geo.layers1.layers.0.linear.weight_v"].shape == (128, (1 + 2 * level) * 24 + 64)
    assert syn.sp_args(18) == {"sp_level": 3, "sp_type": "rel_z_decay", "scale": 1.0, "sigma": 0.1, "n_kpt": 18}
    with pytest.raises(ValueError):
        syn.sp_args(18, sp_type="z")


def test_dz_scale_divides_the_dz_columns_only():
    a = syn.make_weights(18)
    b = syn.make_weights(18, dz_scale=1000.0)
    name = "mlp_geo.layers1.layers.0.linear."
    va, vb = a[name + "weight_v"], b[name + "weight_v"]
    np.testing.assert_allclose(vb[:, :18] * 1000.0, va[:, :18], rtol=1e-6)
    assert np.array_equal(vb[:, 18:], va[:, 18:])
    assert np.allclose(b[name + "weight_g"][:, 0], np.linalg.norm(vb.astype(np.float64), axis=1), rtol=1e-6)
    assert all(np.array_equal(a[k], b[k]) for k in a if not k.startswith(name + "weight"))


def test_oracle_sp_level_0_is_the_dz_row():
    """sp_level 0: the encoding is the decayed dz row alone, equal to the first row of any other level's encoding."""
    scene = syn.make_scene(src_size=64, n_kpt=7)
    pts = torch.from_numpy(np.random.default_rng(0).uniform(-0.3, 0.3, (50, 3)).astype(np.float32))
    e0 = O.encode_rel_z_decay(scene, pts, 0)
    e3 = O.encode_rel_z_decay(scene, pts, 3)
    assert e0.shape == (3, 50, 7) and e3.shape == (3, 50, 49)
    assert torch.equal(e0, e3[..., :7])


def test_model_config_carries_the_sp_args():
    """testing.build_model with sp_args overrides builds the layer-0 width of that level, and a config without sigma takes the
    reference's default of 150 (what KeypointNeRF.marcher() hands to kpn_set_weights)."""
    pytest.importorskip("torch")
    w = syn.make_weights(24, sp_level=4)
    net = build_model(w, 24, "cpu", sp_args={"sp_level": 4, "scale": 2.5, "sigma": 0.25})
    sp = net.sp_encoder
    assert (sp.sp_level, sp.scale, sp.kwargs["sigma"]) == (4, 2.5, 0.25)
    assert net.mlp_geo.layers1.layers[0].linear.weight_v.shape == (128, 280)
    net = build_model(syn.make_weights(18), 18, "cpu", sp_args={"sigma": None})
    assert "sigma" not in net.sp_encoder.kwargs and net.sp_encoder.kwargs.get("sigma", 150.0) == 150.0
