"""Four source views on the CPU: the oracle against the 4-view goldens of the unmodified reference (tests/golden/
make_golden_views.py) at the tolerances of tests/test_oracle_golden.py, and the seeded scenes' view handling."""
import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from oracle import kpnerf_oracle as O
from tests.test_gpu_views import scene_from_meta_views
from tests.test_oracle_golden import check_tile_coarse, check_tile_fine
from tests.util import checksum, load_golden


@pytest.fixture(scope="module", params=["tiny_v4", "rect_v4_k17", "tiny_v4_k32"])
def case(request):
    g, meta, sha = load_golden(request.param)
    assert meta["n_views"] == 4
    scene, weights, target = scene_from_meta_views(meta)
    assert checksum(scene, weights) == sha, "seeded inputs drifted from the ones the golden run used"
    return g, meta, scene, weights, target


def test_query_stages_match_reference(case):
    """Every captured per-sample intermediate of the 4-view query, at the tolerances of the 3-view fixtures."""
    g, meta, scene, weights, target = case
    out, valid, parts = O.query(scene, O.fold_weights(weights), torch.from_numpy(g["query_pts"]),
                                torch.from_numpy(g["query_view"]), return_parts=True)
    sel = g["sel"]
    assert parts["pw"].shape[0] == 4
    assert np.array_equal(valid.numpy(), g["query_valid"])
    np.testing.assert_allclose(parts["pw"][..., 0].numpy(), g["pw"], atol=2e-6)
    np.testing.assert_allclose(parts["f64"].numpy()[:, sel], g["f64"], atol=1e-5)
    np.testing.assert_allclose(parts["f8"].numpy()[:, sel], g["f8"], atol=1e-5)
    np.testing.assert_allclose(parts["enc"].numpy()[:, sel], g["enc"], atol=2e-5)
    np.testing.assert_allclose(parts["x_view"].numpy()[:, sel], g["x_view"], atol=1e-4)
    np.testing.assert_allclose(parts["x_pool"].numpy()[sel], g["x_pool"], atol=1e-4)
    np.testing.assert_allclose(out[:, :2].numpy(), g["geo_out"], atol=2e-3, rtol=1e-4)
    f = torch.cat([parts["rgb_src"], parts["tex"], parts["lat"][None].expand(4, -1, -1)], -1)
    np.testing.assert_allclose(f.permute(1, 0, 2).numpy()[sel], g["ibr_feat"], atol=1e-4)
    np.testing.assert_allclose(parts["ray_diff"].permute(1, 0, 2).numpy()[sel], g["ibr_raydiff"], atol=2e-5)
    v = g["query_valid"]
    np.testing.assert_allclose(out[:, 2:].numpy()[v], g["ibr_rgb"][v], atol=2e-4)
    np.testing.assert_allclose(out.numpy()[v], g["query_out"][v], atol=2e-3, rtol=1e-4)


def test_tile_coarse_matches_reference(case):
    check_tile_coarse(case)


def test_tile_fine_matches_reference(case):
    check_tile_fine(case)


def test_config_size_pass_matches_reference():
    """cfg2_pass_v4: one strided pass of BASELINE config 2 with 4 views, oracle against the reference."""
    g, meta, sha = load_golden("cfg2_pass_v4")
    scene, weights, target = scene_from_meta_views(meta)
    assert checksum(scene, weights) == sha
    r = O.render_tile(scene, O.fold_weights(weights), target, meta["level"], meta["x_off"], meta["y_off"], meta["S_c"],
                      meta["S_f"], meta["fine"])
    np.testing.assert_allclose(r["tex_fg"].numpy(), g["tex_fg"][0], atol=2e-5)
    np.testing.assert_allclose(r["alpha"].numpy(), g["alpha"][0], atol=2e-5)
    np.testing.assert_allclose(r["contrib"].numpy(), g["contrib_coarse"], atol=2e-5)


def test_three_view_scenes_ignore_the_fourth_azimuth():
    """The default azimuths gained a fourth entry; scenes take the first n_views of them, so a 3-view scene is byte-identical to
    one built from the three azimuths alone, and a 4-view scene's first three views are those of the 3-view scene."""
    s3 = syn.make_scene(src_size=64, n_kpt=18, fg_mode="hull")
    s3_old = syn.make_scene(src_size=64, n_kpt=18, fg_mode="hull", src_azimuths=(0.0, 2.1, 4.2))
    s4 = syn.make_scene(src_size=64, n_views=4, n_kpt=18, fg_mode="hull", src_azimuths=(0.0, 2.1, 4.2, 5.25))
    s4_default = syn.make_scene(src_size=64, n_views=4, n_kpt=18, fg_mode="hull")
    w = syn.make_weights(18)
    assert checksum(s3, w) == checksum(s3_old, w)
    assert checksum(s4, w) == checksum(s4_default, w)
    for k in ("KRT", "extrin", "fg"):
        assert np.array_equal(s4[k][:3], s3[k]), k
    assert not np.array_equal(s4["KRT"][3], s4["KRT"][0])
