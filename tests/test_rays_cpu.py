"""Explicit ray batches on the CPU: the ray oracle (tests/rays_oracle.py) against the reference's eval branch run on the same rays
(tests/golden/make_golden_rays.py), the lattice path of the oracle through it, and the ctypes mirror of kpn_rays."""
import os
import re

import numpy as np
import pytest
import torch

from keypointnerf_b200 import _lib as L
from keypointnerf_b200 import synthetic as syn
from oracle import kpnerf_oracle as O
from tests.rays_oracle import render_rays
from tests.rays_util import RAY_CASES, load_rays_case
from tests.util import psnr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=RAY_CASES)
def case(request):
    return load_rays_case(request.param)


def test_fixture_covers_its_edge_cases(case):
    g, meta, scene, weights, o, d, nf = case
    hit = g["hit"].astype(bool)
    assert hit.any() and not hit.all()   # rays that meet the box and rays that miss it
    assert float(g["alpha"].max()) > 0.2
    if meta["kind"] == "ortho":
        b = torch.from_numpy(scene["bounds"]).reshape(2, 3)
        inside = ((o >= b[0]) & (o <= b[1])).all(-1)
        assert int(inside.sum()) > 0 and torch.unique(d, dim=0).shape[0] == 1


def test_oracle_render_rays_coarse_matches_reference(case):
    g, meta, scene, weights, o, d, nf = case
    r = render_rays(scene, O.fold_weights(weights), o, d, nf, meta["S_c"], meta["S_f"], False)
    np.testing.assert_allclose(r["z"].numpy(), g["z_coarse"], atol=2e-6)
    np.testing.assert_allclose(r["contrib"].numpy(), g["contrib_coarse"], atol=2e-5)
    np.testing.assert_allclose(r["tex_fg"].t().numpy(), g["tex_fg"], atol=2e-5)
    np.testing.assert_allclose(r["alpha"].numpy(), g["alpha"], atol=2e-5)
    np.testing.assert_allclose(r["depth"].numpy(), g["depth"], atol=2e-4)


def test_oracle_render_rays_fine_matches_reference(case):
    g, meta, scene, weights, o, d, nf = case
    fw = O.fold_weights(weights)
    r = render_rays(scene, fw, o, d, nf, meta["S_c"], meta["S_f"], True)
    assert np.quantile(np.abs(r["z_fine"].numpy() - g["z_fine"]), 0.99) < 1e-4
    assert psnr(r["tex_fg_fine"].numpy(), g["tex_fg_fine"].T) > 60.0
    r2 = render_rays(scene, fw, o, d, nf, meta["S_c"], meta["S_f"], True, z_fine_override=g["z_fine"])
    np.testing.assert_allclose(r2["tex_fg_fine"].t().numpy(), g["tex_fg_fine"], atol=3e-5)
    np.testing.assert_allclose(r2["alpha_fine"].numpy(), g["alpha_fine"], atol=3e-5)
    np.testing.assert_allclose(r2["sdf"].numpy(), g["sdf"], atol=2e-4)
    np.testing.assert_allclose(r2["depth_fine"].numpy(), g["depth_fine"], atol=3e-4)


def test_render_pixels_is_render_rays_of_the_lattice_rays():
    scene = syn.make_scene(src_size=64, n_kpt=18, fg_mode="hull", fg_hole=True)
    fw = O.fold_weights(syn.make_weights(18))
    target = syn.make_target(size=24, azimuth=2.0, zoom=2.0, width=24, height=16)
    pix = O.pixel_lattice(24, 16, 1, 0, 0)[torch.randperm(24 * 16, generator=torch.Generator().manual_seed(0))[:200]]
    a = O.render_pixels(scene, fw, target, pix, 12, 8, True)
    o, d, n_r, f_r = O.ray_setup(pix, target["K"], target["RT"], float(target["znear"]), float(target["zfar"]))
    b = render_rays(scene, fw, o.expand(d.shape[0], 3), d, torch.cat([n_r, f_r], -1), 12, 8, True)
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert float(a["alpha"].max()) > 0.1


def test_kpn_rays_ctypes_mirror_matches_header():
    header = open(os.path.join(ROOT, "include", "kpnerf_b200.h")).read()
    body = re.search(r"typedef struct \{((?:(?!typedef struct).)*?)\} kpn_rays;", header, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [re.findall(r"(\w+)\s*$", s.strip())[0] for s in body.split(";") if s.strip()]
    assert names == [f[0] for f in L.KpnRays._fields_] == ["origins", "dirs", "near_far", "n", "mem"]
    assert L.KpnRays.n.size == 8 and L.KpnRays.mem.size == 4
    assert {"kpn_render_rays", "kpn_camera_rays"} <= set(L.EXPORTS)
