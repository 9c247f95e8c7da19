"""CPU checks of the mesh path: the committed case table is what tools/gen_mc_table.py generates and makes closed, consistently
wound meshes (through the numpy restatement of the kernels, tests/mesh_ref.py), the KpnGrid mirror matches the header, and the
grid helpers follow the documented formulas."""
import math

import numpy as np
import pytest
import torch

from keypointnerf_b200 import _lib as L
from keypointnerf_b200.model import KeypointNeRF
from tests import mesh_ref as M
from tests.test_host_abi import _header_fields


def test_table_header_is_generated():
    gen = M.mc_table_module()
    assert open(gen.HEADER).read() == gen.render(gen.table())


def test_table_cuts_shared_faces_identically():
    """The segments a case puts on a cube face depend only on that face's four corners, so the cells on both sides agree."""
    gen = M.mc_table_module()
    for fi, (ring, n) in enumerate(gen.FACES):
        other = gen.FACES[fi ^ 1][0]   # the opposite face: the neighbour cell's copy of this face, shifted by one cell
        for bits in range(16):
            case_a = sum(((bits >> i) & 1) << ring[i] for i in range(4))
            case_b = sum(((bits >> i) & 1) << other[i] for i in range(4))
            sa = {frozenset(gen.EDGES[e]) for seg in gen.face_segments(case_a, ring, n) for e in seg}
            sb = {frozenset(gen.EDGES[e]) for seg in gen.face_segments(case_b, other, -n) for e in seg}
            shift = 1 << (fi >> 1)
            sb = {frozenset(c ^ shift for c in s) for s in sb}
            assert sa == sb


def _closed_random(rng, shape):
    f = rng.standard_normal(shape).astype(np.float32)
    f[0] = f[-1] = -1.0
    f[:, 0] = f[:, -1] = -1.0
    f[:, :, 0] = f[:, :, -1] = -1.0
    return f


def test_numpy_marching_cubes_is_closed_and_manifold():
    rng = np.random.default_rng(0)
    for _ in range(150):
        s = rng.integers(3, 9, 3)
        f = _closed_random(rng, tuple(int(x) for x in s))
        v, fa = M.marching_cubes(f, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 0.0)
        if len(fa):
            assert M.is_closed_manifold(fa)
    # every case of one cell inside a closed box
    for case in range(256):
        f = np.full((4, 4, 4), -1.0, np.float32)
        for c in range(8):
            f[1 + (c >> 2), 1 + ((c >> 1) & 1), 1 + (c & 1)] = 1.0 if (case >> c) & 1 else -1.0
        _, fa = M.marching_cubes(f, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 0.0)
        assert len(fa) == 0 or M.is_closed_manifold(fa), case


def test_numpy_sphere_topology_and_orientation():
    n = 32
    g = np.linspace(-1, 1, n, dtype=np.float32)
    Z, Y, X = np.meshgrid(g, g, g, indexing="ij")
    f = (0.7 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32)
    h = 2.0 / (n - 1)
    v, fa = M.marching_cubes(f, (-1.0, -1.0, -1.0), (h, h, h), 0.0)
    assert M.is_closed_manifold(fa) and M.euler(v, fa) == 2
    vol = M.signed_volume(v, fa)
    assert vol > 0 and abs(vol / (4 / 3 * math.pi * 0.7 ** 3) - 1) < 0.02


def test_kpn_grid_mirror_matches_header():
    assert _header_fields("kpn_grid") == [f[0] for f in L.KpnGrid._fields_]


def test_mesh_grid_dims_and_origin():
    bounds = torch.tensor([[-0.5, -1.0, -0.25], [0.5, 1.0, 0.35]])
    origin, spacing, dims = KeypointNeRF.mesh_grid(bounds, 129)
    h = 2.0 / 128
    assert origin == pytest.approx((-0.5, -1.0, -0.25)) and spacing == pytest.approx((h, h, h))
    assert dims == (65, 129, math.ceil(0.6 / h - 1e-6) + 1)
    # the longest axis has exactly `resolution` points; every axis covers its extent
    for e, n in zip((1.0, 2.0, 0.6), dims):
        assert (n - 1) * h >= e - 1e-9 and (n - 2) * h < e
    with pytest.raises(ValueError):
        KeypointNeRF.mesh_grid(bounds, 1)


def test_grid_point_formula():
    origin, spacing, dims = (0.1, -0.3, 2.5), (0.013, 0.007, 0.021), (7, 5, 3)
    P = M.grid_points(origin, spacing, dims)
    assert P.shape == (3, 5, 7, 3) and P.dtype == np.float32
    for (k, j, i) in [(0, 0, 0), (2, 4, 6), (1, 3, 2)]:
        for a, idx in enumerate((i, j, k)):
            want = np.float32(np.float32(origin[a]) + np.float32(np.float32(spacing[a]) * np.float32(idx)))
            assert P[k, j, i, a] == want
    # grid id = (k ny + j) nx + i: x fastest
    flat = P.reshape(-1, 3)
    assert np.array_equal(flat[(2 * 5 + 4) * 7 + 6], P[2, 4, 6])


def test_numpy_vertex_order_and_interpolation():
    f = np.array([[[0.0, 2.0], [2.0, 2.0]], [[2.0, 2.0], [2.0, 2.0]]], np.float32)   # only corner (0,0,0) outside
    v, fa = M.marching_cubes(f, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 1.0)
    assert np.array_equal(v, np.array([[0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5]], np.float32))
    assert fa.shape == (1, 3)
    # seen from the outside corner (f <= level) the triangle is counter-clockwise: its normal points at the corner
    a, b, c = v[fa[0]]
    assert np.dot(np.cross(b - a, c - a), -a) > 0


# ---- the reference's query at grid points (tests/golden/make_golden_grid.py) ----------------------------------------------
@pytest.mark.parametrize("name", ["grid_tiny", "grid_rect_v4_k17", "grid_v2"])
def test_oracle_meets_grid_goldens(name):
    """The oracle's query at the golden grid points meets the reference's [sdf_raw, rad] under the geo_out tolerance of
    test_oracle_golden.py, with the same validity; the seeded inputs are the ones the golden run used."""
    from oracle import kpnerf_oracle as O
    from tests.util import checksum, load_golden, scene_from_meta
    g, meta, sha = load_golden(name)
    scene, weights, _ = scene_from_meta(meta)
    assert checksum(scene, weights) == sha, "seeded inputs drifted from the ones the golden run used"
    gr = meta["grid"]
    pts = torch.from_numpy(M.grid_points(gr["origin"], gr["spacing"], gr["dims"]).reshape(-1, 3))
    view = torch.zeros_like(pts)
    view[:, 2] = 1.0
    out, valid = O.query(scene, O.fold_weights(weights), pts, view)
    assert np.array_equal(valid.numpy(), g["grid_valid"])
    assert 0.05 < g["grid_valid"].mean() < 0.95
    np.testing.assert_allclose(out[:, :2].numpy(), g["grid_out"], atol=2e-3, rtol=1e-4)
