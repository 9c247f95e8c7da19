"""GPU tests of the mesh path: the geometry-only grid query (kpn_query_grid) against kpn_query at the same points, marching cubes
(kpn_mesh_begin / kpn_mesh_emit) against its numpy restatement and on closed / open / degenerate fields, and
KeypointNeRF.extract_mesh end to end."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from keypointnerf_b200 import _lib as L
from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.model import KeypointNeRF
from keypointnerf_b200.renderer import RayMarcher
from keypointnerf_b200.testing import build_model, scene_tensors
from tests import mesh_ref as M
from tests.util import checksum, load_golden, scene_from_meta

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _bound(net, scene, target=None):
    a = scene_tensors(scene, target or syn.make_target(size=16), DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    return m, a


def _scene(n_views, n_kpt=18, src=64, fg_mode="hull", fg_hole=True):
    scene = syn.make_scene(src_size=src, n_views=n_views, n_kpt=n_kpt, fg_mode=fg_mode, fg_hole=fg_hole)
    net = build_model(syn.make_weights(n_kpt), n_kpt, DEV)
    return scene, net


def _grid_over(bounds, dims):
    b = np.asarray(bounds, np.float64).reshape(2, 3)
    spacing = tuple(float(x) for x in (b[1] - b[0]) / (np.array(dims) - 1))
    return tuple(float(x) for x in b[0]), spacing


def _query_points(m, pts, engine):
    p = torch.from_numpy(pts.reshape(-1, 3)).to(DEV)
    view = torch.zeros_like(p)
    view[:, 2] = 1.0
    out, valid = m.query(p, view, engine=engine)
    return out, valid


# ---- grid query ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_views", [3, 4])
@pytest.mark.parametrize("engine", [0, 1, 2])
def test_query_grid_equals_query_bitwise(n_views, engine):
    """More than 4 Mi points (several chunks and a partial one); every point's [sdf_raw, rad, valid] equals kpn_query's."""
    scene, net = _scene(n_views)
    m, _ = _bound(net, scene)
    dims = (161, 163, 165)   # 4 330 395 points
    origin, spacing = _grid_over(scene["bounds"], dims)
    out2, valid = m.query_grid(origin, spacing, dims, engine=engine)
    pts = M.grid_points(origin, spacing, dims)
    out5, valid5 = _query_points(m, pts, engine)
    torch.cuda.synchronize()
    assert valid.reshape(-1).any() and not valid.reshape(-1).all()
    assert torch.equal(valid.reshape(-1), valid5)
    assert torch.equal(out2.reshape(-1, 2), out5[:, :2])
    assert torch.all(out2.reshape(-1, 2)[~valid.reshape(-1)] == 0)


def test_query_grid_two_views_fp32_engine_and_refusal():
    scene, net = _scene(2)
    m, _ = _bound(net, scene)
    dims = (40, 41, 42)
    origin, spacing = _grid_over(scene["bounds"], dims)
    out2, valid = m.query_grid(origin, spacing, dims, engine=1)
    out5, valid5 = _query_points(m, M.grid_points(origin, spacing, dims), 1)
    assert torch.equal(valid.reshape(-1), valid5) and torch.equal(out2.reshape(-1, 2), out5[:, :2])
    with pytest.raises(L.KpnError, match="request engine = 1"):
        m.query_grid(origin, spacing, dims, engine=0)


def test_query_grid_runs_no_colour_work():
    scene, net = _scene(3)
    m, _ = _bound(net, scene)
    dims = (64, 64, 64)
    origin, spacing = _grid_over(scene["bounds"], dims)
    for engine in (0, 1):
        m.stats()
        l0 = m.stats()["kernel_launches"]
        m.query_grid(origin, spacing, dims, engine=engine)
        st = m.stats()
        grid_launches = st["kernel_launches"] - l0
        assert st["samples_total"] == 64 ** 3 and st["samples_valid"] > 0 and st["samples_coloured"] == 0
        _query_points(m, M.grid_points(origin, spacing, dims), engine)
        st2 = m.stats()
        # the tensor-core engine skips the colour work list and the colour kernel; the fp32 engine shades in one kernel
        if engine == 0:
            assert grid_launches < st2["kernel_launches"] - st["kernel_launches"]
        else:
            assert grid_launches == st2["kernel_launches"] - st["kernel_launches"]
        assert st2["samples_valid"] == st["samples_valid"]


def test_refusals():
    scene, net = _scene(3)
    m, _ = _bound(net, scene)
    lib, ctx, stream = m.lib, m.ctx, m._stream()
    op = L.KpnOpts()
    out = torch.empty(1000, device=DEV)

    def grid(o, h, n):
        g = L.KpnGrid()
        g.origin[:], g.spacing[:] = o, h
        g.nx, g.ny, g.nz = n
        return lib.kpn_query_grid(ctx, C.byref(g), out.data_ptr(), None, L.KPN_MEM_DEVICE, C.byref(op), stream)

    assert grid((0, 0, 0), (0.1, 0.1, 0.1), (4, 4, 4)) == 0
    for o, h, n in [((0, 0, 0), (0.1, 0.1, 0.1), (0, 4, 4)), ((0, 0, 0), (0.1, 0.1, 0.1), (4, -1, 4)),
                    ((0, 0, 0), (0.1, 0.0, 0.1), (4, 4, 4)), ((0, 0, 0), (0.1, 0.1, -0.1), (4, 4, 4)),
                    ((0, 0, 0), (float("nan"), 0.1, 0.1), (4, 4, 4)), ((float("inf"), 0, 0), (0.1, 0.1, 0.1), (4, 4, 4)),
                    ((0, 0, 0), (0.1, 0.1, 0.1), (2048, 2048, 1024))]:
        assert grid(o, h, n) == -1, (o, h, n)
    # the Python wrapper refuses before it allocates the outputs
    with pytest.raises(L.KpnError):
        m.query_grid((0, 0, 0), (0.1, 0.1, 0.1), (2048, 2048, 1024))
    # no scene bound
    fresh = RayMarcher(0)
    g = L.KpnGrid()
    g.spacing[:] = (0.1, 0.1, 0.1)
    g.nx = g.ny = g.nz = 4
    assert fresh.lib.kpn_query_grid(fresh.ctx, C.byref(g), out.data_ptr(), None, L.KPN_MEM_DEVICE, C.byref(op), stream) == -3
    # marching cubes: emit without begin, emit on another field, bad dims
    f = torch.zeros(4, 4, 4, device=DEV)
    o3, h3 = (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(1, 1, 1)
    v = torch.empty(64, 3, device=DEV)
    fi = torch.empty(64, 3, dtype=torch.int32, device=DEV)
    assert fresh.lib.kpn_mesh_emit(fresh.ctx, f.data_ptr(), o3, h3, v.data_ptr(), None, fi.data_ptr(), L.KPN_MEM_DEVICE, stream) == -3
    counts = (C.c_longlong * 2)()
    assert fresh.lib.kpn_mesh_begin(fresh.ctx, f.data_ptr(), 4, 4, 4, 0.5, counts, stream) == 0 and list(counts) == [0, 0]
    f2 = torch.zeros(4, 4, 4, device=DEV)
    assert fresh.lib.kpn_mesh_emit(fresh.ctx, f2.data_ptr(), o3, h3, v.data_ptr(), None, fi.data_ptr(), L.KPN_MEM_DEVICE, stream) == -3
    assert fresh.lib.kpn_mesh_begin(fresh.ctx, f.data_ptr(), 0, 4, 4, 0.5, counts, stream) == -1
    assert fresh.lib.kpn_mesh_begin(fresh.ctx, f.data_ptr(), 2048, 2048, 1024, 0.5, counts, stream) == -1
    # a failed begin forgets the previous one
    assert fresh.lib.kpn_mesh_emit(fresh.ctx, f.data_ptr(), o3, h3, v.data_ptr(), None, fi.data_ptr(), L.KPN_MEM_DEVICE, stream) == -3
    fresh.close()


# ---- marching cubes ----------------------------------------------------------------------------------------------------
def _coords(n, lo=-1.0, hi=1.0):
    h = (hi - lo) / (n - 1)
    P = torch.from_numpy(M.grid_points((lo, lo, lo), (h, h, h), (n, n, n))).to(DEV)
    return P[..., 0], P[..., 1], P[..., 2], (lo, lo, lo), (h, h, h)


def _sphere(n, r=0.6, c=(0.0, 0.0, 0.0)):
    X, Y, Z, o, h = _coords(n)
    return r - torch.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2), o, h


def _torus(n, R=0.55, r=0.2):
    X, Y, Z, o, h = _coords(n)
    q = torch.sqrt(X ** 2 + Y ** 2) - R
    return r - torch.sqrt(q ** 2 + Z ** 2), o, h


def _two_spheres(n):
    a, o, h = _sphere(n, 0.3, (-0.45, 0.0, 0.0))
    b, _, _ = _sphere(n, 0.3, (0.45, 0.1, 0.0))
    return torch.maximum(a, b), o, h


def _smoothed_random(n):
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(3)
    f = gaussian_filter(rng.standard_normal((n, n, n)), 2.0).astype(np.float32)
    f[0], f[-1], f[:, 0], f[:, -1], f[:, :, 0], f[:, :, -1] = (-1.0,) * 6
    h = 2.0 / (n - 1)
    return torch.from_numpy(f).to(DEV), (-1.0, -1.0, -1.0), (h, h, h)


def _mc(field, o, h, level=0.0, normals=True):
    m = RayMarcher(0)
    try:
        v, f, nrm = m.marching_cubes(field, o, h, level, normals=normals)
        torch.cuda.synchronize()
    finally:
        m.close()
    return v, f, nrm


def _check_against_numpy(field, o, h, level, faces_too=True):
    v, f, nrm = _mc(field, o, h, level)
    vr, fr = M.marching_cubes(field.cpu().numpy(), o, h, level) if faces_too else (None, None)
    if not faces_too:
        vr = _numpy_vertices(field.cpu().numpy(), o, h, level)
    v = v.cpu().numpy()
    assert v.shape == vr.shape
    assert np.all(np.abs(v - vr) <= 1e-6 * np.asarray(h, np.float32))
    if faces_too:
        assert np.array_equal(f.cpu().numpy(), fr)
    return v, f.cpu().numpy().astype(np.int64), nrm.cpu().numpy()


def _numpy_vertices(f, o, h, level):
    ins = f > np.float32(level)
    nz, ny, nx = f.shape
    cross = np.zeros((nz, ny, nx, 3), bool)
    cross[:, :, :-1, 0] = ins[:, :, :-1] != ins[:, :, 1:]
    cross[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    cross[:-1, :, :, 2] = ins[:-1] != ins[1:]
    pid, ax = np.nonzero(cross.reshape(-1, 3))
    k, j, i = np.unravel_index(pid, (nz, ny, nx))
    idx = np.stack([i, j, k], 1)
    idxb = idx + np.eye(3, dtype=np.int64)[ax]
    fa, fb = f[k, j, i], f[idxb[:, 2], idxb[:, 1], idxb[:, 0]]
    t = ((np.float32(level) - fa) / (fb - fa)).astype(np.float32)
    P = lambda a, n: (np.float32(o[a]) + (np.float32(h[a]) * n.astype(np.float32)).astype(np.float32)).astype(np.float32)
    v = np.stack([P(a, idx[:, a]) for a in range(3)], 1)
    sel = np.arange(len(ax))
    pb = P(0, idxb[sel, 0]) * (ax == 0) + P(1, idxb[sel, 1]) * (ax == 1) + P(2, idxb[sel, 2]) * (ax == 2)
    v[sel, ax] = v[sel, ax] + t * (pb.astype(np.float32) - v[sel, ax])
    return v


@pytest.mark.parametrize("kind,chi", [("sphere", 2), ("torus", 0), ("two_spheres", 4), ("random", None)])
def test_closed_fields(kind, chi):
    field, o, h = {"sphere": _sphere, "torus": _torus, "two_spheres": _two_spheres, "random": _smoothed_random}[kind](48)
    v, f, nrm = _check_against_numpy(field, o, h, 0.0)
    assert M.is_closed_manifold(f)
    if chi is not None:
        assert M.euler(v, f) == chi
    assert M.signed_volume(v, f) > 0


def test_sphere_volume_and_normals_at_128():
    r = 0.6
    field, o, h = _sphere(128, r)
    v, f, nrm = _check_against_numpy(field, o, h, 0.0, faces_too=False)
    f = f.astype(np.int64)
    assert M.is_closed_manifold(f) and M.euler(v, f) == 2
    vol = M.signed_volume(v, f)
    assert abs(vol / (4.0 / 3.0 * math.pi * r ** 3) - 1.0) < 0.01
    radial = v / np.linalg.norm(v, axis=1, keepdims=True)
    assert np.all(np.einsum("ij,ij->i", nrm, radial) > 0.99)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    fn = np.cross(b - a, c - a)
    assert np.mean(np.einsum("ij,ij->i", fn, (a + b + c)) > 0) > 0.999


def test_open_field_boundary_edges_on_grid_faces():
    field, o, h = _sphere(40, 0.8, (0.5, 0.0, 0.0))   # cut by the x = 1 face
    v, f, _ = _check_against_numpy(field, o, h, 0.0)
    (de, dc), (ue, uc) = M.edge_counts(f)
    assert np.all(dc == 1) and np.all(uc <= 2) and np.any(uc == 1)
    bverts = v[np.unique(ue[uc == 1])]
    on_face = np.any(np.isclose(bverts, -1.0, atol=1e-6) | np.isclose(bverts, 1.0, atol=1e-6), axis=1)
    assert np.all(on_face)


def test_degenerate_fields():
    # constant: no crossings
    c = torch.full((9, 10, 11), 0.25, device=DEV)
    v, f, nrm = _mc(c, (0, 0, 0), (1, 1, 1), 0.0)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    # corners exactly at level are outside: vertices may sit on grid points (zero-area triangles allowed only there)
    field, o, h = _sphere(33, 0.5)
    q = torch.round(field * 8) / 8   # many values exactly 0
    v, f, nrm = _check_against_numpy(q, o, h, 0.0)
    assert M.is_closed_manifold(f)
    P = M.grid_points(o, h, (33, 33, 33)).reshape(-1, 3)
    a, b, cc = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    zero = np.linalg.norm(np.cross(b - a, cc - a), axis=1) == 0
    if zero.any():
        on_corner = lambda x: np.isin(x.view(np.uint32).sum(1), P.view(np.uint32).sum(1))
        assert np.all(on_corner(a[zero]) | on_corner(b[zero]) | on_corner(cc[zero]))
    # NaN counts as outside
    n = field.clone()
    n[16, 16, 16] = float("nan")
    v, f, nrm = _check_against_numpy(n, o, h, 0.0)
    assert M.is_closed_manifold(f)
    assert np.all(np.isfinite(v)) and np.all(np.isfinite(nrm))
    # a NaN inside the stencil of a crossing's endpoint: that vertex's normal is (0, 0, 0)
    n2 = field.clone()
    cross = torch.nonzero((field[:, :, :-1] > 0) != (field[:, :, 1:] > 0))[0].tolist()
    n2[cross[0] + 1, cross[1], cross[2]] = float("nan")   # a neighbour of the crossing's lower endpoint, outside the edge
    v, f, nrm = _mc(n2, o, h, 0.0)
    assert torch.all(torch.isfinite(nrm)) and bool((nrm.abs().sum(1) == 0).any())


def test_host_field_is_meshed_and_returned_on_the_host():
    field, o, h = _sphere(24, 0.6)
    vd, fd, nd = _mc(field, o, h, 0.0)
    vh, fh, nh = _mc(field.cpu(), o, h, 0.0)
    assert vh.device.type == "cpu" and fh.device.type == "cpu" and nh.device.type == "cpu"
    assert torch.equal(vh, vd.cpu()) and torch.equal(fh, fd.cpu()) and torch.equal(nh, nd.cpu())


def test_large_grid_and_determinism():
    """More than 2^24 cells; two runs give bit-identical results."""
    n = 260
    X, Y, Z, o, h = _coords(n)
    field = 0.7 - torch.sqrt(X ** 2 + Y ** 2 + Z ** 2) + 0.05 * torch.sin(9 * X) * torch.cos(7 * Y)
    assert (n - 1) ** 3 > 2 ** 24
    v1, f1, n1 = _mc(field, o, h, 0.0)
    v2, f2, n2 = _mc(field, o, h, 0.0)
    assert torch.equal(v1, v2) and torch.equal(f1, f2) and torch.equal(n1, n2)
    vr = _numpy_vertices(field.cpu().numpy(), o, h, 0.0)
    assert v1.shape[0] == vr.shape[0]
    assert np.all(np.abs(v1.cpu().numpy() - vr) <= 1e-6 * np.float32(h[0]))
    f = f1.cpu().numpy().astype(np.int64)
    assert M.is_closed_manifold(f) and M.euler(v1.cpu().numpy(), f) == 2


# ---- extract_mesh ------------------------------------------------------------------------------------------------------
def _extract_case(name):
    if name == "bench_hull":
        scene = syn.make_scene(512, 3, 18, fg_mode="hull")
        net = build_model(syn.make_weights(18), 18, DEV)
        return scene, net
    g, meta, sha = load_golden(name)
    scene, weights, _ = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    return scene, build_model(weights, meta["n_kpt"], DEV)


@pytest.mark.parametrize("name", ["bench_hull", "rect_v4_k17"])
def test_extract_mesh_equals_its_parts(name):
    scene, net = _extract_case(name)
    a = scene_tensors(scene, syn.make_target(size=16), DEV)
    res_n = 96
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    origin, spacing, dims = KeypointNeRF.mesh_grid(a["bounds"], res_n)
    out2, valid = m.query_grid(origin, spacing, dims, engine=net.engine)
    dens = out2[..., 1].clamp_min(0) * valid
    level = float(dens[dens > 0].median())
    with torch.no_grad():
        res = KeypointNeRF.extract_mesh(net, a["img"], a["cam"], a["sp_data"], a["bounds"], level, resolution=res_n,
                                        src_foreground_mask=a["fg"], feat_geo=a["feat_geo"], feat_tex=a["feat_tex"])
    field = torch.nn.functional.pad(dens, (1, 1, 1, 1, 1, 1))
    v, f, nrm = m.marching_cubes(field, tuple(o - h for o, h in zip(origin, spacing)), spacing, level)
    torch.cuda.synchronize()
    assert res["vertices"].shape[0] > 100
    assert torch.equal(res["vertices"], v) and torch.equal(res["faces"], f) and torch.equal(res["normals"], nrm)
    assert M.is_closed_manifold(f.cpu().numpy().astype(np.int64))
    q, _ = m.query(v, -nrm, engine=net.engine)
    assert torch.equal(res["colors"], q[:, 2:5])
    # a level above every density gives an empty mesh, with empty colours
    with torch.no_grad():
        empty = KeypointNeRF.extract_mesh(net, a["img"], a["cam"], a["sp_data"], a["bounds"], float(dens.max()) + 1.0,
                                          resolution=32, src_foreground_mask=a["fg"], feat_geo=a["feat_geo"], feat_tex=a["feat_tex"])
    assert all(empty[k].shape == (0, 3) for k in ("vertices", "faces", "normals", "colors"))


# ---- against the reference (tests/golden/make_golden_grid.py) -----------------------------------------------------------
TOL_RGB = {0: 1e-3, 1: 1e-4}   # the RGB gates of test_gpu_parity.TOL


@pytest.mark.parametrize("name,engine", [("grid_tiny", 0), ("grid_tiny", 1), ("grid_rect_v4_k17", 0), ("grid_rect_v4_k17", 1),
                                         ("grid_v2", 1)])
def test_query_grid_matches_reference(name, engine):
    g, meta, sha = load_golden(name)
    scene, weights, _ = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    net = build_model(weights, meta["n_kpt"], DEV)
    m, _ = _bound(net, scene)
    gr = meta["grid"]
    out2, valid = m.query_grid(gr["origin"], gr["spacing"], gr["dims"], engine=engine)
    out2, valid = out2.reshape(-1, 2).cpu().numpy(), valid.reshape(-1).cpu().numpy()
    v = g["grid_valid"]
    assert np.array_equal(valid, v)
    assert np.all(out2[~v] == 0.0)
    e_sdf = np.abs(out2[v, 0] - g["grid_out"][v, 0]).max()
    e_rad = np.abs(out2[v, 1] - g["grid_out"][v, 1]).max()
    print(f"{name} engine {engine}: sdf_raw {e_sdf:.2e} rad {e_rad:.2e}")
    assert e_sdf <= 10 * TOL_RGB[engine] and e_rad <= (5e-2 if engine != 1 else 3e-3)
