"""Host-memory (KPN_MEM_HOST) paths of the C ABI against the device paths, and the refusals of bad memory kinds and of too many
rays.

Every entry point that takes host arrays stages them through the context's device buffers; its results must equal the device
path's bit for bit.  The calls go through ``RayMarcher.lib`` / ``.ctx`` directly, because the Python wrappers always pass device
memory for the grid query and the mesh, and always pass a validity mask to the point query.
"""
import ctypes as C

import pytest
import torch

from keypointnerf_b200 import _lib as L
from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model, scene_tensors

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BAD_MEM = 2   # neither KPN_MEM_DEVICE nor KPN_MEM_HOST


@pytest.fixture(scope="module")
def bound():
    """(marcher with a 3-view, 18-keypoint scene bound, scene tensors, scene)"""
    scene = syn.make_scene(src_size=64, n_kpt=18, fg_mode="hull", fg_hole=True)
    net = build_model(syn.make_weights(18), 18, DEV)
    target = syn.make_target(size=32, zoom=2.0)
    a = scene_tensors(scene, target, DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    yield m, a, scene, target
    m.check_health()


def _host(t):
    return t.cpu().pin_memory()


def _nan_like(t, pinned):
    """t's shape and dtype filled with NaN (0xFF bytes) on the device or in pinned host memory, so that every output is written"""
    out = torch.empty(t.shape, dtype=t.dtype, pin_memory=True) if pinned else torch.empty_like(t, device=DEV)
    out.view(torch.uint8).fill_(0xFF)
    return out


def _same_bits(a, b):
    a, b = a.cpu().contiguous(), b.cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _run(m, rc, what):
    L.check(m.lib, m.ctx, rc, what)
    torch.cuda.current_stream().synchronize()


def _opts(engine=0, S_c=8):
    op = L.KpnOpts()
    op.engine, op.sample_per_ray_c = engine, S_c
    return op


def _ptr(t):
    return None if t is None else t.data_ptr()


def test_query_host_path(bound):
    """kpn_query over more than 4 Mi points (two chunks), with and without a validity mask"""
    m, a, scene, _ = bound
    n = (4 << 20) + 4099
    gen = torch.Generator().manual_seed(3)
    b = torch.from_numpy(scene["bounds"]).reshape(2, 3)
    pts = b[0] + (b[1] - b[0]) * torch.rand(n, 3, generator=gen)
    view = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen), dim=-1)
    out5 = torch.empty(n, 5)
    valid = torch.empty(n, dtype=torch.uint8)
    op = _opts()
    res = {}
    for mem in (L.KPN_MEM_DEVICE, L.KPN_MEM_HOST):
        host = mem == L.KPN_MEM_HOST
        p, v = (_host(pts), _host(view)) if host else (pts.to(DEV), view.to(DEV))
        for with_valid in (True, False):
            o, va = _nan_like(out5, host), (_nan_like(valid, host) if with_valid else None)
            _run(m, m.lib.kpn_query(m.ctx, p.data_ptr(), v.data_ptr(), n, o.data_ptr(), _ptr(va), mem, C.byref(op), m._stream()),
                 "kpn_query")
            res[mem, with_valid] = (o, va)
    ref_out, ref_valid = res[L.KPN_MEM_DEVICE, True]
    assert 0 < int(ref_valid.sum()) < n
    for (mem, with_valid), (o, va) in res.items():
        assert _same_bits(o, ref_out), (mem, with_valid)
        assert va is None or _same_bits(va, ref_valid), (mem, with_valid)


def test_query_grid_host_path(bound):
    """kpn_query_grid over more than 4 Mi nodes (two chunks), with and without a validity mask"""
    m, a, scene, _ = bound
    dims = (161, 163, 165)   # 4 330 395 nodes
    b = torch.from_numpy(scene["bounds"]).reshape(2, 3).double()
    g = L.KpnGrid()
    g.origin[:] = [float(x) for x in b[0]]
    g.spacing[:] = [float(x) for x in (b[1] - b[0]) / (torch.tensor(dims, dtype=torch.float64) - 1)]
    g.nx, g.ny, g.nz = dims
    n = dims[0] * dims[1] * dims[2]
    out2, valid = torch.empty(n, 2), torch.empty(n, dtype=torch.uint8)
    op = _opts()
    res = {}
    for mem in (L.KPN_MEM_DEVICE, L.KPN_MEM_HOST):
        host = mem == L.KPN_MEM_HOST
        for with_valid in (True, False):
            o, va = _nan_like(out2, host), (_nan_like(valid, host) if with_valid else None)
            _run(m, m.lib.kpn_query_grid(m.ctx, C.byref(g), o.data_ptr(), _ptr(va), mem, C.byref(op), m._stream()), "kpn_query_grid")
            res[mem, with_valid] = (o, va)
    ref_out, ref_valid = res[L.KPN_MEM_DEVICE, True]
    assert 0 < int(ref_valid.sum()) < n
    for (mem, with_valid), (o, va) in res.items():
        assert _same_bits(o, ref_out), (mem, with_valid)
        assert va is None or _same_bits(va, ref_valid), (mem, with_valid)


def _target(a, target, mem, nx=32, ny=32):
    K = a["cam_tar"]["K"].reshape(-1, 4, 4)[0].float().contiguous()
    RT = a["cam_tar"]["RT"].reshape(-1, 4, 4)[0].float().contiguous()
    K, RT = (_host(K), _host(RT)) if mem == L.KPN_MEM_HOST else (K.to(DEV), RT.to(DEV))
    tg = L.KpnTarget()
    tg.K, tg.RT, tg.znear, tg.zfar = K.data_ptr(), RT.data_ptr(), float(target["znear"]), float(target["zfar"])
    tg.x0, tg.y0, tg.step, tg.nx, tg.ny, tg.step_y, tg.mem = 0, 0, 1, nx, ny, 0, mem
    return tg, (K, RT)


def test_camera_rays_host_outputs(bound):
    m, a, _, target = bound
    n = 32 * 32
    res = {}
    for mem in (L.KPN_MEM_DEVICE, L.KPN_MEM_HOST):
        tg, keep = _target(a, target, mem)
        arrs = [_nan_like(torch.empty(n, w), mem == L.KPN_MEM_HOST) for w in (3, 3, 2)]
        _run(m, m.lib.kpn_camera_rays(m.ctx, C.byref(tg), *(t.data_ptr() for t in arrs), mem, m._stream()), "kpn_camera_rays")
        res[mem] = arrs
    for h, d in zip(res[L.KPN_MEM_HOST], res[L.KPN_MEM_DEVICE]):
        assert _same_bits(h, d)


PLANES = {"tex_fg": 3, "depth": 1, "alpha": 1, "tex_fg_fine": 3, "depth_fine": 1, "alpha_fine": 1, "sdf": 1}


def test_render_host_target_and_outputs(bound):
    """kpn_render with a host target and host outputs, including the z_fine and contrib debug outputs"""
    m, a, _, target = bound
    S_c, S_f, n = 16, 8, 32 * 32
    op = _opts(S_c=S_c)
    op.sample_per_ray_f, op.fine = S_f, 1
    shapes = {k: (c, n) for k, c in PLANES.items()}
    shapes.update(z_fine=(n, S_c + S_f), contrib=(n, S_c))
    res = {}
    for mem in (L.KPN_MEM_DEVICE, L.KPN_MEM_HOST):
        tg, keep = _target(a, target, mem)
        outs = {k: _nan_like(torch.empty(s), mem == L.KPN_MEM_HOST) for k, s in shapes.items()}
        out = L.KpnOut()
        for k, t in outs.items():
            setattr(out, k, t.data_ptr())
        out.mem = mem
        _run(m, m.lib.kpn_render(m.ctx, C.byref(tg), C.byref(op), C.byref(out), m._stream()), "kpn_render")
        res[mem] = outs
    assert float(res[L.KPN_MEM_DEVICE]["alpha"].max()) > 0.0
    for k in shapes:
        assert _same_bits(res[L.KPN_MEM_HOST][k], res[L.KPN_MEM_DEVICE][k]), k


def test_mesh_emit_host_outputs(bound):
    """kpn_mesh_emit into host vertices / faces, with and without normals"""
    m = bound[0]
    nz, ny, nx = 37, 41, 43
    z, y, x = torch.meshgrid(*(torch.linspace(-1.0, 1.0, k) for k in (nz, ny, nx)), indexing="ij")
    field = (1.0 - (x * x + 1.3 * y * y + 0.8 * z * z)).to(DEV).contiguous()
    counts = (C.c_longlong * 2)()
    _run(m, m.lib.kpn_mesh_begin(m.ctx, field.data_ptr(), nx, ny, nz, 0.25, counts, m._stream()), "kpn_mesh_begin")
    nv, nf = int(counts[0]), int(counts[1])
    assert nv > 0 and nf > 0
    o, h = (C.c_float * 3)(-1.0, -1.0, -1.0), (C.c_float * 3)(2.0 / (nx - 1), 2.0 / (ny - 1), 2.0 / (nz - 1))
    res = {}
    for mem in (L.KPN_MEM_DEVICE, L.KPN_MEM_HOST):
        host = mem == L.KPN_MEM_HOST
        for with_normals in (True, False):
            v, f = _nan_like(torch.empty(nv, 3), host), _nan_like(torch.empty(nf, 3, dtype=torch.int32), host)
            nrm = _nan_like(torch.empty(nv, 3), host) if with_normals else None
            _run(m, m.lib.kpn_mesh_emit(m.ctx, field.data_ptr(), o, h, v.data_ptr(), _ptr(nrm), f.data_ptr(), mem, m._stream()),
                 "kpn_mesh_emit")
            res[mem, with_normals] = (v, nrm, f)
    ref_v, ref_n, ref_f = res[L.KPN_MEM_DEVICE, True]
    for key, (v, nrm, f) in res.items():
        assert _same_bits(v, ref_v) and _same_bits(f, ref_f), key
        assert nrm is None or _same_bits(nrm, ref_n), key


def _refused(m, rc, what, text):
    assert rc == -1, what
    with pytest.raises(L.KpnError, match=f"status -1: {text}"):
        L.check(m.lib, m.ctx, rc, what)


def test_bad_mem_kinds_are_refused(bound):
    """a memory kind other than device / host is refused by every entry point that reads it (it used to pass as device memory)"""
    m, a, scene, target = bound
    op = _opts()
    tg, keep = _target(a, target, L.KPN_MEM_DEVICE, nx=4, ny=4)
    out = L.KpnOut()   # no outputs: nothing could be written even if a call went through
    out.mem = L.KPN_MEM_DEVICE
    tg.mem = BAD_MEM
    _refused(m, m.lib.kpn_render(m.ctx, C.byref(tg), C.byref(op), C.byref(out), m._stream()), "kpn_render: target", "bad mem kind")
    tg.mem, out.mem = L.KPN_MEM_DEVICE, BAD_MEM
    _refused(m, m.lib.kpn_render(m.ctx, C.byref(tg), C.byref(op), C.byref(out), m._stream()), "kpn_render: outputs", "bad mem kind")

    o, d, nf = (torch.zeros(4, w, device=DEV) for w in (3, 3, 2))
    rays = L.KpnRays()
    rays.origins, rays.dirs, rays.near_far, rays.n, rays.mem = o.data_ptr(), d.data_ptr(), nf.data_ptr(), 4, L.KPN_MEM_DEVICE
    _refused(m, m.lib.kpn_render_rays(m.ctx, C.byref(rays), C.byref(op), C.byref(out), m._stream()), "kpn_render_rays: outputs",
             "bad mem kind")
    rays.mem, out.mem = BAD_MEM, L.KPN_MEM_DEVICE
    _refused(m, m.lib.kpn_render_rays(m.ctx, C.byref(rays), C.byref(op), C.byref(out), m._stream()), "kpn_render_rays: rays",
             "bad mem kind")

    tg.mem = BAD_MEM
    ro, rd, rnf = (torch.empty(16, w, device=DEV) for w in (3, 3, 2))   # the 4 x 4 lattice's rays
    _refused(m, m.lib.kpn_camera_rays(m.ctx, C.byref(tg), ro.data_ptr(), rd.data_ptr(), rnf.data_ptr(), L.KPN_MEM_DEVICE,
                                      m._stream()), "kpn_camera_rays: target", "bad mem kind")

    pts, view = torch.zeros(4, 3, device=DEV), torch.zeros(4, 3, device=DEV)
    out5 = torch.empty(4, 5, device=DEV)
    _refused(m, m.lib.kpn_query(m.ctx, pts.data_ptr(), view.data_ptr(), 4, out5.data_ptr(), None, BAD_MEM, C.byref(op), m._stream()),
             "kpn_query", "bad mem kind")
    torch.cuda.synchronize()
    m.check_health()


def test_render_of_more_than_2_31_rays_is_refused(bound):
    """a 46 341 x 46 341 lattice (2^31 + 4 633 rays) with one sample per ray is within the sample limit but not the ray limit"""
    m, a, _, target = bound
    tg, keep = _target(a, target, L.KPN_MEM_DEVICE, nx=46341, ny=46341)
    out = L.KpnOut()   # no outputs
    out.mem = L.KPN_MEM_DEVICE
    rc = m.lib.kpn_render(m.ctx, C.byref(tg), C.byref(_opts(S_c=1)), C.byref(out), m._stream())
    _refused(m, rc, "kpn_render", "too many rays")
    m.check_health()
